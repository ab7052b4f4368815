"""The benchmark's training step in float32 and under bf16 autocast, alternated in one process; one JSON line.

    python tools/amp_step.py [--steps 20] [--warmup 5] [--rounds 3]

The step is bench.py's: the harness ResNet-50-DWT with fused sites, channels-last, s2d stem, 3 x 64 images at 224^2,
HeadLoss, SGD, replayed from a CUDA graph.  The bf16 arm runs the model's forward under
torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False) (the cast cache cannot live across graph replays):
cuDNN's convolutions return bf16 and the library's norm sites and max-pool run their bf16 kernels.  Parameters,
gradients, optimizer and losses stay float32.

Per arm: images/s of every round (median and max - min), the library's kernel families from one eager profiled pass
(ms and algorithmic GB per step; the norm path is every family but head_loss, as in bench.py), library launches per
step; with the card's name and power limit read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "dwt-domain-adaptation_b200"))

import torch  # noqa: E402

from bench import LAMBDA_MEC, NUM_CLASSES, build_model, make_optimizer, timed_loop, train_step  # noqa: E402


class _Autocast(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, x):
        with torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False):
            return self.model(x)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), None


def _arm(name, bf16, device, images, labels, args):
    import dwt_b200
    from dwt_b200 import _native
    model = build_model(dwt_b200, device, "fused", channels_last=True, stem_s2d=True)
    net = _Autocast(model) if bf16 else model
    opt = make_optimizer(model)
    mec = dwt_b200.MinEntropyConsensusLoss(NUM_CLASSES, device)
    head = dwt_b200.HeadLoss(NUM_CLASSES, LAMBDA_MEC)

    def step():
        train_step(net, mec, opt, images, labels, None, head)
    for _ in range(args.warmup):
        step()
    n0 = _native.launch_count()
    _native.profile_begin()
    timed_loop(step, args.steps, device, False)
    fams = _native.by_family(_native.profile_end())
    launches = (_native.launch_count() - n0) // args.steps
    side = torch.cuda.Stream(device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream(device).wait_stream(side)
    torch.cuda.synchronize(device)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        train_step(net, mec, opt, images, labels, None, head)
    torch.cuda.synchronize(device)
    norm = {k: v for k, v in fams.items() if k != "head_loss"}
    rec = {"norm_path_ms_per_step": sum(v["ms"] for v in fams.values()) / args.steps,
           "norm_path_algorithmic_gb_per_step": sum(v["bytes"] for v in norm.values()) / args.steps / 1e9,
           "families": {k: {"ms_per_step": round(v["ms"] / args.steps, 4), "gb_per_step": round(v["bytes"] / args.steps / 1e9, 4)}
                        for k, v in sorted(fams.items())},
           "launches_per_step": launches, "images_per_s": []}
    # the graph replays into this arm's parameters, buffers and optimizer state: they live as long as the graph
    return graph, rec, (model, net, opt, mec, head)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--per-domain", type=int, default=64)
    args = ap.parse_args()
    from harness.synth import synth_batch
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    card, limit = _card()
    images, labels = synth_batch(seed=100, per_domain=args.per_domain)
    images = images.contiguous(memory_format=torch.channels_last).to(device)
    labels = labels.to(device)
    arms = {name: _arm(name, bf16, device, images, labels, args) for name, bf16 in (("fp32", False), ("bf16", True))}
    per_step = images.shape[0]
    for _ in range(args.rounds):
        for name, (graph, rec, _) in arms.items():
            graph.replay()
            ms = timed_loop(graph.replay, args.steps, device, False)
            rec["images_per_s"].append(round(per_step * args.steps / (ms / 1e3), 1))
    out = {"metric": "ResNet-50-DWT training step images/s, float32 vs bf16 autocast", "images_per_step": per_step,
           "steps": args.steps, "rounds": args.rounds, "gpu": card, "power_limit": limit}
    for name, (_, rec, _) in arms.items():
        ips = rec["images_per_s"]
        rec["median_images_per_s"] = statistics.median(ips)
        rec["spread_images_per_s"] = round(max(ips) - min(ips), 1)
        out[name] = rec
    out["bf16_over_fp32"] = out["bf16"]["median_images_per_s"] / out["fp32"]["median_images_per_s"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
