"""NCHW norm sites in float32 and in bfloat16, with and without the bf16 small-group kernels, alternated; one JSON line.

    python tools/amp_nchw.py [--steps 10] [--warmup 3] [--rounds 3] [--per-domain 64] [--workloads modules,fused,stem]

Workloads (NCHW throughout, the layout the reference scripts run):
  modules  the harness ResNet-50-DWT with site_mode="modules" (split -> 3 modules -> cat -> affine -> relu, the
           reference's topology as the drop-in layers run it), 3 x per-domain images at 224^2, full training step
           (forward, HeadLoss, backward, SGD);
  fused    the same model with site_mode="fused" (one DomainTripleNorm call per site);
  stem     the stem site alone: DomainTripleNorm("whiten", 64, 4) with gamma / beta / ReLU on 3 x per-domain x 64 x 112^2,
           forward + backward.
Arms, per workload:
  fp32    float32 activations;
  bf16    torch.autocast(bfloat16) (the stem: bf16 input and gradient) on the bf16 small-group kernels;
  upcast  the same bf16 step with functional._bf16_small patched to False in-process: every NCHW bf16 norm call at group
          sizes 1, 2, 4 runs the float32 kernels on upcast copies, as before those kernels had a bf16 build.
Each step is replayed from a CUDA graph when it captures (else timed eager; `timing` says which).  The arms alternate
for --rounds rounds; per arm: ms per step and images/s of every round, median and max - min.  One profiled eager pass
per arm, run separately, gives the library's norm path: ms and algorithmic GB per step and per kernel family.  The
card's name and power limit are read in the same process.
"""
from __future__ import annotations

import argparse
import contextlib
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

ARMS = ("fp32", "bf16", "upcast")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), None


@contextlib.contextmanager
def _routing(arm):
    """The upcast arm: the bf16 small-group routing patched off for the duration."""
    from dwt_b200 import functional as F
    if arm != "upcast":
        yield
        return
    keep = F._bf16_small
    F._bf16_small = lambda *a, **k: False
    try:
        yield
    finally:
        F._bf16_small = keep


class _Autocast(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, x):
        with torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False):
            return self.model(x)


def _model_arm(arm, site_mode, device, images, labels):
    """-> (step, images per step, objects the step keeps alive)"""
    import dwt_b200
    model = build_model(dwt_b200, device, site_mode)
    net = model if arm == "fp32" else _Autocast(model)
    opt = make_optimizer(model)
    mec = dwt_b200.MinEntropyConsensusLoss(NUM_CLASSES, device)
    head = dwt_b200.HeadLoss(NUM_CLASSES, LAMBDA_MEC)

    def step():
        train_step(net, mec, opt, images, labels, None, head)
    return step, images.shape[0], (model, net, opt, mec, head)


def _stem_arm(arm, device, per_domain):
    import dwt_b200
    gen = torch.Generator(device=device).manual_seed(3)
    shape = (3 * per_domain, 64, 112, 112)
    x0 = torch.randn(shape, device=device, generator=gen).add_(0.5)
    dy = torch.randn(shape, device=device, generator=gen)
    if arm != "fp32":
        x0, dy = x0.to(torch.bfloat16), dy.to(torch.bfloat16)
    mods = [dwt_b200.WTransform2d(64, 4).to(device).train() for _ in range(3)]
    site = dwt_b200.DomainTripleNorm("whiten", 64, 4)
    gamma = torch.ones(64, 1, 1, device=device, requires_grad=True)
    beta = torch.zeros(64, 1, 1, device=device, requires_grad=True)

    def step():
        x = x0.detach().requires_grad_(True)          # a fresh leaf per step (no accumulator across a capture)
        y = site(x, mods, gamma, beta, relu=True)
        torch.autograd.grad(y, (x, gamma, beta), dy)
    return step, shape[0], (x0, dy, mods, site, gamma, beta)


def _capture(step, device):
    """A CUDA graph of one step, or None when the step does not capture."""
    try:
        side = torch.cuda.Stream(device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):
            for _ in range(3):
                step()
        torch.cuda.current_stream(device).wait_stream(side)
        torch.cuda.synchronize(device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        graph.replay()
        torch.cuda.synchronize(device)
        return graph
    except RuntimeError as e:
        print(f"# capture failed, timing eager: {str(e).splitlines()[0]}", file=sys.stderr)
        torch.cuda.synchronize(device)
        return None


def _profile(step, steps):
    from dwt_b200 import _native
    _native.profile_begin()
    for _ in range(steps):
        step()
    fams = _native.by_family(_native.profile_end())
    norm = {k: v for k, v in fams.items() if k != "head_loss"}
    return {"norm_path_ms_per_step": round(sum(v["ms"] for v in norm.values()) / steps, 3),
            "norm_path_algorithmic_gb_per_step": round(sum(v["bytes"] for v in norm.values()) / steps / 1e9, 3),
            "families": {k: {"ms": round(v["ms"] / steps, 4), "gb": round(v["bytes"] / steps / 1e9, 4),
                             "launches": v["launches"] // steps} for k, v in sorted(norm.items())}}


def run_workload(name, args, device):
    from harness.synth import synth_batch
    images = labels = None
    if name != "stem":
        images, labels = synth_batch(seed=100, per_domain=args.per_domain)
        images, labels = images.contiguous().to(device), labels.to(device)
    arms = {}
    for arm in ARMS:
        with _routing(arm):
            step, per_step, keep = (_stem_arm(arm, device, args.per_domain) if name == "stem"
                                    else _model_arm(arm, name, device, images, labels))
            for _ in range(args.warmup):
                step()
            prof = _profile(step, args.profile_steps)
            graph = _capture(step, device)
        arms[arm] = {"step": step, "graph": graph, "keep": keep, "per_step": per_step, "ms": [], "prof": prof}
    for _ in range(args.rounds):
        for arm in ARMS:
            a = arms[arm]
            with _routing(arm):
                fn = a["graph"].replay if a["graph"] is not None else a["step"]
                fn()
                ms = timed_loop(fn, args.steps, device, False) / args.steps
            a["ms"].append(round(ms, 3))
    out = {}
    for arm in ARMS:
        a = arms[arm]
        med = statistics.median(a["ms"])
        out[arm] = {"timing": "cuda-graph replay" if a["graph"] is not None else "eager",
                    "ms_per_step": a["ms"], "median_ms_per_step": med, "spread_ms": round(max(a["ms"]) - min(a["ms"]), 3),
                    "median_images_per_s": round(a["per_step"] * 1e3 / med, 1), **a["prof"]}
    out["bf16_speedup_over_upcast"] = round(out["upcast"]["median_ms_per_step"] / out["bf16"]["median_ms_per_step"], 3)
    out["bf16_speedup_over_fp32"] = round(out["fp32"]["median_ms_per_step"] / out["bf16"]["median_ms_per_step"], 3)
    del arms
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--per-domain", type=int, default=64)
    ap.add_argument("--workloads", default="modules,fused,stem")
    args = ap.parse_args()
    if args.rounds < 3:
        ap.error("--rounds must be at least 3")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    card, limit = _card()
    out = {"metric": "NCHW norm sites: float32 vs bf16 small-group kernels vs bf16 upcast, ms/step and images/s",
           "per_domain": args.per_domain, "steps": args.steps, "rounds": args.rounds, "gpu": card, "power_limit": limit}
    for name in args.workloads.split(","):
        out[name] = run_workload(name, args, device)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
