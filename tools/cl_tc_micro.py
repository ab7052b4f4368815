"""Channels-last whitening at group size 64 on the tensor-core kernels, against what a channels-last caller paid before
they took the layout, and against NCHW; one JSON line.

    python tools/cl_tc_micro.py [--steps 30] [--warmup 5] [--rounds 3] [--model-steps 5] [--no-model]

WTransform2d N=256 C=256 56^2 group_size=64 (BASELINE config 2), forward + backward (y = m(x), dx = grad(y, x, dy)),
replayed from a CUDA graph, arms alternated round by round, each in float32 and in bfloat16 (what torch.autocast hands
the layer after a bf16 convolution):
  a_nhwc      channels-last x and dy on the NHWC tensor-core kernels (y and dx come back channels-last);
  b_copy      channels-last x and dy on the route channels-last calls took before (functional._nhwc_tensor_core patched
              off): x copied to NCHW, the NCHW kernels (bf16: x.float() first, the float32 kernels, a cast back), y and dx
              made channels-last again for the caller;
  c_nchw      NCHW x and dy on the NCHW kernels.
Per arm: ms/iter of every round (median and max - min), the library's kernel families from one eager profiled pass (ms and
algorithmic GB per iteration), and the peak device memory one eager step adds.

Model arm (unless --no-model): the harness ResNet-50-DWT with group_size=64 (its stem site whitens in groups of 64),
fused sites, 3 x 64 images of 224^2, one training step (forward, head loss, backward), channels-last against NCHW, in
images/s (eager steps), alternated round by round.  The card's name and power limit are read in the same process.
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

from bench import timed_loop  # noqa: E402

CL = torch.channels_last
BF = torch.bfloat16


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), None


class _CopyRoute:
    """Context: channels-last whitening takes the route it took before the NHWC tensor-core kernels (the predicate off)."""

    def __enter__(self):
        from dwt_b200 import functional as F
        self.F, self.saved = F, F._nhwc_tensor_core
        F._nhwc_tensor_core = lambda *a, **k: False

    def __exit__(self, *exc):
        self.F._nhwc_tensor_core = self.saved


def _arm(name, x0, dy0, gs, device):
    """-> (module, step): one forward + backward of arm `name` on its own copy of the input."""
    import dwt_b200
    torch.manual_seed(1)
    m = dwt_b200.WTransform2d(x0.shape[1], gs).to(device).train()
    fmt = torch.contiguous_format if name == "c_nchw" else CL
    x = x0.contiguous(memory_format=fmt)
    dy = dy0.contiguous(memory_format=fmt)

    def step(keep=None):
        # a fresh leaf per step: its gradient accumulator is made on the stream the step runs on.  One that survives an
        # eager step is tied to the default stream, and autograd's end-of-backward sync with that stream is illegal
        # inside a capture (a PyTorch rule: it fails alike for every layout and dtype)
        xi = x.detach().requires_grad_(True)
        if name == "b_copy":
            with _CopyRoute():
                y = m(xi).contiguous(memory_format=CL)
                (dx,) = torch.autograd.grad(y, xi, dy)
            dx = dx.contiguous(memory_format=CL)
        else:
            y = m(xi)
            (dx,) = torch.autograd.grad(y, xi, dy)
        if keep is not None:
            keep["y"], keep["dx"] = y.detach(), dx
    return m, step


def _families(step, steps):
    from dwt_b200 import _native
    _native.profile_begin()
    for _ in range(steps):
        step()
    prof = _native.by_family(_native.profile_end())
    return {f: {"ms": round(v["ms"] / steps, 4), "algorithmic_gb": round(v["bytes"] / steps / 1e9, 4)}
            for f, v in sorted(prof.items())}


def _peak(step, device):
    torch.cuda.synchronize(device)
    base = torch.cuda.memory_allocated(device)
    torch.cuda.reset_peak_memory_stats(device)
    step()
    torch.cuda.synchronize(device)
    return round((torch.cuda.max_memory_allocated(device) - base) / 2 ** 30, 3)


def _layer(args, device):
    N, C, H = args.n, 256, 56
    torch.manual_seed(0)                             # bench.py's microbench input
    mix = torch.randn(C, C, device=device) / C ** 0.5 + torch.eye(C, device=device)
    x32 = (torch.einsum("dc,nchw->ndhw", mix, torch.randn(N, C, H, H, device=device)) + 2.0).contiguous()
    dy32 = torch.randn(N, C, H, H, device=device)
    names = [(dt, a) for dt in ("fp32", "bf16") for a in ("a_nhwc", "b_copy", "c_nchw")]
    arms, recs, eager = {}, {}, {}
    for dt, a in names:
        x0, dy0 = (x32, dy32) if dt == "fp32" else (x32.to(BF), dy32.to(BF))
        m, step = _arm(a, x0, dy0, args.gs, device)
        keep = {}
        step(keep)
        eager[(dt, a)] = keep
        for _ in range(args.warmup):
            step()
        fams = _families(step, args.steps)
        peak = _peak(step, device)
        side = torch.cuda.Stream(device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):
            for _ in range(3):
                step()
        torch.cuda.current_stream(device).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        graph.replay()
        torch.cuda.synchronize(device)
        arms[(dt, a)] = (graph, m, step)
        recs[(dt, a)] = {"kernels": fams,
                         "kernel_ms_per_iter": round(sum(v["ms"] for v in fams.values()), 4),
                         "algorithmic_gb_per_iter": round(sum(v["algorithmic_gb"] for v in fams.values()), 4),
                         "peak_gib_added": peak, "ms_per_iter": []}
    for _ in range(args.rounds):
        for key in names:
            graph = arms[key][0]
            graph.replay()
            recs[key]["ms_per_iter"].append(round(timed_loop(graph.replay, args.steps, device, False) / args.steps, 4))
    out = {}
    for dt, a in names:
        r = recs[(dt, a)]
        r["median_ms_per_iter"] = statistics.median(r["ms_per_iter"])
        r["spread_ms_per_iter"] = round(max(r["ms_per_iter"]) - min(r["ms_per_iter"]), 4)
        out.setdefault(dt, {})[a] = r
    for dt in ("fp32", "bf16"):
        e = {a: eager[(dt, a)] for a in ("a_nhwc", "b_copy", "c_nchw")}
        out[dt]["a_equals_c"] = bool(torch.equal(e["a_nhwc"]["y"].contiguous(), e["c_nchw"]["y"])
                                     and torch.equal(e["a_nhwc"]["dx"].contiguous(), e["c_nchw"]["dx"]))
        out[dt]["speedup_a_over_b"] = round(out[dt]["b_copy"]["median_ms_per_iter"] / out[dt]["a_nhwc"]["median_ms_per_iter"], 3)
        out[dt]["speedup_a_over_c"] = round(out[dt]["c_nchw"]["median_ms_per_iter"] / out[dt]["a_nhwc"]["median_ms_per_iter"], 3)
    return out


def _model(args, device):
    """ResNet-50-DWT at group_size=64, fused sites, one training step, channels-last vs NCHW: images/s."""
    import dwt_b200
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    sd = {k: v.to(device) for k, v in synth_state_dict(seed=1).items()}
    sd["bn1.wh.running_variance"] = synth_state_dict(seed=1, group_size=64, with_convs=False)["bn1.wh.running_variance"].to(device)
    images, labels = synth_batch(seed=2, per_domain=args.per_domain, size=224)
    images, labels = images.to(device), labels.to(device)
    head = dwt_b200.HeadLoss(65, 0.1)
    steps = {}
    for fmt in ("channels_last", "nchw"):
        cl = fmt == "channels_last"
        model = build_resnet50_dwt({k: v.clone() for k, v in sd.items()}, dwt_b200, site_mode="fused", channels_last=cl,
                                   group_size=64).to(device).train()
        x = images.contiguous(memory_format=CL) if cl else images.contiguous()

        def step(model=model, x=x):
            loss = head(model(x), labels)
            loss.backward()
            model.zero_grad(set_to_none=True)
        for _ in range(2):
            step()
        steps[fmt] = step
    ips = {fmt: [] for fmt in steps}
    for _ in range(args.rounds):
        for fmt, step in steps.items():
            ms = timed_loop(step, args.model_steps, device, False) / args.model_steps
            ips[fmt].append(round(images.shape[0] / (ms / 1e3), 1))
    out = {"config": f"harness ResNet-50-DWT group_size=64, fused sites, {images.shape[0]} images of 224^2, one training step"}
    for fmt, v in ips.items():
        out[fmt] = {"images_per_s": v, "median_images_per_s": statistics.median(v), "spread_images_per_s": round(max(v) - min(v), 1)}
    out["speedup_channels_last_over_nchw"] = round(out["channels_last"]["median_images_per_s"] / out["nchw"]["median_images_per_s"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--gs", type=int, default=64)
    ap.add_argument("--per-domain", type=int, default=64)
    ap.add_argument("--model-steps", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    card, limit = _card()
    from dwt_b200 import _native
    out = {"metric": "channels-last WTransform2d gs 64 fwd+bwd ms/iter: NHWC tensor-core kernels vs NCHW copy vs NCHW input",
           "config": f"N={args.n} C=256 H=W=56 group_size={args.gs}, cuda-graph replay", "steps": args.steps,
           "rounds": args.rounds, "gpu": card, "power_limit": limit}
    out.update(_layer(args, device))
    torch.cuda.empty_cache()
    if not args.no_model:
        out["model"] = _model(args, device)
    out["status_word"] = _native.status_all(device)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
