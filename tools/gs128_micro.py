"""Whitening at group size 128 at BASELINE config 2's shape; one JSON line.

    python tools/gs128_micro.py [--steps 20] [--warmup 3] [--rounds 3]

WTransform2d N=256 C=256 56^2, forward + backward (y = m(x), dx = grad(y, x, dy)), input built as bench.py's microbench
builds it.  Arms, alternated round by round in one process:
  gs128_nchw   group size 128, NCHW, CUDA-graph replay;
  gs128_nhwc   group size 128, channels-last x and dy, CUDA-graph replay;
  gs64_nchw    group size 64, NCHW, CUDA-graph replay (the benchmark's own layer, for scale);
  ref_gs128    the reference's operator sequence (oracle/torch_port.py) on the GPU at group size 128, eager (its
               Cholesky and inverse are not capturable).
Per tensor-core arm: the library's kernel families from one eager profiled pass (ms and algorithmic GB per iteration), and
the lower bound from shapes: max(algorithmic bytes / 3.35 TB/s, tf32 tensor-core flops / 495 TFLOP/s) -- H100 SXM data
sheet rates -- naming which of the two binds.  The card's name and power limit are read in the same process.

Nobody's model reaches this shape at group size 128 today (the reference ResNet forwards group_size only to its stem
site); it measures the layer as a user's own network would call it.
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

HBM_BPS = 3.35e12           # H100 SXM HBM3, data sheet
TF32_FLOPS = 495e12         # H100 SXM dense TF32 tensor core, data sheet
MMA = 2 * 64 * 64           # flops of one 64 x 64 block product per pixel


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return tuple(s.strip() for s in out.split(","))
    except Exception:
        return torch.cuda.get_device_name(), None


def bound(n, c, hw, gs, elem_bytes=4):
    """Least time of one forward + backward from shapes: algorithmic bytes (stats x, apply x + y, bwd reduce x + dy,
    bwd apply x + dy + dx) and the tf32 block products the kernels issue per pixel.  Group size 128, per group: Gram 2 x 2
    split products on the diagonal blocks + 3 off it; apply 2 output blocks x 2 halves x 4 split products; R 4 blocks x 1;
    bwd apply 2 x 2 x 2 inputs x 4.  Group size <= 64, per 64-channel super-block: 2, 4, 1, 8."""
    pixels, e = n * hw, elem_bytes * n * c * hw
    if gs == 128:
        per = {"stats": 7, "apply": 16, "bwd_reduce": 4, "bwd_apply": 32}
        units = c // 128
    else:
        per = {"stats": 2, "apply": 4, "bwd_reduce": 1, "bwd_apply": 8}
        units = c // 64
    byts = {"stats": e, "apply": 2 * e, "bwd_reduce": 2 * e, "bwd_apply": 3 * e}
    out = {}
    for k in per:
        fl = per[k] * MMA * pixels * units
        tb, tf = byts[k] / HBM_BPS * 1e3, fl / TF32_FLOPS * 1e3
        out[k] = {"gb": round(byts[k] / 1e9, 3), "tflop": round(fl / 1e12, 3), "ms_bytes": round(tb, 3), "ms_flops": round(tf, 3),
                  "bound_by": "bytes" if tb >= tf else "tf32 flops"}
    out["total_ms"] = round(sum(max(v["ms_bytes"], v["ms_flops"]) for v in out.values()), 3)
    return out


def _step_fn(m, x, dy, keep=None):
    def step():
        xi = x.detach().requires_grad_(True)          # a fresh leaf per step (capturable: see tools/cl_tc_micro.py)
        y = m(xi)
        (dx,) = torch.autograd.grad(y, xi, dy)
        if keep is not None:
            keep["y"], keep["dx"] = y.detach(), dx
    return step


def _families(step, steps):
    from dwt_b200 import _native
    _native.profile_begin()
    for _ in range(steps):
        step()
    prof = _native.by_family(_native.profile_end())
    return {f: {"ms": round(v["ms"] / steps, 4), "algorithmic_gb": round(v["bytes"] / steps / 1e9, 4)} for f, v in sorted(prof.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gs128_micro.py measures on a CUDA device; none is visible")
    import dwt_b200
    import oracle.torch_port as port
    dev = torch.device("cuda", 0)
    N, C, H = args.n, 256, 56
    torch.manual_seed(0)
    mix = torch.randn(C, C, device=dev) / C ** 0.5 + torch.eye(C, device=dev)
    x = (torch.einsum("dc,nchw->ndhw", mix, torch.randn(N, C, H, H, device=dev)) + 2.0).contiguous()
    dy = torch.randn(N, C, H, H, device=dev)
    arms, recs, eager = {}, {}, {}
    for name, gs, fmt in (("gs128_nchw", 128, torch.contiguous_format), ("gs128_nhwc", 128, torch.channels_last),
                          ("gs64_nchw", 64, torch.contiguous_format)):
        m = dwt_b200.WTransform2d(C, gs).to(dev).train()
        xa, dya = x.contiguous(memory_format=fmt), dy.contiguous(memory_format=fmt)
        keep = {}
        _step_fn(m, xa, dya, keep)()
        eager[name] = keep
        step = _step_fn(m, xa, dya)
        for _ in range(args.warmup):
            step()
        fams = _families(step, args.steps)
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(3):
                step()
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        graph.replay()
        torch.cuda.synchronize(dev)
        arms[name] = graph.replay
        b = bound(N, C, H * H, gs)
        recs[name] = {"kernels": fams, "kernel_ms_per_iter": round(sum(v["ms"] for v in fams.values()), 4),
                      "algorithmic_gb_per_iter": round(sum(v["algorithmic_gb"] for v in fams.values()), 4),
                      "lower_bound": b, "ms_per_iter": []}
    ref = port.WTransform2d(C, 128).to(dev).train()
    ref_step = _step_fn(ref, x, dy)
    for _ in range(args.warmup):
        ref_step()
    arms["ref_gs128"] = ref_step
    recs["ref_gs128"] = {"ms_per_iter": []}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            fn()
            recs[name]["ms_per_iter"].append(round(timed_loop(fn, args.steps, dev, False) / args.steps, 4))
    for r in recs.values():
        r["median_ms_per_iter"] = statistics.median(r["ms_per_iter"])
        r["spread_ms_per_iter"] = round(max(r["ms_per_iter"]) - min(r["ms_per_iter"]), 4)
        if "lower_bound" in r:
            r["share_of_lower_bound"] = round(r["lower_bound"]["total_ms"] / r["median_ms_per_iter"], 3)
    name, limit = _card()
    print(json.dumps({
        "config": f"WTransform2d N={N} C={C} H=W={H}, forward + backward", "card": name, "power_limit": limit,
        "steps": args.steps, "rounds": args.rounds, "arms": recs,
        "nhwc_equals_nchw": bool(torch.equal(eager["gs128_nhwc"]["y"].contiguous(), eager["gs128_nchw"]["y"])
                                 and torch.equal(eager["gs128_nhwc"]["dx"].contiguous(), eager["gs128_nchw"]["dx"])),
        "speedup_over_ref_gs128": round(recs["ref_gs128"]["median_ms_per_iter"] / recs["gs128_nchw"]["median_ms_per_iter"], 2),
    }))


if __name__ == "__main__":
    main()
