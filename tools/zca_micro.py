"""Whitening in the ZCA basis at BASELINE config 2's shape; one JSON line.

    python tools/zca_micro.py [--steps 20] [--warmup 3] [--rounds 3]

N=256 C=256 56^2, group size 64, forward + backward (y = m(x), dx = grad(y, x, dy)), input built as bench.py's
microbench builds it.  Arms, alternated round by round in one process:
  chol        WTransform2d (the inverse Cholesky factor), CUDA-graph replay;
  zca_t5      ZCAWTransform2d, 5 Newton-Schulz iterations (the default), CUDA-graph replay;
  zca_t16     ZCAWTransform2d, 16 iterations, CUDA-graph replay;
  exact       ExactZCAWTransform2d (Jacobi eigendecomposition), CUDA-graph replay;
  exact_bf16  ExactZCAWTransform2d on bfloat16 x and dy, CUDA-graph replay;
  aten_t5     the same ZCA function as an ATen op sequence (tests/support/zca_reference.py: mean, bmm, the iterations,
              a grouped 1x1 convolution; autograd backward) in float32 on the same GPU, CUDA-graph replay.
Per library arm: the kernel families from one eager profiled pass (ms per iteration), dense_*_zca / dense_*_eigh among
them, and the share of the basis's dense kernels (partial reduction + per-group algebra) in that pass.  The card's name
and power limit are read in the same process.
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
sys.path.insert(0, os.path.join(ROOT, "tests", "support"))

import torch  # noqa: E402

from bench import timed_loop  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return tuple(s.strip() for s in out.split(","))
    except Exception:
        return torch.cuda.get_device_name(), None


def _step_fn(fwd, x, dy):
    def step():
        xi = x.detach().requires_grad_(True)
        y = fwd(xi)
        torch.autograd.grad(y, xi, dy)
    return step


def _families(step, steps):
    from dwt_b200 import _native
    _native.profile_begin()
    for _ in range(steps):
        step()
    prof = _native.by_family(_native.profile_end())
    return {f: round(v["ms"] / steps, 4) for f, v in sorted(prof.items())}


def _graphed(step, dev):
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
    return graph.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("zca_micro.py measures on a CUDA device; none is visible")
    import dwt_b200
    import zca_reference
    dev = torch.device("cuda", 0)
    N, C, H, GS = 256, 256, 56, 64
    torch.manual_seed(0)
    mix = torch.randn(C, C, device=dev) / C ** 0.5 + torch.eye(C, device=dev)
    x = (torch.einsum("dc,nchw->ndhw", mix, torch.randn(N, C, H, H, device=dev)) + 2.0).contiguous()
    dy = torch.randn(N, C, H, H, device=dev)
    mods = {"chol": dwt_b200.WTransform2d(C, GS), "zca_t5": dwt_b200.ZCAWTransform2d(C, GS, iterations=5),
            "zca_t16": dwt_b200.ZCAWTransform2d(C, GS, iterations=16), "exact": dwt_b200.ExactZCAWTransform2d(C, GS),
            "exact_bf16": dwt_b200.ExactZCAWTransform2d(C, GS)}
    arms, recs = {}, {}
    for name, m in mods.items():
        bf16 = name.endswith("_bf16")
        step = _step_fn(m.to(dev).train(), x.bfloat16() if bf16 else x, dy.bfloat16() if bf16 else dy)
        for _ in range(args.warmup):
            step()
        fams = _families(step, args.steps)
        arms[name] = _graphed(step, dev)
        total = sum(fams.values())
        dense = sum(v for f, v in fams.items() if f.startswith("dense_"))
        recs[name] = {"kernels_ms": fams, "kernel_ms_per_iter": round(total, 4), "dense_share": round(dense / total, 3),
                      "ms_per_iter": []}
    aten = _step_fn(lambda xi: zca_reference.zca_torch(xi, GS, 5)[0], x, dy)
    for _ in range(args.warmup):
        aten()
    arms["aten_t5"] = _graphed(aten, dev)
    recs["aten_t5"] = {"ms_per_iter": []}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            fn()
            recs[name]["ms_per_iter"].append(round(timed_loop(fn, args.steps, dev, False) / args.steps, 4))
    for r in recs.values():
        r["median_ms_per_iter"] = statistics.median(r["ms_per_iter"])
        r["spread_ms_per_iter"] = round(max(r["ms_per_iter"]) - min(r["ms_per_iter"]), 4)
    med = {k: v["median_ms_per_iter"] for k, v in recs.items()}
    name, limit = _card()
    print(json.dumps({
        "config": f"N={N} C={C} H=W={H} group_size={GS}, forward + backward", "card": name, "power_limit": limit,
        "steps": args.steps, "rounds": args.rounds, "arms": recs,
        "zca_t5_over_chol_ms": round(med["zca_t5"] - med["chol"], 4),
        "zca_t16_over_chol_ms": round(med["zca_t16"] - med["chol"], 4),
        "exact_over_chol_ms": round(med["exact"] - med["chol"], 4),
        "speedup_over_aten_t5": round(med["aten_t5"] / med["zca_t5"], 2),
    }))


if __name__ == "__main__":
    main()
