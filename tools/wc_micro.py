"""Whitening followed by a learnable colouring at BASELINE config 2's shape; one JSON line.

    python tools/wc_micro.py [--steps 20] [--warmup 3] [--rounds 3]

N=256 C=256 56^2, group size 64, forward + backward (y = m(x); dx, and dweight / dbias where there are parameters), the
input built as bench.py's microbench builds it, a non-trivial colouring (I + 0.3 randn / sqrt(gs)).  Arms, alternated
round by round in one process, each replayed from a CUDA graph:
  w           WTransform2d (whitening only);
  wc          WCTransform2d: colouring inside the whitening kernels (dwt_whiten_color_*);
  wc_bf16     WCTransform2d on bfloat16 x and dy;
  w_conv      WTransform2d followed by a grouped 1x1 F.conv2d with bias (cuDNN): the same function unfused.
Per library arm: the kernel families from one eager profiled pass (ms per iteration).  The card's name and power limit
are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "dwt-domain-adaptation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
import torch.nn.functional as Fn  # noqa: E402

from bench import timed_loop  # noqa: E402
from zca_micro import _card, _families, _graphed  # noqa: E402


def _step_fn(fwd, x, dy, params):
    def step():
        xi = x.detach().requires_grad_(True)
        torch.autograd.grad(fwd(xi), (xi, *params), dy)
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wc_micro.py measures on a CUDA device; none is visible")
    import dwt_b200
    dev = torch.device("cuda", 0)
    N, C, H, GS = 256, 256, 56, 64
    G = C // GS
    torch.manual_seed(0)
    mix = torch.randn(C, C, device=dev) / C ** 0.5 + torch.eye(C, device=dev)
    x = (torch.einsum("dc,nchw->ndhw", mix, torch.randn(N, C, H, H, device=dev)) + 2.0).contiguous()
    dy = torch.randn(N, C, H, H, device=dev)
    color = torch.eye(GS, device=dev) + 0.3 * torch.randn(G, GS, GS, device=dev) / GS ** 0.5
    bias = 0.1 * torch.randn(C, device=dev)

    def wc():
        m = dwt_b200.WCTransform2d(C, GS).to(dev).train()
        with torch.no_grad():
            m.weight.copy_(color)
            m.bias.copy_(bias)
        return m
    w_plain, w_conv, m_wc, m_wc16 = dwt_b200.WTransform2d(C, GS).to(dev), dwt_b200.WTransform2d(C, GS).to(dev), wc(), wc()
    cw, cb = color.reshape(C, GS, 1, 1).clone().requires_grad_(True), bias.clone().requires_grad_(True)
    steps = {
        "w": _step_fn(w_plain, x, dy, ()),
        "wc": _step_fn(m_wc, x, dy, (m_wc.weight, m_wc.bias)),
        "wc_bf16": _step_fn(m_wc16, x.bfloat16(), dy.bfloat16(), (m_wc16.weight, m_wc16.bias)),
        "w_conv": _step_fn(lambda xi: Fn.conv2d(w_conv(xi), cw, cb, groups=G), x, dy, (cw, cb)),
    }
    arms, recs = {}, {}
    for name, step in steps.items():
        for _ in range(args.warmup):
            step()
        fams = _families(step, args.steps)
        recs[name] = {"kernels_ms": fams, "kernel_ms_per_iter": round(sum(fams.values()), 4), "ms_per_iter": []}
        arms[name] = _graphed(step, dev)
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
        "wc_over_w_ms": round(med["wc"] - med["w"], 4),
        "w_conv_over_wc_ms": round(med["w_conv"] - med["wc"], 4),
    }))


if __name__ == "__main__":
    main()
