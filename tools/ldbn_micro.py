"""Latent-domain batch norm (LatentDomainBatchNorm2d, dwt_bn_latent_*) forward + backward; one JSON line.

    python tools/ldbn_micro.py [--steps 20] [--warmup 3] [--rounds 3] [--shapes 56,28,14,7]

Configurations: the ResNet-50 norm-site shapes [192, 256, 56, 56], [192, 512, 28, 28], [192, 1024, 14, 14] and
[192, 2048, 7, 7], each with 3 and 8 latent domains, float32 and bfloat16, NCHW and channels-last.  x is randn with a
per-image mean, dy is randn, the domain weights are the softmax of per-image logits and the gradient flows to the logits,
gamma and beta.  Per configuration three arms on the same tensors, all in training mode, each replayed from a CUDA graph,
alternated round by round (median of the rounds):
  ldbn   LatentDomainBatchNorm2d, y = m(x, softmax(logits)): dx, the logits' gradient, dgamma, dbeta;
  bn     the package's BatchNorm2d (one domain, the batch's statistics): dx, dgamma, dbeta;
  aten   the same latent-domain batch norm as the ATen operator sequence with autograd (per-image moments, the weighted
         domain moments, a_n and b_n, y = gamma (a_n x + b_n) + beta; float32 statistics).
"ldbn_over_bn" is the ratio of the medians of ldbn and bn of the same configuration, in the same run.  Per library arm:
the kernel families from one eager profiled pass (CUDA events around every launch, ms per iteration) and the finalize
share of that kernel time.  The card's name, power limit, maximum SM clock and the SM clock at the end are read in the
same process.  Each configuration's graphs are freed before the next one is built; every graph is captured on one stream
whose workspace is sized for all of them first.
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

from bench import timed_loop  # noqa: E402
from sw_micro import _card  # noqa: E402
from zca_micro import _families  # noqa: E402

SHAPES = {"56": (192, 256, 56, 56), "28": (192, 512, 28, 28), "14": (192, 1024, 14, 14), "7": (192, 2048, 7, 7)}


def aten_ldbn(x, w, gamma, beta, eps=1e-5):
    n, c = x.shape[:2]
    xr = x.float().reshape(n, c, -1)
    m = xr.mean(-1)
    v = xr.var(-1, unbiased=False)
    s = w.sum(0)
    mu = (w.t() @ m) / s[:, None]
    var = torch.einsum("nd,dnc->dc", w, v.unsqueeze(0) + (m.unsqueeze(0) - mu.unsqueeze(1)) ** 2) / s[:, None]
    r = (var + eps).rsqrt()
    a, b = w @ r, -(w @ (r * mu))
    y = (a[:, :, None, None] * x + b[:, :, None, None]) * gamma[:, None, None] + beta[:, None, None]
    return y.to(x.dtype)


def _graphed(step, dev, cap):
    """step captured into a CUDA graph on the capture stream cap -> its replay."""
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=cap):
        step()
    graph.replay()
    torch.cuda.synchronize(dev)
    return graph.replay


def _step(fwd, x, dy, params):
    def step():
        xi = x.detach().requires_grad_(True)
        torch.autograd.grad(fwd(xi), (xi, *params), dy)
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="56,28,14,7")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ldbn_micro.py measures on a CUDA device; none is visible")
    import dwt_b200
    dev = torch.device("cuda", 0)
    recs = {}
    # A graph keeps the workspace pointer it was captured with, and a call that needs a larger workspace replaces the
    # stream's buffer (_native.grow_workspace): size the capture stream's buffer for every arm once, before any capture.
    from dwt_b200 import _native as nv
    lib = nv.lib()
    cap = torch.cuda.Stream(dev)
    need = max(max(lib.dwt_bn_latent_workspace_bytes(s[0], s[1], s[2] * s[3], 8), lib.dwt_workspace_bytes(s[0], s[1], s[2] * s[3], 1, 1))
               for s in SHAPES.values())
    with torch.cuda.stream(cap):
        nv.grow_workspace(dev, need)
    torch.cuda.synchronize(dev)
    for sk in args.shapes.split(","):
        shape = SHAPES[sk]
        n, c = shape[:2]
        g = torch.Generator(device=dev).manual_seed(0)
        x32 = torch.randn(shape, device=dev, generator=g) + torch.randn(n, c, 1, 1, device=dev, generator=g)
        dy32 = torch.randn(shape, device=dev, generator=g)
        for dtype in (torch.float32, torch.bfloat16):
            for layout in ("nchw", "nhwc"):
                fmt = torch.channels_last if layout == "nhwc" else torch.contiguous_format
                x = x32.to(dtype).contiguous(memory_format=fmt)
                dy = dy32.to(dtype).contiguous(memory_format=fmt)
                for d in (3, 8):
                    name = f"{sk}sq_d{d}_{'bf16' if dtype == torch.bfloat16 else 'fp32'}_{layout}"
                    logits = torch.randn(n, d, device=dev, generator=g).requires_grad_(True)
                    ld = dwt_b200.LatentDomainBatchNorm2d(c, d).to(dev).train()
                    bn = dwt_b200.BatchNorm2d(c, torch.zeros(c, device=dev), torch.ones(c, device=dev)).to(dev).train()
                    gamma = torch.ones(c, device=dev, requires_grad=True)
                    beta = torch.zeros(c, device=dev, requires_grad=True)
                    steps = {
                        "ldbn": _step(lambda t, m=ld, lg=logits: m(t, torch.softmax(lg, 1)), x, dy, (logits, ld.weight, ld.bias)),
                        "bn": _step(bn, x, dy, (bn.weight, bn.bias)),
                        "aten": _step(lambda t, lg=logits: aten_ldbn(t, torch.softmax(lg, 1), gamma, beta), x, dy,
                                      (logits, gamma, beta)),
                    }
                    arms = {}
                    for arm, step in steps.items():
                        for _ in range(args.warmup):
                            step()
                        torch.cuda.synchronize(dev)
                        r = recs[f"{name}/{arm}"] = {"ms_per_iter": []}
                        if arm != "aten":
                            fams = _families(step, args.steps)
                            tot = sum(fams.values())
                            fin = sum(v for f, v in fams.items() if "finalize" in f)
                            r.update(kernels_ms=fams, kernel_ms_per_iter=round(tot, 4), finalize_ms_per_iter=round(fin, 4),
                                     finalize_share=round(fin / tot, 4) if tot else None)
                        try:
                            arms[arm] = _graphed(step, dev, cap)
                            r["replay"] = "graph"
                        except Exception as e:               # an operator that syncs the host cannot be captured
                            torch.cuda.synchronize(dev)
                            arms[arm] = step
                            r["replay"] = f"eager ({type(e).__name__})"
                    for _ in range(args.rounds):
                        for arm, fn in arms.items():
                            fn()
                            recs[f"{name}/{arm}"]["ms_per_iter"].append(
                                round(timed_loop(fn, args.steps, dev, False) / args.steps, 4))
                    for arm in arms:
                        r = recs[f"{name}/{arm}"]
                        r["median_ms_per_iter"] = statistics.median(r["ms_per_iter"])
                        r["spread_ms_per_iter"] = round(max(r["ms_per_iter"]) - min(r["ms_per_iter"]), 4)
                    recs[f"{name}/ldbn"]["ldbn_over_bn"] = round(
                        recs[f"{name}/ldbn"]["median_ms_per_iter"] / recs[f"{name}/bn"]["median_ms_per_iter"], 4)
                    del arms, steps
                    torch.cuda.synchronize(dev)
                    torch.cuda.empty_cache()
    print(json.dumps({"what": "latent-domain batch norm forward + backward", **_card(), "steps": args.steps,
                      "rounds": args.rounds, "arms": recs}))


if __name__ == "__main__":
    main()
