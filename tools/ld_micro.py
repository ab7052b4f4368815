"""Latent-domain whitening (LatentDomainWTransform2d, dwt_whiten_latent_*) forward + backward; one JSON line.

    python tools/ld_micro.py [--steps 20] [--warmup 3] [--rounds 3]

Configurations: [192, 256, 56, 56] at group size 64 (NCHW fp32) with 3 and 8 latent domains.  Inputs have a per-image
channel mixing and mean; dy is randn; the domain weights are the softmax of per-image logits, and the gradient flows to
the logits.  Arms, alternated round by round in one process, each replayed from a CUDA graph (median of the rounds), all
in training mode:
  ld            LatentDomainWTransform2d, y = m(x, softmax(logits)), dx and the gradient of the logits;
  iw            InstanceWTransform2d;
  sw            SwitchableWTransform2d(components=("bw", "iw")), dx and the gradient of its mixing logits;
  aten          the same latent-domain whitening as the ATen operator sequence with autograd: per-image moments (matmul),
                the weighted domain moments, cholesky_ex -> inv_ex, A_n = sum_d w_nd W_d and y = A_n x - sum_d w_nd W_d mu_d,
                fp32 NCHW (TF32 off, PyTorch's default for matmul), replayed eagerly if it cannot be captured.
"ld_over_iw" is the ratio of the medians of ld and iw of the same configuration, in the same run.
Per library arm: the kernel families from one eager profiled pass (CUDA events around every launch, ms per iteration) and
the finalize share of that kernel time.  The card's name, power limit, maximum SM clock and the SM clock at the end of the
timed rounds are read in the same process.
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
from sw_micro import _card, _inputs, _step_fn  # noqa: E402
from zca_micro import _families, _graphed  # noqa: E402

CONFIGS = [  # (name, shape, gs, latent domains)
    ("56sq_gs64_d3", (192, 256, 56, 56), 64, 3),
    ("56sq_gs64_d8", (192, 256, 56, 56), 64, 8),
]


def aten_ld(x, gs, w, eps=1e-3):
    n, c = x.shape[:2]
    xg = x.reshape(n, c // gs, gs, -1)
    m = xg.mean(-1)
    xc = xg - m.unsqueeze(-1)
    cov = xc @ xc.transpose(-1, -2) / xg.shape[-1]
    s = w.sum(0)
    mu = torch.einsum("nd,ngi->dgi", w, m) / s[:, None, None]
    u = m.unsqueeze(0) - mu.unsqueeze(1)                               # [D, N, G, gs]
    sig = (torch.einsum("nd,ngij->dgij", w, cov) + torch.einsum("nd,dngi,dngj->dgij", w, u, u)) / s[:, None, None, None]
    eye = torch.eye(gs, device=x.device, dtype=x.dtype)
    wm = torch.linalg.inv_ex(torch.linalg.cholesky_ex((1 - eps) * sig + eps * eye)[0])[0]
    a = torch.einsum("nd,dgij->ngij", w, wm)
    b = torch.einsum("nd,dgi->ngi", w, (wm @ mu.unsqueeze(-1)).squeeze(-1))
    return (a @ xg - b.unsqueeze(-1)).reshape(x.shape)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ld_micro.py measures on a CUDA device; none is visible")
    import dwt_b200
    dev = torch.device("cuda", 0)
    steps, recs = {}, {}
    x = dy = None
    for name, shape, gs, d in CONFIGS:
        if x is None:
            x, dy = _inputs(shape, dev)
        logits = torch.randn(shape[0], d, device=dev, generator=torch.Generator(device=dev).manual_seed(d)).requires_grad_(True)
        ld = dwt_b200.LatentDomainWTransform2d(shape[1], gs, d).to(dev).train()
        steps[f"{name}/ld"] = _step_fn(lambda t, m=ld, lg=logits: m(t, torch.softmax(lg, 1)), x, dy, (logits,))
        iw = dwt_b200.InstanceWTransform2d(shape[1], gs).to(dev)
        steps[f"{name}/iw"] = _step_fn(iw, x, dy)
        sw = dwt_b200.SwitchableWTransform2d(shape[1], gs, ("bw", "iw")).to(dev).train()
        steps[f"{name}/sw"] = _step_fn(sw, x, dy, tuple(sw.parameters()))
        steps[f"{name}/aten"] = _step_fn(lambda t, gs=gs, lg=logits: aten_ld(t, gs, torch.softmax(lg, 1)), x, dy, (logits,))
    arms = {}
    for key, step in steps.items():
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize(dev)
        r = recs[key] = {"ms_per_iter": []}
        if not key.endswith("/aten"):
            fams = _families(step, args.steps)
            r["kernels_ms"] = fams
            tot = sum(fams.values())
            r["kernel_ms_per_iter"] = round(tot, 4)
            fin = sum(v for f, v in fams.items() if "finalize" in f)
            r["finalize_ms_per_iter"] = round(fin, 4)
            r["finalize_share"] = round(fin / tot, 4) if tot else None
        try:
            arms[key] = _graphed(step, dev)
            r["replay"] = "graph"
        except Exception as e:                       # an operator that syncs the host cannot be captured
            torch.cuda.synchronize(dev)
            arms[key] = step
            r["replay"] = f"eager ({type(e).__name__})"
    for _ in range(args.rounds):
        for key, fn in arms.items():
            fn()
            recs[key]["ms_per_iter"].append(round(timed_loop(fn, args.steps, dev, False) / args.steps, 4))
    for r in recs.values():
        r["median_ms_per_iter"] = statistics.median(r["ms_per_iter"])
        r["spread_ms_per_iter"] = round(max(r["ms_per_iter"]) - min(r["ms_per_iter"]), 4)
    for name, *_ in CONFIGS:
        recs[f"{name}/ld"]["ld_over_iw"] = round(recs[f"{name}/ld"]["median_ms_per_iter"] / recs[f"{name}/iw"]["median_ms_per_iter"], 4)
    print(json.dumps({"what": "latent-domain whitening forward + backward", **_card(), "steps": args.steps,
                      "rounds": args.rounds, "arms": recs}))


if __name__ == "__main__":
    main()
