"""Latent-domain whitening (LatentDomainWTransform2d, dwt_whiten_latent_* and dwt_whiten_latent_small_*) forward +
backward; one JSON line.

    python tools/ld_micro.py [--steps 20] [--warmup 3] [--rounds 3]

Configurations: [192, 256, 56, 56] at group size 64 (NCHW fp32) with 3 and 8 latent domains (the tensor-core kernels),
and at group size 4 (the register-resident kernels) ResNet-50-DWT's stem [192, 64, 112, 112] with 3 domains and its
layer1 site [192, 256, 56, 56] with 3 and 8, NCHW and channels-last fp32, and NCHW bf16.  Inputs have a per-image channel
mixing and mean; dy is randn; the domain weights are the softmax of per-image logits, and the gradient flows to the
logits.  Arms, alternated round by round in one process (one configuration at a time), each replayed from a CUDA
graph (median of the rounds), all in training mode:
  ld            LatentDomainWTransform2d, y = m(x, softmax(logits)), dx and the gradient of the logits;
  iw            InstanceWTransform2d (group size 64);
  sw            SwitchableWTransform2d(components=("bw", "iw")), dx and the gradient of its mixing logits (group size 64);
  wt            WTransform2d(C, 4) on the whole batch: the same passes and bytes without domains (group size 4);
  ldbn          LatentDomainBatchNorm2d(C, D, affine=False) under the same weights: the same bytes per element (group size 4);
  aten          the same latent-domain whitening as the ATen operator sequence with autograd: per-image moments (matmul),
                the weighted domain moments, cholesky_ex -> inv_ex, A_n = sum_d w_nd W_d and y = A_n x - sum_d w_nd W_d mu_d,
                fp32 NCHW (TF32 off, PyTorch's default for matmul), replayed eagerly if it cannot be captured (fp32 only).
"ld_over_iw", "ld_over_wt" and "ld_over_ldbn" are the ratios of the medians of ld and that arm of the same configuration,
in the same run.  Per library arm: the kernel families from one eager profiled pass (CUDA events around every launch, ms
per iteration) and the finalize share of that kernel time.  The card's name, power limit, maximum SM clock and the SM
clock at the end of the timed rounds are read in the same process.
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

CONFIGS = [  # (name, shape, gs, latent domains, channels-last, dtype)
    ("56sq_gs64_d3", (192, 256, 56, 56), 64, 3, False, torch.float32),
    ("56sq_gs64_d8", (192, 256, 56, 56), 64, 8, False, torch.float32),
    ("stem_gs4_d3", (192, 64, 112, 112), 4, 3, False, torch.float32),
    ("stem_gs4_d3_nhwc", (192, 64, 112, 112), 4, 3, True, torch.float32),
    ("56sq_gs4_d3", (192, 256, 56, 56), 4, 3, False, torch.float32),
    ("56sq_gs4_d8", (192, 256, 56, 56), 4, 8, False, torch.float32),
    ("56sq_gs4_d3_nhwc", (192, 256, 56, 56), 4, 3, True, torch.float32),
    ("56sq_gs4_d3_bf16", (192, 256, 56, 56), 4, 3, False, torch.bfloat16),
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
    recs = {}
    inputs = {}
    # one configuration at a time (its arms alternated round by round), its graphs released before the next: every
    # configuration's graphs at once do not fit in 80 GB
    for name, shape, gs, d, cl, dtype in CONFIGS:
        if shape not in inputs:
            inputs = {shape: _inputs(shape, dev)}
        fmt = torch.channels_last if cl else torch.contiguous_format
        x, dy = (t.to(dtype).contiguous(memory_format=fmt) for t in inputs[shape])
        logits = torch.randn(shape[0], d, device=dev, generator=torch.Generator(device=dev).manual_seed(d)).requires_grad_(True)
        steps = {}
        ld = dwt_b200.LatentDomainWTransform2d(shape[1], gs, d).to(dev).train()
        steps[f"{name}/ld"] = _step_fn(lambda t, m=ld, lg=logits: m(t, torch.softmax(lg, 1)), x, dy, (logits,))
        if gs > 4:
            iw = dwt_b200.InstanceWTransform2d(shape[1], gs).to(dev)
            steps[f"{name}/iw"] = _step_fn(iw, x, dy)
            sw = dwt_b200.SwitchableWTransform2d(shape[1], gs, ("bw", "iw")).to(dev).train()
            steps[f"{name}/sw"] = _step_fn(sw, x, dy, tuple(sw.parameters()))
        else:
            wt = dwt_b200.WTransform2d(shape[1], gs).to(dev).train()
            steps[f"{name}/wt"] = _step_fn(wt, x, dy)
            ldbn = dwt_b200.LatentDomainBatchNorm2d(shape[1], d, affine=False).to(dev).train()
            steps[f"{name}/ldbn"] = _step_fn(lambda t, m=ldbn, lg=logits: m(t, torch.softmax(lg, 1)), x, dy, (logits,))
        if dtype == torch.float32:
            steps[f"{name}/aten"] = _step_fn(lambda t, gs=gs, lg=logits: aten_ld(t, gs, torch.softmax(lg, 1)), x, dy,
                                             (logits,))
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
        del arms, steps, x, dy
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
    for r in recs.values():
        r["median_ms_per_iter"] = statistics.median(r["ms_per_iter"])
        r["spread_ms_per_iter"] = round(max(r["ms_per_iter"]) - min(r["ms_per_iter"]), 4)
    for name, *_ in CONFIGS:
        for arm in ("iw", "wt", "ldbn"):
            if f"{name}/{arm}" in recs:
                recs[f"{name}/ld"][f"ld_over_{arm}"] = round(recs[f"{name}/ld"]["median_ms_per_iter"]
                                                             / recs[f"{name}/{arm}"]["median_ms_per_iter"], 4)
    print(json.dumps({"what": "latent-domain whitening forward + backward", **_card(), "steps": args.steps,
                      "rounds": args.rounds, "arms": recs}))


if __name__ == "__main__":
    main()
