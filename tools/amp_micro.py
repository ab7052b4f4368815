"""The whitening microbench (BASELINE config 2) in float32 and in bfloat16, alternated in one process; one JSON line.

    python tools/amp_micro.py [--steps 50] [--warmup 5] [--rounds 5]

WTransform2d N=256 C=256 56^2 group_size=64, NCHW, forward + backward (y = m(x), dx = grad(y, x, dy)), replayed from a
CUDA graph, in three arms:
  fp32    the float32 tensor-core kernels;
  bf16    bf16 x and dy on the bf16 tensor-core kernels (what torch.autocast hands the layer after a bf16 convolution);
  upcast  bf16 x and dy the way the layer ran them before it had bf16 kernels: x.float() -> the float32 kernels ->
          .to(bfloat16), with the two casts' backward.
The fp32 arm runs on the bf16 input widened (x_bf16.float(), dy_bf16.float()), so its y and dx rounded to bf16 must equal
the bf16 arm's bit for bit; that is checked on one eager step of each arm.

Per arm: ms/iter of every round (median and max - min), and the library's kernel families from one eager profiled pass:
ms and algorithmic GB per iteration, each one's fraction of the H100 SXM data sheet's 3.35 TB/s and, for the apply
kernels, of the TF32 bound (495 TFLOP/s dense: 4 split-TF32 products x 64 channels x 2 flop per element and input);
`bound` names the larger of the two.  The card's name and power limit are read in the same process.
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

HBM_BYTES_PER_S = 3.35e12
TF32_FLOP_PER_S = 495e12
APPLY_FLOP_PER_ELEMENT = {"tc_apply": 512.0, "tc_bwd_apply": 1024.0}   # 4 products x 64 channels x 2 flop, per input


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), None


def _arm(name, xb, dyb, gs, device):
    import dwt_b200
    torch.manual_seed(1)
    m = dwt_b200.WTransform2d(xb.shape[1], gs).to(device).train()
    if name == "fp32":
        x, dy = xb.float().requires_grad_(True), dyb.float()
    else:
        x, dy = xb.detach().clone().requires_grad_(True), dyb

    def step(keep=None):
        y = m(x.float()).to(torch.bfloat16) if name == "upcast" else m(x)
        (dx,) = torch.autograd.grad(y, x, dy)
        if keep is not None:
            keep["y"], keep["dx"] = y.detach(), dx
    return m, x, step


def _families(step, steps, elems):
    from dwt_b200 import _native
    _native.profile_begin()
    for _ in range(steps):
        step()
    prof = _native.by_family(_native.profile_end())
    out = {}
    for fam, v in sorted(prof.items()):
        ms, gb = v["ms"] / steps, v["bytes"] / steps / 1e9
        rec = {"ms": round(ms, 4), "algorithmic_gb": round(gb, 4), "launches": v["launches"] // steps}
        hbm_ms = gb * 1e9 / HBM_BYTES_PER_S * 1e3
        if gb > 0:
            rec["frac_of_hbm"] = round(hbm_ms / ms, 3)
        flops = APPLY_FLOP_PER_ELEMENT.get(fam.replace("_bf16", ""))
        bound_ms = hbm_ms
        rec["bound"] = "hbm" if gb > 0 else None
        if flops:
            tf32_ms = flops * elems / TF32_FLOP_PER_S * 1e3
            rec["frac_of_tf32"] = round(tf32_ms / ms, 3)
            if tf32_ms > hbm_ms:
                rec["bound"], bound_ms = "tf32", tf32_ms
        if rec["bound"]:
            rec["bound_ms"] = round(bound_ms, 4)
        out[fam] = rec
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--gs", type=int, default=64)
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    card, limit = _card()
    N, C, H = args.n, 256, 56
    torch.manual_seed(0)                             # bench.py's microbench input
    mix = torch.randn(C, C, device=device) / C ** 0.5 + torch.eye(C, device=device)
    xb = (torch.einsum("dc,nchw->ndhw", mix, torch.randn(N, C, H, H, device=device)) + 2.0).contiguous().to(torch.bfloat16)
    dyb = torch.randn(N, C, H, H, device=device).to(torch.bfloat16)
    elems = N * C * H * H
    names = ("fp32", "bf16", "upcast")
    arms, recs, eager = {}, {}, {}
    for name in names:
        m, x, step = _arm(name, xb, dyb, args.gs, device)
        keep = {}
        step(keep)                                   # first step of a fresh module: the outputs compared below
        eager[name] = (keep["y"], keep["dx"], m.running_mean.clone(), m.running_variance.clone())
        for _ in range(args.warmup):
            step()
        fams = _families(step, args.steps, elems)
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
        arms[name] = (graph, m, x, step)
        recs[name] = {"kernels": fams, "kernel_ms_per_iter": round(sum(v["ms"] for v in fams.values()), 4),
                      "algorithmic_gb_per_iter": round(sum(v["algorithmic_gb"] for v in fams.values()), 4), "ms_per_iter": []}
    for _ in range(args.rounds):
        for name in names:
            graph = arms[name][0]
            graph.replay()
            ms = timed_loop(graph.replay, args.steps, device, False)
            recs[name]["ms_per_iter"].append(round(ms / args.steps, 4))
    y32, dx32, rm32, rv32 = eager["fp32"]
    yb, dxb, rmb, rvb = eager["bf16"]
    check = {"y": torch.equal(yb, y32.to(torch.bfloat16)), "dx": torch.equal(dxb, dx32.to(torch.bfloat16)),
             "running_buffers": torch.equal(rmb, rm32) and torch.equal(rvb, rv32)}
    from dwt_b200 import _native
    out = {"metric": "WTransform2d fwd+bwd microbench ms/iter, float32 vs bf16 kernels vs bf16 upcast",
           "config": f"N={N} C={C} H=W={H} group_size={args.gs} NCHW, cuda-graph replay", "steps": args.steps,
           "rounds": args.rounds, "gpu": card, "power_limit": limit,
           "bf16_equals_fp32_rounded": check, "status_word": _native.status_all(device)}
    for name in names:
        ms = recs[name]["ms_per_iter"]
        recs[name]["median_ms_per_iter"] = statistics.median(ms)
        recs[name]["spread_ms_per_iter"] = round(max(ms) - min(ms), 4)
        out[name] = recs[name]
    out["bf16_speedup_over_fp32"] = round(out["fp32"]["median_ms_per_iter"] / out["bf16"]["median_ms_per_iter"], 3)
    out["bf16_speedup_over_upcast"] = round(out["upcast"]["median_ms_per_iter"] / out["bf16"]["median_ms_per_iter"], 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
