"""Switchable whitening (SwitchableWTransform2d, dwt_whiten_switch_*) forward + backward; one JSON line.

    python tools/sw_micro.py [--steps 20] [--warmup 3] [--rounds 3]

Configurations: [192, 256, 56, 56] at group sizes 16 and 64 (NCHW fp32), and the stem shape [192, 64, 112, 112] at group
size 64 in NCHW and channels-last, fp32 and bf16.  Inputs have a per-image channel mixing and mean; dy is randn.  Arms,
alternated round by round in one process, each replayed from a CUDA graph (median of the rounds), all in training mode:
  swa           SwitchableWTransform2d(components=("bw", "iw")), y = m(x), dx and the gradient of the mixing logits;
  swb           the same with ("bw", "iw", "bn", "in");
  iw            InstanceWTransform2d;
  wt            WTransform2d (batch whitening, running statistics updated);
  aten          SW^a as the ATen operator sequence with autograd: per-image and batch mean and covariance (matmul), the
                softmax mix, cholesky_ex -> inv_ex -> matmul, fp32 NCHW (TF32 off, PyTorch's default for matmul),
                replayed eagerly if it cannot be captured.
"swa_over_iw" is the ratio of the medians of swa and iw of the same configuration, in the same run.
Per library arm: the kernel families from one eager profiled pass (CUDA events around every launch, ms per iteration),
the finalize share of that kernel time, and the algorithmic HBM bound: 32 bytes per element in fp32 (forward: x read
twice and y written; backward: x and dy read twice and dx written), 16 in bf16, at the 3.35 TB/s of the H100 SXM data
sheet.  The card's name, power limit, maximum SM clock and the SM clock at the end of the timed rounds are read in the
same process.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench import timed_loop  # noqa: E402
from zca_micro import _families, _graphed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
CONFIGS = [  # (name, shape, gs, channels-last, bf16, with an ATen arm)
    ("56sq_gs16", (192, 256, 56, 56), 16, False, False, True),
    ("56sq_gs64", (192, 256, 56, 56), 64, False, False, True),
    ("stem_nchw", (192, 64, 112, 112), 64, False, False, True),
    ("stem_nhwc", (192, 64, 112, 112), 64, True, False, False),
    ("stem_nchw_bf16", (192, 64, 112, 112), 64, False, True, False),
    ("stem_nhwc_bf16", (192, 64, 112, 112), 64, True, True, False),
]


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit, sm, sm_max = (s.strip() for s in out.split(","))
        return {"card": name, "power_limit": limit, "sm_clock_at_end": sm, "sm_clock_max": sm_max}
    except Exception:
        return {"card": torch.cuda.get_device_name(), "power_limit": None}


def aten_swa(x, gs, mean_logits, var_logits, eps=1e-3):
    n, c = x.shape[:2]
    xg = x.reshape(n, c // gs, gs, -1)
    m = xg.shape[-1]
    mu_n = xg.mean(-1, keepdim=True)
    xc = xg - mu_n
    cov_n = xc @ xc.transpose(-1, -2) / m
    mu_b = mu_n.mean(0, keepdim=True)
    xb = (xg - mu_b).transpose(0, 1).reshape(c // gs, gs, -1)
    cov_b = xb @ xb.transpose(-1, -2) / (n * m)
    am, av = torch.softmax(mean_logits, 0), torch.softmax(var_logits, 0)
    s = (1 - eps) * (av[0] * cov_b + av[1] * cov_n) + eps * torch.eye(gs, device=x.device, dtype=x.dtype)
    w = torch.linalg.inv_ex(torch.linalg.cholesky_ex(s)[0])[0]
    return (w @ (xg - (am[0] * mu_b + am[1] * mu_n))).reshape(x.shape)


def _step_fn(fwd, x, dy, params=()):
    def step():
        xi = x.detach().requires_grad_(True)
        torch.autograd.grad(fwd(xi), (xi, *params), dy)
    return step


def _inputs(shape, dev, seed=0):
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    mix = torch.eye(c, device=dev) + torch.randn(n, c, c, device=dev, generator=g) / c ** 0.5
    x = mix @ torch.randn(n, c, h * w, device=dev, generator=g) + torch.randn(n, c, 1, device=dev, generator=g) + 1.0
    return x.reshape(shape).contiguous(), torch.randn(shape, device=dev, generator=g)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sw_micro.py measures on a CUDA device; none is visible")
    import dwt_b200
    dev = torch.device("cuda", 0)
    steps, recs = {}, {}
    base = {}
    for name, shape, gs, nhwc, bf16, aten in CONFIGS:
        if shape not in base:
            base[shape] = _inputs(shape, dev)
        x, dy = base[shape]
        fmt = torch.channels_last if nhwc else torch.contiguous_format
        xa, dya = (t.to(torch.bfloat16 if bf16 else torch.float32).contiguous(memory_format=fmt) for t in (x, dy))
        elems = x.numel()
        bound_ms = (16 if bf16 else 32) * elems / HBM_BYTES_PER_S * 1e3
        mods = {"swa": dwt_b200.SwitchableWTransform2d(shape[1], gs, ("bw", "iw")),
                "swb": dwt_b200.SwitchableWTransform2d(shape[1], gs, ("bw", "iw", "bn", "in")),
                "iw": dwt_b200.InstanceWTransform2d(shape[1], gs), "wt": dwt_b200.WTransform2d(shape[1], gs)}
        for arm, m in mods.items():
            m.to(dev).train()
            steps[f"{name}/{arm}"] = _step_fn(m, xa, dya, tuple(m.parameters()))
            recs[f"{name}/{arm}"] = {"hbm_bound_ms": round(bound_ms, 4)}
        if aten:
            logits = [torch.ones(2, device=dev, requires_grad=True) for _ in range(2)]
            steps[f"{name}/aten"] = _step_fn(lambda t, gs=gs, lg=logits: aten_swa(t, gs, *lg), xa, dya, tuple(logits))
            recs[f"{name}/aten"] = {"hbm_bound_ms": round(bound_ms, 4)}
    arms = {}
    for key, step in steps.items():
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize(dev)
        r = recs[key]
        r["ms_per_iter"] = []
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
        r["hbm_bound_share"] = round(r["hbm_bound_ms"] / r["median_ms_per_iter"], 4)
    for name, *_ in CONFIGS:
        recs[f"{name}/swa"]["swa_over_iw"] = round(recs[f"{name}/swa"]["median_ms_per_iter"] / recs[f"{name}/iw"]["median_ms_per_iter"], 4)
    print(json.dumps({"what": "switchable whitening forward + backward", **_card(), "steps": args.steps,
                      "rounds": args.rounds, "arms": recs}))


if __name__ == "__main__":
    main()
