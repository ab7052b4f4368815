"""Channels-last norm sites at widths whose C/4 is not a power of two: the channels-last kernels against the route such
calls took before (a copy to NCHW), and against NCHW input; one JSON line.

    python tools/cl_width_micro.py [--steps 10] [--warmup 3] [--rounds 3] [--per-domain 64] [--no-lenet]

Workloads: a DomainTripleNorm site (3 domains x --per-domain images, training statistics, gamma / beta, ReLU) at widths
real backbones use -- C = 96 @ 56^2, 192 @ 28^2, 320 @ 28^2, 576 @ 14^2, 1280 @ 7^2 (C/4 = 320 > 256) and the LeNet's
conv2 site, C = 48 @ 14^2 -- as group-size-4 whitening and as batch norm, each plain (AFFINE|RELU) and residual
(relu(site(x) + identity)); forward + backward, replayed from a CUDA graph.  Three arms, alternated round by round
within each workload, in float32 and bfloat16:
  a_cl     channels-last x, dy (and identity) on the channels-last kernels; y, dx come back channels-last;
  b_old    the same tensors on the route they took before (_native.channels_last_supported patched back to C/4 a power
           of two): x copied to NCHW, the NCHW kernels (bf16: upcast to float32 first), y and dx made channels-last
           again for the next convolution;
  c_nchw   NCHW x and dy on the NCHW kernels.
Per arm: ms/iter of every round (median, max - min), the algorithmic GB of the library's launches (one eager profiled
step) and the peak device memory one eager step adds.  Per workload, float32 (a) against (b): max |a - b| / max |b| of y,
dx norm-wise and elementwise off the elements whose ReLU decision the two roundings of y split (counted); and
whether the bf16 arm (a) equals the float32 arm (a) on the widened bf16 inputs, rounded.  LeNet arm (unless
--no-lenet): the harness LeNet with channels-last conv weights and input, one training step, a_cl against b_old, in
images/s.  The card's name and power limit are read in the same process.
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
from cl_tc_micro import _card, _peak  # noqa: E402

CL = torch.channels_last
BF = torch.bfloat16
WIDTHS = [(96, 56), (192, 28), (320, 28), (576, 14), (1280, 7), (48, 14)]
SITES = [("whiten", 4, False), ("whiten", 4, True), ("bn", 1, False), ("bn", 1, True)]


def _pow2_rule(channels, group_size):
    """channels_last_supported as it was: C/4 a power of two."""
    c4 = channels // 4
    return group_size in (1, 2, 4) and channels % 4 == 0 and 0 < c4 <= 16384 and c4 & (c4 - 1) == 0


class _OldRoute:
    def __enter__(self):
        from dwt_b200 import _native
        self.nv, self.saved = _native, _native.channels_last_supported
        _native.channels_last_supported = _pow2_rule

    def __exit__(self, *exc):
        self.nv.channels_last_supported = self.saved


def _site(kind, c, gs, device):
    import dwt_b200
    torch.manual_seed(1)
    if kind == "whiten":
        mods = [dwt_b200.WTransform2d(c, gs).to(device).train() for _ in range(3)]
    else:
        mods = [dwt_b200.BatchNorm2d(c, torch.zeros(c, device=device), torch.ones(c, device=device), affine=False).train()
                for _ in range(3)]
    g = torch.ones(c, 1, 1, device=device, requires_grad=True)
    b = torch.zeros(c, 1, 1, device=device, requires_grad=True)
    return dwt_b200.DomainTripleNorm(kind, c, gs, n_domains=3), mods, g, b


def _arm(name, kind, c, gs, res, x0, r0, dy0, device):
    """-> step(keep=None): one forward + backward of arm `name`.  The closure owns the arm's tensors and modules: a
    graph captured from it replays on them, so it must live as long as the graph."""
    norm, mods, g, b = _site(kind, c, gs, device)
    fmt = torch.contiguous_format if name == "c_nchw" else CL
    x, dy = x0.contiguous(memory_format=fmt), dy0.contiguous(memory_format=fmt)
    r = r0.contiguous(memory_format=fmt) if res else None

    def step(keep=None):
        xi = x.detach().requires_grad_(True)          # a fresh leaf per step (see cl_tc_micro.py)
        if name == "b_old":
            with _OldRoute():
                y = norm(xi, mods, g, b, True, residual=r).contiguous(memory_format=CL)
                (dx,) = torch.autograd.grad(y, xi, dy)
            dx = dx.contiguous(memory_format=CL)
        else:
            y = norm(xi, mods, g, b, True, residual=r)
            (dx,) = torch.autograd.grad(y, xi, dy)
        if keep is not None:
            keep["y"], keep["dx"] = y.detach(), dx
    return step


def _gb(step):
    from dwt_b200 import _native
    _native.profile_begin()
    step()
    prof = _native.by_family(_native.profile_end())
    return round(sum(v["bytes"] for v in prof.values()) / 1e9, 4), sorted(prof)


def _rel_max(a, b):
    a, b = a.float().contiguous(), b.float().contiguous()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _workload(args, device, kind, c, hw, gs, res):
    n = 3 * args.per_domain
    gen = torch.Generator(device=device).manual_seed(c)
    x32 = torch.randn(n, hw, hw, c, device=device, generator=gen).permute(0, 3, 1, 2)
    x32 = (x32 + 0.6 * x32.roll(1, 1) + 0.5).contiguous(memory_format=CL)
    r32 = torch.randn(n, hw, hw, c, device=device, generator=gen).permute(0, 3, 1, 2).contiguous(memory_format=CL)
    dy32 = torch.randn(n, hw, hw, c, device=device, generator=gen).permute(0, 3, 1, 2).contiguous(memory_format=CL)
    names = [(dt, a) for dt in ("fp32", "bf16") for a in ("a_cl", "b_old", "c_nchw")]
    recs, eager, arms = {}, {}, {}
    for dt, a in names:
        cast = (lambda t: t) if dt == "fp32" else (lambda t: t.to(BF))
        step = _arm(a, kind, c, gs, res, cast(x32), cast(r32), cast(dy32), device)
        keep = {}
        step(keep)
        eager[(dt, a)] = keep
        for _ in range(args.warmup):
            step()
        gb, fams = _gb(step)
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
        arms[(dt, a)] = (graph, step)                 # the step keeps the graph's inputs and modules alive
        recs[(dt, a)] = {"algorithmic_gb_per_iter": gb, "families": fams, "peak_gib_added": peak, "ms_per_iter": []}
    for _ in range(args.rounds):
        for key in names:
            graph = arms[key][0]
            graph.replay()
            recs[key]["ms_per_iter"].append(round(timed_loop(graph.replay, args.steps, device, False) / args.steps, 4))
    out = {"site": f"{kind} gs{gs} C={c} {hw}x{hw} {'residual' if res else 'plain'}"}
    for dt, a in names:
        r = recs[(dt, a)]
        r["median_ms_per_iter"] = statistics.median(r["ms_per_iter"])
        r["spread_ms_per_iter"] = round(max(r["ms_per_iter"]) - min(r["ms_per_iter"]), 4)
        out.setdefault(dt, {})[a] = r
    for dt in ("fp32", "bf16"):
        out[dt]["speedup_a_over_b"] = round(out[dt]["b_old"]["median_ms_per_iter"] / out[dt]["a_cl"]["median_ms_per_iter"], 3)
        out[dt]["speedup_a_over_c"] = round(out[dt]["c_nchw"]["median_ms_per_iter"] / out[dt]["a_cl"]["median_ms_per_iter"], 3)
    # (a) against (b) in float32: y; dx norm-wise, and elementwise away from the elements whose ReLU decision the two
    # arms' roundings of y put on opposite sides of zero (there dx is dy in one arm and 0 in the other)
    ea, eb = eager[("fp32", "a_cl")], eager[("fp32", "b_old")]
    flip = (ea["y"] > 0) != (eb["y"] > 0)
    dxa, dxb = ea["dx"].float().contiguous(), eb["dx"].float().contiguous()
    out["fp32_a_vs_b"] = {"y_rel_max": _rel_max(ea["y"], eb["y"]),
                          "dx_rel_norm": float((dxa - dxb).norm() / dxb.norm()),
                          "dx_rel_max_off_flips": _rel_max(dxa.masked_fill(flip, 0), dxb.masked_fill(flip, 0)),
                          "relu_flips": int(flip.sum())}
    # bf16 arm (a) == the float32 arm (a) on the same (widened) values, rounded
    keep = {}
    _arm("a_cl", kind, c, gs, res, x32.to(BF).float(), r32.to(BF).float(), dy32.to(BF).float(), device)(keep)
    eb16 = eager[("bf16", "a_cl")]
    out["bf16_a_equals_fp32_a_rounded"] = bool(all(torch.equal(eb16[k], keep[k].to(BF)) for k in ("y", "dx")))
    torch.cuda.synchronize(device)
    del arms, eager, keep
    torch.cuda.empty_cache()
    return out


def _lenet(args, device):
    """The harness LeNet, channels-last conv weights and input, one training step: a_cl against b_old, images/s."""
    import copy

    import dwt_b200
    from harness.lenet_dwt import LeNetDWT
    torch.manual_seed(5)
    proto = LeNetDWT(dwt_b200).to(device).train().to(memory_format=CL)
    images = torch.randn(2 * 64, 1, 28, 28, device=device).contiguous(memory_format=CL)
    steps = {}
    for arm in ("a_cl", "b_old"):
        model = copy.deepcopy(proto)

        def step(model=model, old=arm == "b_old"):
            if old:
                with _OldRoute():
                    model(images).logsumexp(1).mean().backward()
            else:
                model(images).logsumexp(1).mean().backward()
            model.zero_grad(set_to_none=True)
        for _ in range(3):
            step()
        steps[arm] = step
    ips = {a: [] for a in steps}
    for _ in range(args.rounds):
        for a, step in steps.items():
            ms = timed_loop(step, args.steps, device, False) / args.steps
            ips[a].append(round(images.shape[0] / (ms / 1e3), 1))
    out = {"config": "harness LeNet-DWT, 2 x 64 images of 28^2, channels-last, one training step (eager)"}
    for a, v in ips.items():
        out[a] = {"images_per_s": v, "median_images_per_s": statistics.median(v)}
    out["speedup_a_over_b"] = round(out["a_cl"]["median_images_per_s"] / out["b_old"]["median_images_per_s"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--per-domain", type=int, default=64)
    ap.add_argument("--no-lenet", action="store_true")
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    card, limit = _card()
    from dwt_b200 import _native
    out = {"metric": "channels-last norm site fwd+bwd ms/iter at C/4 not a power of two: channels-last kernels vs the "
                     "old NCHW-copy route vs NCHW input",
           "config": f"DomainTripleNorm, 3 x {args.per_domain} images, cuda-graph replay", "steps": args.steps,
           "rounds": args.rounds, "gpu": card, "power_limit": limit, "workloads": []}
    for c, hw in WIDTHS:
        for kind, gs, res in SITES:
            out["workloads"].append(_workload(args, device, kind, c, hw, gs, res))
            print(f"done {out['workloads'][-1]['site']}", file=sys.stderr, flush=True)
    if not args.no_lenet:
        out["lenet"] = _lenet(args, device)
    out["status_word"] = _native.status_all(device)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
