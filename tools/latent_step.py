"""Latent-domain sites: fused against the ATen composition, per site and in the ResNet-50-DWT training step.

    python tools/latent_step.py [--sites] [--model] [--rounds 3] [--reps 20]

(a) --sites: each ResNet-50-DWT site shape (whitening gs 4 at [192, 64, 112, 112] and [192, 256, 56, 56], batch norm at
    [192, 512, 28, 28], [192, 1024, 14, 14], [192, 2048, 7, 7]), NCHW and channels-last, fp32 and bf16, 3 domains under
    softmax weights, training forward + backward of two sites: relu(site(x)) and relu(site(x) + residual).  Arms: "fused"
    (the epilogue arguments, dwt_latent_site_*) and "aten" (the layer, then gamma / beta, the add and the ReLU as ATen
    ops).
(b) --model: the latent ResNet-50-DWT training step (forward, loss, backward; no optimizer) at 3 x 64 images of 224^2,
    channels-last, K = 3: latent fused, latent modules, and the domain-triple DWT model with fused sites in the same run,
    in fp32 and under bf16 autocast.

Every arm is a CUDA graph, captured after a warm-up on its capture stream; the arms of one configuration are replayed
alternately, `reps` replays per arm and round, timed by CUDA events; the median of `rounds` rounds is reported in ms.
The card's name and power limit are read in the same call.  One JSON line per configuration on stdout.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "dwt-domain-adaptation_b200"), ROOT]

SITES = [("whiten", (192, 64, 112, 112), 4), ("whiten", (192, 256, 56, 56), 4), ("bn", (192, 512, 28, 28), 1),
         ("bn", (192, 1024, 14, 14), 1), ("bn", (192, 2048, 7, 7), 1)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    return q


def graph_of(fn, pool=None):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, pool=pool, stream=s):
        fn()
    torch.cuda.synchronize()
    return g


def alternate(graphs, rounds, reps):
    """{arm: median ms per replay} over `rounds` rounds of `reps` replays per arm, arms alternated."""
    times = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            g.replay()
            a.record()
            for _ in range(reps):
                g.replay()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / reps)
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def site_arms(kind, shape, gs, layout, dtype, residual):
    from dwt_b200 import functional as F
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    n, c = shape[:2]
    fmt = torch.channels_last if layout == "cl" else torch.contiguous_format
    x = (torch.randn(shape, device=dev, generator=g) + 0.5).to(dtype).contiguous(memory_format=fmt).requires_grad_(True)
    r = torch.randn(shape, device=dev, generator=g).to(dtype).contiguous(memory_format=fmt).requires_grad_(True)
    dout = torch.randn(shape, device=dev, generator=g).to(dtype).contiguous(memory_format=fmt)
    w = torch.softmax(torch.randn(n, 3, device=dev, generator=g), 1).requires_grad_(True)
    gam = (1 + 0.1 * torch.randn(c, device=dev, generator=g)).requires_grad_(True)
    bet = (0.1 * torch.randn(c, device=dev, generator=g)).requires_grad_(True)
    rm = torch.zeros(3, c, device=dev)
    rv = torch.ones(3, c, device=dev) if kind == "bn" else torch.eye(gs, device=dev).expand(3, c // gs, gs, gs).contiguous()
    kw = dict(training_stats=True, eps=1e-5 if kind == "bn" else 1e-3, momentum=0.1, update_running=True,
              running=(rm, rv))
    res = r if residual else None
    inputs = (x, w, gam, bet) + ((r,) if residual else ())

    def fused():
        if kind == "bn":
            y = F.latent_domain_batch_norm(x, w, gam, bet, relu=True, residual=res, **kw)
        else:
            y = F.latent_domain_whiten(x, w, group_size=gs, weight=gam, bias=bet, relu=True, residual=res, **kw)
        torch.autograd.grad(y, inputs, dout)

    def aten():
        if kind == "bn":
            y = F.latent_domain_batch_norm(x, w, gam, bet, **kw)
        else:
            y = F.latent_domain_whiten(x, w, group_size=gs, **kw)
            y = y * gam.to(dtype).view(1, -1, 1, 1) + bet.to(dtype).view(1, -1, 1, 1)
        if residual:
            y = y + r
        torch.autograd.grad(torch.relu(y), inputs, dout)

    return {"fused": fused, "aten": aten}


def run_sites(args, gpu):
    for kind, shape, gs in SITES:
        for layout in ("nchw", "cl"):
            for dtype in (torch.float32, torch.bfloat16):
                for residual in (False, True):
                    arms = site_arms(kind, shape, gs, layout, dtype, residual)
                    graphs = {k: graph_of(f) for k, f in arms.items()}
                    t = alternate(graphs, args.rounds, args.reps)
                    print(json.dumps({"part": "site", "kind": kind, "shape": list(shape), "gs": gs, "layout": layout,
                                      "dtype": str(dtype).split(".")[1], "site": "relu+residual" if residual else "relu",
                                      "fused_ms": round(t["fused"], 4), "aten_ms": round(t["aten"], 4),
                                      "aten_over_fused": round(t["aten"] / t["fused"], 3), "gpu": gpu}), flush=True)
                    del graphs, arms
                    torch.cuda.empty_cache()


def run_model(args, gpu):
    import dwt_b200
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    dev = torch.device("cuda")
    torch.backends.cudnn.benchmark = True
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
    x, y = synth_batch(seed=2, per_domain=64, size=224)
    x, y = x.to(dev).contiguous(memory_format=torch.channels_last), y.to(dev)
    w = torch.softmax(torch.randn(192, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(3)), 1)
    models = {
        "latent_fused": (build_resnet50_dwt(sd, dwt_b200, site_mode="fused", domains="latent", channels_last=True), True),
        "latent_modules": (build_resnet50_dwt(sd, dwt_b200, site_mode="modules", domains="latent", channels_last=True),
                           True),
        "dwt_fused": (build_resnet50_dwt(sd, dwt_b200, site_mode="fused", channels_last=True), False)}
    for autocast in (False, True):
        graphs, pool = {}, torch.cuda.graph_pool_handle()
        for name, (m, latent) in models.items():
            m.to(dev).train()

            def step(m=m, latent=latent):
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                    logits = m(x, w) if latent else m(x)
                    loss = torch.nn.functional.cross_entropy(logits[:64].float(), y)
                loss.backward()
            graphs[name] = graph_of(step, pool)
        t = alternate(graphs, args.rounds, args.reps)
        print(json.dumps({"part": "model", "images": 192, "layout": "channels_last",
                          "dtype": "bf16 autocast" if autocast else "fp32",
                          **{f"{k}_ms": round(v, 3) for k, v in t.items()},
                          "modules_over_fused": round(t["latent_modules"] / t["latent_fused"], 3),
                          "latent_fused_over_dwt_fused": round(t["latent_fused"] / t["dwt_fused"], 3), "gpu": gpu}),
              flush=True)
        del graphs
        for m, _ in models.values():
            m.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sites", action="store_true")
    ap.add_argument("--model", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("latent_step.py measures on a CUDA device")
    gpu = card()
    if args.sites or not args.model:
        run_sites(args, gpu)
    if args.model or not args.sites:
        run_model(args, gpu)


if __name__ == "__main__":
    main()
