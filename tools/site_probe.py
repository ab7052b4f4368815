"""Scratch: run a few norm sites (fused domain triple, fwd+bwd) in isolation -- for ncu captures and
quick CUDA-event timings of single kernels.  Analysis only."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "dwt-domain-adaptation_b200"), ROOT]
import torch
import dwt_b200
from dwt_b200 import _native

SITES = [("whiten", 256, 56, 4), ("whiten", 64, 112, 4), ("whiten", 64, 56, 4), ("bn", 512, 28, 1),
         ("bn", 1024, 14, 1), ("bn", 2048, 7, 1), ("bn", 128, 28, 1), ("bn", 256, 14, 1), ("bn", 512, 7, 1)]

def main():
    dev = torch.device("cuda", 0)
    which = [int(a) for a in sys.argv[1:] if a.isdigit()] or range(len(SITES))
    cl = "cl" in sys.argv
    tail = "tail" in sys.argv           # residual tail + two gradient addends (fork_for_sum): the Bottleneck's last site
    iters = 3
    res = {}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for i in which:
        kind, c, h, gs = SITES[i]
        n = 64
        x = torch.randn(3 * n, c, h, h, device=dev)
        if cl:
            x = x.contiguous(memory_format=torch.channels_last)
        x.requires_grad_(True)
        dout = torch.randn_like(x)
        res_in = torch.randn_like(x).requires_grad_(True) if tail else None
        dout2 = torch.randn_like(x) if tail else None

        def fwd_bwd():
            if not tail:
                site(x, mods, g, b, relu=True).backward(dout)
                return
            a, bb = dwt_b200.fork_for_sum(site(x, mods, g, b, True, residual=res_in))
            torch.autograd.backward([a, bb], [dout, dout2])
        if kind == "whiten":
            mods = [dwt_b200.WTransform2d(c, gs).to(dev).train() for _ in range(3)]
        else:
            rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
            mods = [dwt_b200.BatchNorm2d(c, rm, rv, affine=False).train() for _ in range(3)]
        site = dwt_b200.DomainTripleNorm(kind, c, gs)
        g = torch.ones(c, 1, 1, device=dev, requires_grad=True); b = torch.zeros(c, 1, 1, device=dev, requires_grad=True)
        for _ in range(2):
            fwd_bwd()
        torch.cuda.synchronize()
        _native.profile_begin()
        for _ in range(iters):
            flush.zero_()                      # cold L2 between iterations
            fwd_bwd()
        prof = _native.profile_end()
        for k, v in prof.items():
            res[k] = dict(us=1e3 * v["ms"] / v["launches"], gbs=v["bytes"] / v["ms"] / 1e6)
    for k, v in sorted(res.items()):
        print(f"{k:40s} {v['us']:8.1f} us {v['gbs']:7.0f} GB/s  {v['gbs']/3350.0:5.2f}")

if __name__ == "__main__":
    main()
