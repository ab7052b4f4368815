"""CPU emulation of the backward contraction R = sum dy xc^T (csrc/norm_tc.cu, tc_contract_kernel) against fp64: how
far does dx land from fp64 when the output gradient has a per-channel offset or lies mostly along y?

  1-pass          R = RN_tf32(dy) RN_tf32(xc)^T                          (the kernel before it was split and centred)
  split+centred   e = dy - K (K: mean of image 0's 32 mid pixels per channel, the kernel's pilot shift), hi =
                  trunc_tf32(s), lo = s - hi for s = e and s = xc, then
                  R = Eh Xh^T + El Xh^T + Eh Xl^T                         (the kernel now; sum xc = 0 up to rounding)
  centred only    R = RN_tf32(e) RN_tf32(xc)^T + K (sum xc)^T             (for contrast: fixes the offset, not y-aligned dy)
  plain fp32      R in float32 (numpy matmul): about what the reference's float32 operator sequence reaches
Products are exact (fp64); the tensor core's fp32 accumulation, the CTA-level tiling and accumulation over many tiles
are not modelled, so the tool says nothing about long accumulations (tests/test_tc_backward_fp64.py measures those).
xc is formed with the fp32-rounded batch mean, as the kernel forms it from save_mean.  With dy's per-channel mean in
the product, that rounding puts a floor under 'plain fp32' and 'centred only' (for example 4.4e-4 at offset 100 sigma
and condition number 1e3); 'split+centred' multiplies e = dy - K, whose mean is small, so the floor mostly goes.  R is pushed through
oracle/dwt_oracle.whiten_backward's closed form; prints the norm-wise relative error of dx against fp64, one group of
gs = 64 channels at M = N*HW = 4096 samples (the fewest the tensor-core kernels take).  Pure numpy; no GPU.

    python tools/tf32_contract_accuracy.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import dwt_oracle as O  # noqa: E402


def rn_tf32(a):
    u = np.asarray(a, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def trunc_tf32(a):
    return (np.asarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def conditioned(rng, n, gs, hw, cond):
    """[n, gs, hw] samples of covariance eigenvalues 1 .. 1/cond in a random basis, mean 2."""
    q, _ = np.linalg.qr(rng.standard_normal((gs, gs)))
    a = q * np.sqrt(np.logspace(0, -np.log10(cond), gs))[None, :]
    return np.einsum("ij,njm->nim", a, rng.standard_normal((n, gs, hw))) + 2.0


def dx_from_r(xc, gy, w, r, eps=1e-3):
    """oracle.whiten_backward's closed form for one group with dW = R given: xc, gy [gs, M], w [gs, gs]."""
    p = np.tril(-r @ w.T)
    p[np.diag_indices_from(p)] *= 0.5
    s = w.T @ p @ w
    s = 0.5 * (s + s.T)
    return w.T @ (gy - gy.mean(1, keepdims=True)) + (2.0 * (1.0 - eps) / xc.shape[1]) * (s @ xc)


def run(cond, kind, seed=0, n=128, gs=64, hw=32):
    rng = np.random.default_rng(seed)
    x = conditioned(rng, n, gs, hw, cond).astype(np.float32)                 # [n, gs, hw], what the kernel reads
    y, mean, w, *_ = O.whiten_forward(x.astype(np.float64)[:, :, :, None], gs)
    y, w = y[..., 0], w[0]
    gain = rng.uniform(0.5, 1.5, (1, gs, 1))
    sign = np.where(rng.random((1, gs, 1)) < 0.5, -1.0, 1.0) * rng.uniform(0.5, 1.5, (1, gs, 1))
    sigma, off, aligned = {"randn": (1.0, 0, 0), "offset10": (1.0, 10, 0), "offset100": (1.0, 100, 0),
                           "y+0.01": (0.01, 0, 1), "y+0.1,offset10": (0.1, 10, 1)}[kind]
    dy = (aligned * y * gain + sigma * rng.standard_normal(x.shape) + off * sign).astype(np.float32)
    flat = lambda a: np.moveaxis(a, 1, 0).reshape(gs, -1)                   # noqa: E731  [n, gs, hw] -> [gs, M]
    xc32 = flat((x - mean.astype(np.float32).reshape(1, gs, 1)).astype(np.float32))
    gy32 = flat(dy)
    xc64, gy = flat(x.astype(np.float64)) - mean[:, None], gy32.astype(np.float64)
    dx64 = dx_from_r(xc64, gy, w, gy @ xc64.T)
    d64 = lambda a: np.asarray(a, np.float64)                                # noqa: E731
    p0 = (hw - 32) // 2 & ~3
    k = dy[0, :, p0:p0 + 32].mean(1, dtype=np.float32)[:, None]              # the pilot shift of dy
    e32 = (gy32 - k).astype(np.float32)
    fold = d64(k) @ d64(xc32.sum(1, dtype=np.float32))[None, :]
    eh, el = trunc_tf32(e32), e32 - trunc_tf32(e32)
    xh, xl = trunc_tf32(xc32), xc32 - trunc_tf32(xc32)
    rs = {
        "1-pass": d64(rn_tf32(gy32)) @ d64(rn_tf32(xc32)).T,
        "split+centred": d64(eh) @ d64(xh).T + d64(trunc_tf32(el)) @ d64(xh).T + d64(eh) @ d64(trunc_tf32(xl)).T,
        "centred only": d64(rn_tf32(e32)) @ d64(rn_tf32(xc32)).T + fold,
        "plain fp32": d64(gy32 @ xc32.T),
    }
    return {name: float(np.linalg.norm(dx_from_r(xc64, gy, w, r) - dx64) / np.linalg.norm(dx64)) for name, r in rs.items()}


if __name__ == "__main__":
    names = ("1-pass", "split+centred", "centred only", "plain fp32")
    print(f"{'dy':>16} {'cond':>6} | " + " ".join(f"{v:>14}" for v in names))
    for kind in ("randn", "offset10", "offset100", "y+0.01", "y+0.1,offset10"):
        for cond in (1.0, 1e3):
            r = run(cond, kind)
            print(f"{kind:>16} {cond:6.0e} | " + " ".join(f"{r[v]:14.2e}" for v in names))
