"""CPU emulation of the tf32 Gram contraction of the forward statistics (csrc/norm_tc.cu): covariance and y error of

  single   G = sum RN_tf32(s) RN_tf32(s)^T                        (round-1 kernel: one tf32 pass)
  split    G = HH + LH + LH^T,  hi = trunc_tf32(s), lo = trunc_tf32(s - hi): the products of tc_gram_kernel -- the
           tensor core reads the top 19 bits of the fp32 words it is handed (s itself for hi, s - trunc(s) for lo)
  split-rn the same with hi = RN_tf32(s) (the first round-2 kernel: two more instructions per element)
  fp32     the same sums with fp32 operands                        (what the reference's torch.bmm computes)

against the fp64 covariance, over condition number, activation scale and |mean|/sigma.  s = x - K with the pilot
shift K; products are exact in fp32 and the accumulation is emulated in fp64; optionally with a truncating fp32
accumulator per 8-sample MMA step (--rz) as a pessimistic model of the tensor core's accumulate.  The kernel's per-CTA
partials are not a few thousand samples: a Gram CTA covers N*HW*SB / (2 SMs) samples of its super-block, about 12,000
(380 tiles of 32 pixels) at BASELINE config 2 on 132 SMs.  So it sums each 32-pixel tile in a fresh tensor-core
accumulator and the tiles in fp32 registers; one accumulator per CTA drifted 3.9e-5 from the fp64 covariance there
(tests/test_tc_forward_stats_fp64.py), which the fp64 accumulation here does not model.  Pure numpy.
      python tools/tf32_gram_accuracy.py [--rz]
"""
import sys

import numpy as np


def rn(a):
    u = a.astype(np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)


def tr(a):
    return (a.astype(np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)


def acc(a, b, rz, chunk=2048):
    """sum_m a[:, m] b[:, m]^T; rz: per-CTA chunks accumulated 8 samples at a time into a TRUNCATED fp32 accumulator."""
    if not rz:
        return a @ b.T
    tot = np.zeros((a.shape[0], b.shape[0]))
    for c0 in range(0, a.shape[1], chunk):
        d = np.zeros((a.shape[0], b.shape[0]), np.float32)
        for k in range(c0, min(c0 + chunk, a.shape[1]), 8):
            t = d.astype(np.float64) + a[:, k:k + 8] @ b[:, k:k + 8].T
            t32 = t.astype(np.float32)
            over = np.abs(t32.astype(np.float64)) > np.abs(t)          # RN went away from zero: step back one ulp
            d = np.where(over, np.nextafter(t32, np.float32(0)), t32)
        tot += d.astype(np.float64)
    return tot


def run(M, gs=64, cond=1e2, scale=1.0, mos=2.0, seed=0, rz=False):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((gs, gs)))
    x = (q * (scale * np.sqrt(np.logspace(0, -np.log10(cond), gs)))) @ rng.standard_normal((gs, M))
    x = x + mos * x.std(1, keepdims=True)
    K = x[:, M // 2 - 16:M // 2 + 16].mean(1, keepdims=True) if M >= 32 else x.mean(1, keepdims=True)   # pilot shift
    xs = (x.astype(np.float32) - K.astype(np.float32)).astype(np.float32).astype(np.float64)
    s1 = xs.sum(1, keepdims=True) / M
    exact = np.cov(x, bias=True)
    w = lambda c: np.linalg.inv(np.linalg.cholesky((1 - 1e-3) * c + 1e-3 * np.eye(gs)))       # noqa: E731
    xc = x - x.mean(1, keepdims=True)
    y64 = w(exact) @ xc
    hi = tr(xs)
    lh = acc(tr(xs - hi), hi, rz)
    hr = rn(xs)
    lhr = acc(tr(xs - hr), hr, rz)
    grams = {"single": acc(rn(xs), rn(xs), rz), "split": acc(hi, hi, rz) + lh + lh.T,
             "split-rn": acc(hr, hr, rz) + lhr + lhr.T, "fp32": acc(xs, xs, False)}
    out = {}
    for name, g in grams.items():
        c = g / M - s1 @ s1.T
        out[name] = (np.linalg.norm(c - exact) / np.linalg.norm(exact), np.linalg.norm(w(c) @ xc - y64) / np.linalg.norm(y64))
    return out


NAMES = ("single", "split", "split-rn", "fp32")


if __name__ == "__main__":
    rz = "--rz" in sys.argv
    M = 4704 if rz else 65536
    print(f"M = {M}, gs = 64, eps = 1e-3" + (", truncating fp32 accumulator per 8-sample step" if rz else ""))
    print(f"{'cond':>6} {'scale':>6} {'|mu|/sd':>8} | " + " | ".join(f"{n + ' cov':>11} {n + ' y':>10}" for n in NAMES))
    for cond, scale, mos in [(1e2, 1, 2), (1e3, 10, 0), (1e4, 30, 0), (1e4, 100, 0), (1e1, 1, 50), (1e3, 10, 50)]:
        r = run(M, cond=cond, scale=scale, mos=mos, rz=rz)
        print(f"{cond:6.0e} {scale:6.0f} {mos:8.0f} | " + " | ".join(f"{r[n][0]:11.2e} {r[n][1]:10.2e}" for n in NAMES))
