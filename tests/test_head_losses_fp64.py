"""The MEC loss and the fused head loss (csrc/mec.cu) against an fp64 reference, at their launch edges and in the value
regimes where a log-softmax kernel goes wrong.

The benchmark step ends in dwt_head_loss_fwd_bwd (NLL of the source logits + lambda * MEC of the target pair): the loss
users watch and the gradient that starts the whole backward pass both come from it.  dwt_mec_fwd_bwd is the same MEC
term behind MinEntropyConsensusLoss.  Both are one CTA of min(32 * rows, kMecThreads) threads, one warp per row (pair).

Reference: the formulas of oracle/dwt_oracle.py in torch float64 on the device, so the large cases stay fast:
log_softmax as z - log(sum exp z) with z = a - max a; the MEC term of mec_loss, s = -(lsm(x) + lsm(y)) / 2, the first
minimum per row with a NaN winning (np.argmin / torch.min: the first NaN), gradient (softmax - onehot(k*)) / 2N; the
classification term NLL(log_softmax) with F.nll_loss's ignore_index = -100 (such rows leave the sum and the
denominator; every label outside [0, K) is dropped like one and sets STATUS_BAD_LABEL).  The inputs are fp32 values and
the reference sees exactly those values.  test_fp64_reference_matches_the_oracle pins the restatement to
oracle.dwt_oracle.mec_loss (numpy) and to F.nll_loss on the CPU.

Compared for every case: the loss, HeadLoss.parts (total, classification, lambda * MEC) and every gradient row at an
upstream gradient of 1.7; the launch profile (exactly one mec or head_loss launch) and the status word.  Rows whose fp32
minimum lies within rounding of another class may legitimately take a different class than fp64: the kernel's class k*
is read from its gradient (the one negative entry of gx + gy), s64[k*] - min s64 must be at most 1e-6 (1 + |min s64|),
and the gradient is compared with the fp64 gradient built with that k*.  Exact ties (duplicated columns) must take the
first class.

Bounds: gradients 1e-5 norm-wise over the tensor and per row, max-elementwise 5e-5, each relative to the reference
gradient and never to less than its one-hot scale (G / 2N, G lambda / 2B or G / #valid labels per row); losses 1e-6
relative plus the fp32 summation bound of the kernels' two-level sum of non-negative row terms, 2^-24 (rows per warp +
warps).  Rows whose max is below 64 in magnitude keep the earlier log-softmax form x - (mx + log sx) bit for bit; rows
beyond it, every offset case here, take (x - mx) - log sx.
"""
import ctypes
import math
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEC_CU = os.path.join(ROOT, "dwt-domain-adaptation_b200", "dwt_b200", "csrc", "mec.cu")
gpu = pytest.mark.gpu


def _kernel_threads():
    m = re.search(r"constexpr int kMecThreads = (\d+);", open(MEC_CU).read())
    assert m, "kMecThreads not found in csrc/mec.cu"
    return int(m.group(1))


THREADS = _kernel_threads()     # the CTA's thread cap
LANES = 32                      # one warp per row: lane l reads classes l, l + 32, ...
WARPS = THREADS // LANES
B_CAP = THREADS // (2 * LANES)  # the head loss's 2B rows fill every warp from here on
UPSTREAM = 1.7
LAM = 0.1
TOL_GRAD = 1e-5
TOL_MAX = 5e-5
TOL_LOSS = 1e-6
TOL_TIE = 1e-6
U32 = 2.0 ** -24

# [N, K] of the MEC calls: every N edge (1, 2, one warp short of / at / past the warp count, two rows per warp, one
# thread short of / at / past the thread count, many rows per warp) with one K below and one above the 32 lanes
K_LO, K_EDGE, K_HI = (1, 2, 10, LANES - 1), (LANES,), (LANES + 1, 2 * LANES, 2 * LANES + 1, 345, 1000)
MEC_SHAPES = [(1, 1), (1, LANES + 1), (1, 1000), (2, 2), (2, 2 * LANES + 1), (WARPS - 1, LANES - 1),
              (WARPS - 1, 2 * LANES), (WARPS, LANES), (WARPS, 10), (WARPS, 2 * LANES + 1), (WARPS + 1, 1),
              (WARPS + 1, LANES + 1), (2 * WARPS, 10), (2 * WARPS, 2 * LANES + 1), (2 * WARPS, 345),
              (THREADS - 1, LANES - 1), (THREADS - 1, LANES + 1), (THREADS, 2), (THREADS, 2 * LANES + 1),
              (THREADS + 1, 10), (THREADS + 1, 2 * LANES), (4096, 1), (4096, LANES), (4096, 345), (4096, 1000),
              (65536, 10), (65536, 2 * LANES + 1)]
MEC_N = (1, 2, WARPS - 1, WARPS, WARPS + 1, 2 * WARPS, THREADS - 1, THREADS, THREADS + 1, 4096, 65536)
# [B, K] of the head-loss calls (3B logit rows, 2B warp rows): B at the thread cap, and where 2B meets the thread count
HEAD_SHAPES = [(1, 1), (1, 2 * LANES + 1), (2, 10), (2, LANES + 1), (B_CAP - 1, LANES - 1), (B_CAP - 1, 2 * LANES),
               (B_CAP, LANES), (B_CAP, 2), (B_CAP, 2 * LANES + 1), (B_CAP + 1, 10), (B_CAP + 1, 345),
               (4 * B_CAP, 1), (4 * B_CAP, 2 * LANES + 1), (THREADS // 2 - 1, LANES - 1), (THREADS // 2 - 1, LANES + 1),
               (THREADS // 2, 10), (THREADS // 2, 2 * LANES + 1), (THREADS // 2 + 1, 2), (THREADS // 2 + 1, 2 * LANES),
               (4096, 10), (4096, 2 * LANES + 1), (4096, 1000)]
HEAD_B = (1, 2, B_CAP - 1, B_CAP, B_CAP + 1, 4 * B_CAP, THREADS // 2 - 1, THREADS // 2, THREADS // 2 + 1, 4096)


def _ids(shapes, a):
    return [f"{a}{s[0]}-K{s[1]}" for s in shapes]


# --------------------------------------------------------------------------- the fp64 reference (device-agnostic)
def _lsm64(a):
    z = a.double() - a.double().amax(dim=1, keepdim=True)
    return z - z.exp().sum(dim=1, keepdim=True).log()


def _first_min(s):
    """np.argmin's class per row: the first NaN if the row has one, else the first minimum."""
    k = s.shape[1]
    idx = torch.arange(k, device=s.device).expand_as(s)
    nan = s.isnan()
    first_nan = torch.where(nan, idx, k).amin(dim=1)
    first_min = torch.where(s == s.amin(dim=1, keepdim=True), idx, k).amin(dim=1)
    return torch.where(nan.any(dim=1), first_nan, first_min)


def _mec64(x, y):
    """-> s [N, K], softmax(x), softmax(y) in float64."""
    lx, ly = _lsm64(x), _lsm64(y)
    return -0.5 * (lx + ly), lx.exp(), ly.exp()


def _onehot(k, n_cls):
    return torch.nn.functional.one_hot(k, n_cls).double()


def _nll64(src, labels):
    """F.nll_loss(log_softmax(src), labels) (mean, ignore_index -100; other out-of-range labels dropped) and its
    gradient; -> (loss, grad [B, K], number of counted rows)."""
    k = src.shape[1]
    ls = _lsm64(src)
    valid = (labels >= 0) & (labels < k)
    nv = int(valid.sum())
    y = torch.where(valid, labels, 0)
    picked = -ls.gather(1, y[:, None])[:, 0]
    loss = torch.where(valid, picked, 0.0).sum() / nv if nv else torch.tensor(float("nan"), dtype=torch.float64)
    grad = torch.where(valid[:, None], ls.exp() - _onehot(y, k), 0.0) / max(nv, 1)
    return loss, grad, nv


# --------------------------------------------------------------------------- CPU part
def test_shape_sets_cover_the_launch_edges():
    """Every N (B) edge of the kernels is run with at least one K below and one above the 32 lanes, every K edge is run,
    and the edges follow kMecThreads."""
    assert THREADS % LANES == 0 and WARPS >= 2
    for shapes, edges in ((MEC_SHAPES, MEC_N), (HEAD_SHAPES, HEAD_B)):
        assert {s[0] for s in shapes} == set(edges)
        assert {s[1] for s in shapes} == set(K_LO + K_EDGE + K_HI)
        for n in edges:
            ks = [k for m, k in shapes if m == n]
            assert any(k < LANES for k in ks) and any(k > LANES for k in ks), (n, ks)
    assert 2 * B_CAP * LANES == THREADS


def test_fp64_reference_matches_the_oracle():
    """The torch float64 restatement used on the device equals oracle.dwt_oracle.mec_loss (numpy, pinned to the
    reference by test_oracle_vs_golden.py) and F.nll_loss, on random rows, exact ties, a NaN, +inf and -inf."""
    import numpy as np
    import torch.nn.functional as Fn
    from oracle import dwt_oracle as O
    gen = torch.Generator().manual_seed(0)
    x, y = 3 * torch.randn(12, 70, generator=gen), 3 * torch.randn(12, 70, generator=gen)
    x[1, 40] = y[1, 40] = 20.0                           # a tie 3 / 40 as the row minimum
    x[1, 3], y[1, 3] = x[1, 40], y[1, 40]
    x[2, [0, 31, 32]] = y[2, [0, 31, 32]] = 25.0         # a three-way tie across the lane wrap
    x[4, 9] = float("nan")
    y[5, 60] = float("nan")
    x[6, 2] = float("inf")
    x[7, :50] = float("-inf")                            # masked classes: finite loss (the oracle's value)
    y[8, 10:] = float("-inf")
    for a, b in ((x, y), (x[:, :1], y[:, :1]), (x[:, :31], y[:, :31])):
        with np.errstate(invalid="ignore"):              # the NaN / inf rows
            loss_o, gx_o, gy_o, k_o = O.mec_loss(a.double().numpy(), b.double().numpy())
        s, px, py = _mec64(a, b)
        k = _first_min(s)
        assert np.array_equal(k.numpy(), k_o)
        n = a.shape[0]
        hot = _onehot(k, a.shape[1])
        loss = s.gather(1, k[:, None]).mean()
        np.testing.assert_allclose(loss.numpy(), loss_o, rtol=1e-14, equal_nan=True)
        np.testing.assert_allclose(((px - hot) / (2 * n)).numpy(), gx_o, rtol=1e-12, atol=1e-15, equal_nan=True)
        np.testing.assert_allclose(((py - hot) / (2 * n)).numpy(), gy_o, rtol=1e-12, atol=1e-15, equal_nan=True)
    k = _first_min(_mec64(x, y)[0])
    assert k[1] == 3 and k[2] == 0 and k[4] == k[5] == k[6] == 0      # first of a tie; first NaN of a NaN row
    with np.errstate(invalid="ignore"):
        assert math.isnan(O.mec_loss(x.double().numpy(), y.double().numpy())[0])
    assert math.isfinite(O.mec_loss(x[7:9].double().numpy(), y[7:9].double().numpy())[0])
    for labels in ([3, -100, 7, 0, -100, 69, 1, 2, 5, 9, 11, 4], [-100] * 12):
        lab = torch.tensor(labels)
        src = x[9:12].repeat(4, 1).double().requires_grad_(True)
        want = Fn.nll_loss(Fn.log_softmax(src, dim=1), lab)
        got, grad, nv = _nll64(src.detach(), lab)
        assert nv == sum(v != -100 for v in labels)
        np.testing.assert_allclose(got.numpy(), want.detach().numpy(), rtol=1e-14, equal_nan=True)
        if nv:
            want.backward()
            np.testing.assert_allclose(grad.numpy(), src.grad.numpy(), rtol=1e-12, atol=1e-15)


@pytest.fixture(scope="module")
def built_lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native


def test_c_abi_refusals(built_lib):
    """Both entry points refuse null pointers and out-of-range shapes before touching a pointer (fake ones here: every
    call below is refused, none reaches a launch)."""
    lib = built_lib.lib()
    p = ctypes.c_void_p(0x1000)

    def mec(n, k, nulls=()):
        args = [None if i in nulls else p for i in range(5)]
        rc = lib.dwt_mec_fwd_bwd(args[0], args[1], n, k, args[2], args[3], args[4], None)
        return rc, lib.dwt_last_error().decode()

    def head(b, k, nulls=()):
        args = [None if i in nulls else p for i in range(4)]
        rc = lib.dwt_head_loss_fwd_bwd(args[0], args[1], b, k, 0.1, args[2], args[3], None, None)
        return rc, lib.dwt_last_error().decode()
    for i in range(5):
        assert mec(4, 5, nulls=(i,)) == (-1, "null pointer argument"), i
    for i in range(4):
        assert head(4, 5, nulls=(i,)) == (-1, "null pointer argument"), i
    for n, k in ((0, 5), (-1, 5), (4, 0), (4, -3), (1 << 24, 5), (4, 1 << 24), (1 << 40, 1 << 40)):
        assert mec(n, k) == (-1, f"bad logits shape [{n},{k}]"), (n, k)
    for b, k in ((0, 5), (-2, 5), (4, 0), (1 << 22, 5), (4, 1 << 24), (1 << 40, 7)):
        assert head(b, k) == (-1, f"bad logits shape [3*{b},{k}]"), (b, k)


def test_python_shape_refusals(built_lib):
    """Shape errors are raised before any device check: MEC inputs of different or non-2-D shapes, logits that are not
    [3B, K] against labels [B]."""
    import dwt_b200
    mec, head = dwt_b200.MinEntropyConsensusLoss(5, "cpu"), dwt_b200.HeadLoss(5, 0.1)
    for a, b in (((4, 5), (4, 6)), ((4, 5), (3, 5)), ((20,), (20,)), ((2, 2, 5), (2, 2, 5))):
        with pytest.raises(ValueError, match=r"expected two \[N, K\] logit tensors"):
            mec(torch.zeros(a), torch.zeros(b))
    for shape, nl in (((6, 5), 3), ((7, 5), 2), ((6, 5), 1), ((30,), 10)):
        with pytest.raises(ValueError, match=r"expected logits \[3B, K\] and labels \[B\]"):
            head(torch.zeros(shape), torch.zeros(nl, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"labels \[B\]"):
        head(torch.zeros(6, 5), torch.zeros(2, 1, dtype=torch.int64))


# --------------------------------------------------------------------------- GPU harness
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst(dev):
    """Worst error per case group, printed at the end."""
    table = {}
    yield table
    print("\nworst errors per case group (loss: relative; grad: norm-wise / worst row / max-elementwise; "
          "tie: (s64[k*] - min s64) / (1 + |min s64|)):")
    for group in sorted(table):
        print("  %-16s %s" % (group, "  ".join(f"{k} {v:.1e}" for k, v in sorted(table[group].items()))))


def _upstream(dev):
    return torch.tensor(UPSTREAM, device=dev)


G64 = float(torch.tensor(UPSTREAM))          # the float32 upstream gradient, as the reference's factor


def _logits(gen, shape, dev, scale=3.0, offset=0.0):
    """scale * randn, plus a common offset per row of magnitude offset .. 2 offset and random sign."""
    z = scale * torch.randn(shape, device=dev, generator=gen)
    if offset:
        sign = torch.randint(0, 2, (shape[0], 1), device=dev, generator=gen) * 2 - 1
        z += sign * offset * (1 + torch.rand(shape[0], 1, device=dev, generator=gen))
    return z


def _labels(gen, b, k, dev, mode="mixed"):
    """valid: all in [0, K); mixed: every fifth from the second on is -100; ignored: all -100; bad: mixed, plus
    labels K, K + 7, -1, -3 and 2^40 where B allows."""
    lab = torch.randint(0, k, (b,), device=dev, generator=gen)
    if mode in ("mixed", "bad"):
        lab[1::5] = -100
    if mode == "ignored":
        lab[:] = -100
    if mode == "bad":
        for i, v in zip(range(0, b, 3), (k, k + 7, -1, -3, 1 << 40)):
            lab[i] = v
    return lab


def _profiled(fn):
    from dwt_b200 import _native
    _native.profile_begin()
    try:
        out = fn()
    finally:
        prof = _native.by_family(_native.profile_end())
    return out, prof


def _mec_call(x, y, dev):
    """MinEntropyConsensusLoss on x, y (as they are: views, bf16) -> loss, gx, gy at the upstream gradient, the launch
    profile and the status word."""
    import dwt_b200
    from dwt_b200 import _native
    xl, yl = x.detach().requires_grad_(True), y.detach().requires_grad_(True)
    _native.clear_status(dev)
    loss, prof = _profiled(lambda: dwt_b200.MinEntropyConsensusLoss(x.shape[1], dev)(xl, yl))
    gx, gy = torch.autograd.grad(loss, (xl, yl), _upstream(dev))
    return loss.detach(), gx, gy, prof, _native.status(dev)


def _head_call(logits, labels, dev, lam=LAM):
    """HeadLoss -> total, parts, grad at the upstream gradient, the launch profile and the status word."""
    import dwt_b200
    from dwt_b200 import _native
    head = dwt_b200.HeadLoss(logits.shape[1], lam)
    ll = logits.detach().requires_grad_(True)
    _native.clear_status(dev)
    total, prof = _profiled(lambda: head(ll, labels))
    (grad,) = torch.autograd.grad(total, ll, _upstream(dev))
    status = _native.status(dev)
    _native.clear_status(dev)
    return total.detach(), head.parts, grad, prof, status


def _loss_tol(rows):
    """1e-6 plus the fp32 summation bound of the kernels' loss: each warp adds its rows in order, thread 0 the warps."""
    warps = min(WARPS, rows)
    return TOL_LOSS + U32 * (-(-rows // warps) + warps + 4)


def _scalar(label, name, got, ref, tol):
    got, ref = float(got), float(ref)
    if math.isnan(ref):
        assert math.isnan(got), (label, name, got, ref)
        return 0.0
    assert math.isfinite(got), (label, name, got, ref)
    rel = abs(got - ref) / abs(ref) if ref else abs(got)
    assert rel <= tol, (label, name, got, ref, rel, tol)
    return rel


def _grad_err(label, got, ref, row_scale):
    """(norm-wise, worst row relative to its one-hot scale, max-elementwise) over the rows the reference keeps finite;
    NaN exactly where the reference has NaN.  The norm-wise and max-elementwise errors are relative to the gradient but
    never to less than its one-hot scale: where a row's softmax saturates at k*, p - 1 cancels and the gradient can be
    far smaller than the fp32 rounding of p allows to resolve."""
    nan = ref.isnan()
    assert torch.equal(got.isnan(), nan), (label, "NaN pattern", got.isnan().nonzero()[:8].tolist(), nan.nonzero()[:8].tolist())
    keep = ~nan.any(dim=1)
    if not keep.any():
        return 0.0, 0.0, 0.0
    d, r, sc = got.double()[keep] - ref[keep], ref[keep], row_scale[keep]
    normwise = (d.norm() / torch.maximum(r.norm(), sc.norm()).clamp_min(1e-300)).item()
    row = (d.norm(dim=1) / sc).max().item()
    mx = (d.abs().max() / torch.maximum(r.abs().max(), sc.max()).clamp_min(1e-300)).item()
    return normwise, row, mx


def _kernel_class(g_pair, s, k_ref):
    """The kernel's class per MEC row, from its gradient: the one negative entry of gx + gy ((p_x + p_y - 2) / 2N at
    k*).  Rows without one (p_x = p_y = 1 in fp32 at k*) and rows the reference makes NaN keep the reference's class."""
    mn, am = g_pair.double().min(dim=1)
    return torch.where((mn < 0) & ~s.isnan().any(dim=1), am, k_ref)


def _tie_margin(label, s, k_star, k_ref, exact_k):
    rows = ~s.isnan().any(dim=1)
    if exact_k:
        assert torch.equal(k_star, k_ref), (label, (k_star != k_ref).nonzero()[:8].tolist())
    if not rows.any():
        return 0.0
    smin = s.gather(1, k_ref[:, None])[:, 0][rows]
    margin = ((s.gather(1, k_star[:, None])[:, 0][rows] - smin) / (1 + smin.abs())).max().item()
    assert margin <= TOL_TIE, (label, "k* is not an fp64 near-minimum", margin)
    return margin


def _record(worst, group, **errs):
    t = worst.setdefault(group, {})
    for k, v in errs.items():
        t[k] = max(t.get(k, 0.0), v)


def _check_grads(label, errs):
    for name, (normwise, row, mx) in errs.items():
        assert normwise <= TOL_GRAD and row <= TOL_GRAD and mx <= TOL_MAX, (label, name, normwise, row, mx)


def check_mec(dev, worst, group, x, y, label, exact_k=False):
    """One MinEntropyConsensusLoss call against the fp64 reference."""
    n, k = x.shape
    loss, gx, gy, prof, status = _mec_call(x, y, dev)
    assert set(prof) == {"mec"} and prof["mec"]["launches"] == 1, (label, prof)
    assert status == 0, (label, status)
    s, px, py = _mec64(x, y)
    k_ref = _first_min(s)
    k_star = _kernel_class(gx + gy, s, k_ref)
    tie = _tie_margin(label, s, k_star, k_ref, exact_k)
    hot, sc = _onehot(k_star, k), G64 / (2 * n)
    rel = _scalar(label, "loss", loss, s.gather(1, k_star[:, None]).mean(), _loss_tol(n))
    row_scale = torch.full((n,), sc, dtype=torch.float64, device=x.device)
    errs = {"gx": _grad_err(label, gx, sc * (px - hot), row_scale), "gy": _grad_err(label, gy, sc * (py - hot), row_scale)}
    _record(worst, group, loss=rel, grad=max(e[0] for e in errs.values()), row=max(e[1] for e in errs.values()),
            max=max(e[2] for e in errs.values()), tie=tie)
    print(label, "loss %.1e tie %.1e" % (rel, tie), {k: "%.1e %.1e %.1e" % e for k, e in errs.items()})
    _check_grads(label, errs)
    return loss, gx, gy


def check_head(dev, worst, group, logits, labels, label, lam=LAM, exact_k=False, bad_label=False):
    """One HeadLoss call against the fp64 reference."""
    from dwt_b200 import _native
    b, k = labels.shape[0], logits.shape[1]
    total, parts, grad, prof, status = _head_call(logits, labels, dev, lam)
    assert set(prof) == {"head_loss"} and prof["head_loss"]["launches"] == 1, (label, prof)
    assert status == (_native.STATUS_BAD_LABEL if bad_label else 0), (label, status)
    assert torch.allclose(total, parts[0], rtol=0, atol=0, equal_nan=True), label
    lamf = float(torch.tensor(lam))                      # the kernel's float lambda
    cls, g_src, nv = _nll64(logits[:b], labels)
    s, px, py = _mec64(logits[b:2 * b], logits[2 * b:])
    k_ref = _first_min(s)
    k_star = _kernel_class(grad[b:2 * b] + grad[2 * b:], s, k_ref)
    tie = _tie_margin(label, s, k_star, k_ref, exact_k)
    hot, sc = _onehot(k_star, k), G64 * lamf / (2 * b)
    mec = lamf * s.gather(1, k_star[:, None]).mean()
    tol = _loss_tol(2 * b)
    rel = max(_scalar(label, "total", parts[0], cls + mec, tol), _scalar(label, "classification", parts[1], cls, tol),
              _scalar(label, "lambda*MEC", parts[2], mec, tol))
    row_scale = torch.cat([torch.full((b,), G64 / max(nv, 1), dtype=torch.float64, device=logits.device),
                           torch.full((2 * b,), sc, dtype=torch.float64, device=logits.device)])
    ref = torch.cat([G64 * g_src, sc * (px - hot), sc * (py - hot)])
    errs = {"grad": _grad_err(label, grad, ref, row_scale)}
    ignored = ~((labels >= 0) & (labels < k))
    assert torch.equal(grad[:b][ignored], torch.zeros_like(grad[:b][ignored])), (label, "dropped source rows")
    _record(worst, group, loss=rel, grad=errs["grad"][0], row=errs["grad"][1], max=errs["grad"][2], tie=tie)
    print(label, "loss %.1e tie %.1e" % (rel, tie), {k: "%.1e %.1e %.1e" % e for k, e in errs.items()})
    _check_grads(label, errs)
    return total, parts, grad


# --------------------------------------------------------------------------- 1. launch edges
@gpu
@pytest.mark.parametrize("n,k", MEC_SHAPES, ids=_ids(MEC_SHAPES, "N"))
def test_mec_shapes(n, k, dev, worst):
    gen = torch.Generator(device=dev).manual_seed(n + 7 * k)
    check_mec(dev, worst, "mec_shapes", _logits(gen, (n, k), dev), _logits(gen, (n, k), dev), f"mec {n}x{k}")


@gpu
@pytest.mark.parametrize("b,k", HEAD_SHAPES, ids=_ids(HEAD_SHAPES, "B"))
def test_head_loss_shapes(b, k, dev, worst):
    gen = torch.Generator(device=dev).manual_seed(b + 7 * k)
    check_head(dev, worst, "head_shapes", _logits(gen, (3 * b, k), dev), _labels(gen, b, k, dev), f"head {b}x{k}")


LABEL_MODES = [("valid", 17, 65), ("valid", 513, 33), ("mixed", 1, 10), ("ignored", 17, 65), ("ignored", 1, 65),
               ("bad", 17, 65), ("bad", 513, 10)]


@gpu
@pytest.mark.parametrize("mode,b,k", LABEL_MODES, ids=[f"{m}-B{b}-K{k}" for m, b, k in LABEL_MODES])
def test_head_loss_labels(mode, b, k, dev, worst):
    """All valid, some -100, all -100 (classification NaN as F.nll_loss gives it, source rows' gradient zero, status
    clear) and labels outside [0, K) (those rows dropped, STATUS_BAD_LABEL and nothing else)."""
    gen = torch.Generator(device=dev).manual_seed(b + k)
    labels = _labels(gen, b, k, dev, mode)
    total, parts, grad = check_head(dev, worst, "labels", _logits(gen, (3 * b, k), dev), labels,
                                    f"labels {mode} {b}x{k}", bad_label=mode == "bad")
    if mode == "ignored":
        assert math.isnan(parts[1].item()) and math.isnan(total.item()) and math.isfinite(parts[2].item())
        assert not grad[:b].any() and grad[b:].isfinite().all()


# --------------------------------------------------------------------------- 2. value regimes
REGIMES = {"scale1e-3": (1e-3, 0.0), "scale3": (3.0, 0.0), "scale30": (30.0, 0.0), "scale300": (300.0, 0.0),
           "offset1e2": (3.0, 1e2), "offset1e3": (3.0, 1e3), "offset1e4": (3.0, 1e4)}
REGIME_SHAPES = [("mec", 2 * WARPS, 2 * LANES + 1), ("mec", THREADS + 1, 1000), ("head", 64, 2 * LANES + 1),
                 ("head", THREADS // 2 + 1, 345)]


@gpu
@pytest.mark.parametrize("kind,rows,k", REGIME_SHAPES, ids=[f"{a}-{b}x{c}" for a, b, c in REGIME_SHAPES])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_value_regimes(regime, kind, rows, k, dev, worst):
    """Nearly uniform rows (ties come near), ordinary and saturated softmax, and a large common offset per row: the
    log-softmax must keep its absolute precision at |logit| ~ 1e4."""
    scale, offset = REGIMES[regime]
    gen = torch.Generator(device=dev).manual_seed(rows + k + int(scale))
    label = f"{regime} {kind} {rows}x{k}"
    if kind == "mec":
        check_mec(dev, worst, regime, _logits(gen, (rows, k), dev, scale, offset),
                  _logits(gen, (rows, k), dev, scale, offset), label)
    else:
        check_head(dev, worst, regime, _logits(gen, (3 * rows, k), dev, scale, offset), _labels(gen, rows, k, dev),
                   label)


# --------------------------------------------------------------------------- 3. exact ties
TIES = [  # K, the tied classes (duplicated columns, the row minimum), as lanes see them
    (65, (5, 6)),           # adjacent lanes
    (65, (3, 35)),          # one lane, two iterations
    (65, (31, 32)),         # across the lane wrap
    (65, (3, 33)),          # the later index in a lower lane
    (65, (3, 34)),
    (65, (3, 33, 34)),      # three-way
    (65, (0, 31, 32)),
    (345, (2, 33, 64, 300)),
    (10, (2, 7)),           # fewer classes than lanes
    (10, (0, 9)),
    (1, (0,)),
]


def _tied(gen, shape, dev, tie):
    """Logits whose classes `tie` hold the same (largest) column in x and y: s ties exactly at the row minimum."""
    z = _logits(gen, shape, dev)
    top = z.amax(dim=1) + 2.0
    for c in tie:
        z[:, c] = top
    return z


@gpu
@pytest.mark.parametrize("k,tie", TIES, ids=[f"K{k}-" + "_".join(map(str, t)) for k, t in TIES])
def test_exact_ties(k, tie, dev, worst):
    """Exact ties take the first class, as torch.min and the oracle do: the MEC call at several rows per warp and the
    head loss's MEC rows."""
    gen = torch.Generator(device=dev).manual_seed(k + sum(tie))
    n = 3 * WARPS + 5
    check_mec(dev, worst, "ties", _tied(gen, (n, k), dev, tie), _tied(gen, (n, k), dev, tie), f"ties mec {k} {tie}",
              exact_k=True)
    b = B_CAP + 3
    logits = torch.cat([_logits(gen, (b, k), dev), _tied(gen, (b, k), dev, tie), _tied(gen, (b, k), dev, tie)])
    check_head(dev, worst, "ties", logits, _labels(gen, b, k, dev), f"ties head {k} {tie}", exact_k=True)


# --------------------------------------------------------------------------- 4. non-finite logits
NONFINITE = ["nan_x", "nan_y", "nan_x_and_y", "posinf_x", "neginf_masked", "neginf_all_but_one"]


def _poison(x, y, case):
    """Non-finite values in a few rows of x / y (in place)."""
    nan, inf = float("nan"), float("inf")
    if case in ("nan_x", "nan_x_and_y"):
        x[1, 17 % x.shape[1]] = nan
    if case in ("nan_y", "nan_x_and_y"):
        y[x.shape[0] - 1, x.shape[1] - 1] = nan
    if case == "nan_x_and_y":
        x[3, 0] = nan
        y[3, 0] = nan
    if case == "posinf_x":
        x[2, x.shape[1] // 2] = inf
    if case == "neginf_masked":      # some classes masked out in x, others in y, one class in both
        x[:, 1::3] = -inf
        y[:, 2::3] = -inf
        y[:, 1] = -inf
    if case == "neginf_all_but_one":
        x[0, 1:] = -inf
        y[4, :-1] = -inf


@gpu
@pytest.mark.parametrize("case", NONFINITE)
@pytest.mark.parametrize("n,k", [(2 * WARPS, 2 * LANES + 1), (THREADS + 1, LANES - 1)], ids=["N64-K65", "N1025-K31"])
def test_non_finite_mec(case, n, k, dev, worst):
    """A NaN (or +inf) logit makes the loss NaN and its row's gradient NaN; the other input's row is
    (softmax - onehot(0)) / 2N, 0 being the first NaN class of that row's s; every other row is unaffected.
    -inf classes give a finite loss: the reference's NaN there is an artefact of 0 * (-inf) in its eye broadcast, not
    part of the loss's definition, and the oracle gives the finite value."""
    gen = torch.Generator(device=dev).manual_seed(n + k)
    x, y = _logits(gen, (n, k), dev), _logits(gen, (n, k), dev)
    _poison(x, y, case)
    loss, gx, gy = check_mec(dev, worst, "non_finite", x, y, f"{case} mec {n}x{k}")
    nan_rows = (x.isnan() | y.isnan() | x.isposinf() | y.isposinf()).any(dim=1)
    assert math.isnan(loss.item()) == bool(nan_rows.any()), (case, loss.item())
    for r in nan_rows.nonzero()[:, 0].tolist():
        other = gy[r] if (x[r].isnan() | x[r].isposinf()).any() else gx[r]
        if other.isfinite().all():          # the one-hot of the first NaN class reaches the other input's row
            assert other[0] < 0 and (other[1:] >= 0).all(), (case, r, other[:4].tolist())


@gpu
@pytest.mark.parametrize("case", ["nan_source", "nan_target", "nan_aug", "posinf_source", "neginf_masked"])
def test_non_finite_head_loss(case, dev, worst):
    """The same rules inside the head loss: a NaN source row makes the classification term NaN (F.nll_loss) and leaves
    lambda * MEC finite; a NaN target or augmented row does the opposite."""
    gen = torch.Generator(device=dev).manual_seed(len(case))
    b, k = B_CAP + 1, 2 * LANES + 1
    logits = _logits(gen, (3 * b, k), dev)
    labels = _labels(gen, b, k, dev, "valid")
    if case == "nan_source":
        logits[2, 5] = float("nan")
    elif case == "nan_target":
        logits[b + 4, 40] = float("nan")
    elif case == "nan_aug":
        logits[3 * b - 1, 0] = float("nan")
    elif case == "posinf_source":
        logits[0, 9] = float("inf")
    else:
        masked = torch.ones(k, dtype=torch.bool, device=dev)
        masked[::4] = False
        logits[:, masked] = float("-inf")
        labels = torch.randint(0, k // 4, (b,), device=dev, generator=gen) * 4     # labels on unmasked classes
    total, parts, _ = check_head(dev, worst, "non_finite", logits, labels, f"{case} head")
    want_nan = {"nan_source": (1, 0), "posinf_source": (1, 0), "nan_target": (0, 1), "nan_aug": (0, 1),
                "neginf_masked": (0, 0)}[case]
    assert (math.isnan(parts[1].item()), math.isnan(parts[2].item())) == tuple(map(bool, want_nan)), (case, parts)


# --------------------------------------------------------------------------- 5. dtypes, layouts, autograd
BF16_MEC = [(1, 1), (WARPS + 1, LANES + 1), (THREADS + 1, 10), (4096, 2 * LANES + 1)]
BF16_HEAD = [(1, 2 * LANES + 1), (B_CAP, LANES), (THREADS // 2 + 1, 2), (4096, 2 * LANES + 1)]


@gpu
def test_bf16_logits_equal_the_float32_call(dev):
    """bf16 logits (what a Linear head hands over under autocast) across the shape edges: the loss is the float32 call
    on the upcast values bit for bit, the gradient the float32 gradient rounded to bf16."""
    bf = torch.bfloat16
    gen = torch.Generator(device=dev).manual_seed(11)
    for n, k in BF16_MEC:
        x, y = _logits(gen, (n, k), dev).to(bf), _logits(gen, (n, k), dev).to(bf)
        la, gxa, gya, _, _ = _mec_call(x, y, dev)
        lb, gxb, gyb, _, _ = _mec_call(x.float(), y.float(), dev)
        assert torch.equal(la, lb) and gxa.dtype == bf, (n, k)
        assert torch.equal(gxa, gxb.to(bf)) and torch.equal(gya, gyb.to(bf)), (n, k)
    for b, k in BF16_HEAD:
        logits, labels = _logits(gen, (3 * b, k), dev).to(bf), _labels(gen, b, k, dev)
        ta, pa, ga, _, _ = _head_call(logits, labels, dev)
        tb, pb, gb, _, _ = _head_call(logits.float(), labels, dev)
        assert torch.equal(ta, tb) and torch.equal(pa, pb), (b, k)
        assert ga.dtype == bf and torch.equal(ga, gb.to(bf)), (b, k)


@gpu
def test_autocast_linear_head(dev):
    """A Linear head under torch.autocast: its bf16 logits reach both losses, which equal the float32 calls on them."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(12)
    b, k = 64, 65
    fc = torch.nn.Linear(256, k).to(dev)
    feats = torch.randn(3 * b, 256, device=dev, generator=gen)
    labels = _labels(gen, b, k, dev)
    head = dwt_b200.HeadLoss(k, LAM)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits = fc(feats)
        logits.retain_grad()
        total = head(logits, labels)
        mec = dwt_b200.MinEntropyConsensusLoss(k, dev)(logits[b:2 * b], logits[2 * b:])
    assert logits.dtype == torch.bfloat16 and total.dtype == torch.float32
    (total * UPSTREAM).backward()
    t32, p32, g32, _, _ = _head_call(logits.detach().float(), labels, dev)
    assert torch.equal(total.detach(), t32) and torch.equal(head.parts, p32)
    assert torch.equal(logits.grad, g32.to(torch.bfloat16))
    m32, _, _, _, _ = _mec_call(logits.detach()[b:2 * b].float(), logits.detach()[2 * b:].float(), dev)
    assert torch.equal(mec.detach(), m32)


@gpu
def test_non_contiguous_inputs(dev, worst):
    """A transposed [K, N] view, a column slice and the target slices of a [3B, K] batch: bit for bit the contiguous
    call, and within the fp64 bounds."""
    gen = torch.Generator(device=dev).manual_seed(13)
    n, k = THREADS + 1, LANES + 1
    xt, yt = _logits(gen, (k, n), dev).t(), _logits(gen, (k, n), dev).t()
    wide = _logits(gen, (n, k + 9), dev)
    xs, ys = wide[:, 4:4 + k], _logits(gen, (n, k + 3), dev)[:, :k]
    batch = _logits(gen, (3 * n, k), dev)
    cases = {"transposed": (xt, yt), "column_slice": (xs, ys), "target_slices": (batch[n:2 * n], batch[2 * n:]),
             "mixed": (xt, batch[2 * n:])}
    for name, (x, y) in cases.items():
        assert name == "target_slices" or not (x.is_contiguous() and y.is_contiguous())
        got = check_mec(dev, worst, "layouts", x, y, f"layout {name}")
        want = _mec_call(x.contiguous(), y.contiguous(), dev)[:3]
        assert all(torch.equal(a, c) for a, c in zip(got, want)), name
    b = B_CAP + 1
    logits_t = _logits(gen, (k, 3 * b), dev).t()
    labels = _labels(gen, b, k, dev)
    labels_s = torch.stack([labels, labels], dim=1)[:, 0]                 # a strided label view
    assert not logits_t.is_contiguous() and not labels_s.is_contiguous()
    got = check_head(dev, worst, "layouts", logits_t, labels_s, "layout head transposed")
    want = _head_call(logits_t.contiguous(), labels, dev)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]) and torch.equal(got[2], want[2])


@gpu
def test_one_input_requires_grad_and_accumulation(dev):
    """Only x (or only y) requires grad: its gradient is the two-input call's.  The loss used twice (two backward
    passes through one call, and a second call) accumulates the same gradient each time."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(14)
    n, k = 2 * WARPS + 3, 2 * LANES + 1
    x, y = _logits(gen, (n, k), dev), _logits(gen, (n, k), dev)
    _, gx, gy, _, _ = _mec_call(x, y, dev)
    mec = dwt_b200.MinEntropyConsensusLoss(k, dev)
    g = _upstream(dev)
    for which in (0, 1):
        leaf = (x if which == 0 else y).detach().requires_grad_(True)
        other = (y if which == 0 else x).detach()
        loss = mec(leaf, other) if which == 0 else mec(other, leaf)
        loss.backward(g)
        assert torch.equal(leaf.grad, gx if which == 0 else gy)
    xl = x.detach().requires_grad_(True)
    loss = mec(xl, y)
    loss.backward(g, retain_graph=True)
    loss.backward(g)
    mec(xl, y).backward(g)
    assert torch.equal(xl.grad, gx + gx + gx)
    b = B_CAP
    logits, labels = _logits(gen, (3 * b, k), dev), _labels(gen, b, k, dev)
    _, _, grad, _, _ = _head_call(logits, labels, dev)
    ll = logits.detach().requires_grad_(True)
    head = dwt_b200.HeadLoss(k, LAM)
    total = head(ll, labels)
    (total * 2).backward(g / 2)            # upstream 1.7 reaching the loss, as a product
    head(ll, labels).backward(g)
    assert torch.equal(ll.grad, grad + grad)
    with torch.no_grad():
        assert torch.equal(head(logits, labels), total.detach())


# --------------------------------------------------------------------------- 6. consistency and replay
@gpu
@pytest.mark.parametrize("b,k", [(1, 65), (B_CAP + 1, 33), (THREADS // 2 + 1, 345), (4096, 65)])
def test_head_mec_part_equals_mec_loss(b, k, dev):
    """HeadLoss.parts[2] is lambda * MinEntropyConsensusLoss on the same target slices, and its MEC gradient rows are
    lambda times the MEC call's, to rounding."""
    gen = torch.Generator(device=dev).manual_seed(b * k)
    logits, labels = _logits(gen, (3 * b, k), dev), _labels(gen, b, k, dev)
    _, parts, grad, _, _ = _head_call(logits, labels, dev, lam=0.3)
    loss, gx, gy, _, _ = _mec_call(logits[b:2 * b], logits[2 * b:], dev)
    lamf = float(torch.tensor(0.3))
    assert abs(parts[2].item() - lamf * loss.item()) <= 1e-6 * abs(lamf * loss.item()), (parts[2].item(), loss.item())
    want = lamf * torch.cat([gx, gy]).double()
    assert ((grad[b:].double() - want).norm() / want.norm()).item() <= 1e-6


@gpu
def test_runs_are_bit_identical(dev):
    gen = torch.Generator(device=dev).manual_seed(15)
    x, y = _logits(gen, (65536, 65), dev), _logits(gen, (65536, 65), dev)
    a, b = _mec_call(x, y, dev)[:3], _mec_call(x, y, dev)[:3]
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    logits, labels = _logits(gen, (3 * 4096, 65), dev), _labels(gen, 4096, 65, dev)
    a, b = _head_call(logits, labels, dev)[:3], _head_call(logits, labels, dev)[:3]
    assert all(torch.equal(p, q) for p, q in zip(a, b))


@gpu
def test_graph_replay_equals_eager(dev):
    """Both losses and their gradients captured in a CUDA graph and replayed twice: bit for bit the eager calls."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(16)
    b, k = 64, 65
    logits, labels = _logits(gen, (3 * b, k), dev), _labels(gen, b, k, dev)
    x, y = _logits(gen, (THREADS + 1, 33), dev), _logits(gen, (THREADS + 1, 33), dev)
    g = _upstream(dev)
    head, mec = dwt_b200.HeadLoss(k, LAM), dwt_b200.MinEntropyConsensusLoss(33, dev)

    def step():
        ll, xl, yl = (t.detach().requires_grad_(True) for t in (logits, x, y))
        total = head(ll, labels)
        loss = mec(xl, yl)
        return (total, head.parts, loss) + torch.autograd.grad(total, ll, g) + torch.autograd.grad(loss, (xl, yl), g)
    eager = [t.detach().clone() for t in step()]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize(dev)
        assert all(torch.equal(p, q) for p, q in zip(got, eager))


@gpu
def test_label_refusals(dev):
    """Labels must be an int64 CUDA tensor; logits must be float32 or bfloat16."""
    import dwt_b200
    from dwt_b200 import _native
    head = dwt_b200.HeadLoss(5, 0.1)
    logits = torch.zeros(6, 5, device=dev)
    for labels in (torch.zeros(2, dtype=torch.int32, device=dev), torch.zeros(2, dtype=torch.int64)):
        with pytest.raises(_native.NativeError, match="labels must be an int64 CUDA tensor"):
            head(logits, labels)
    with pytest.raises(_native.NativeError, match="float32"):
        head(logits.half(), torch.zeros(2, dtype=torch.int64, device=dev))
