"""Whitening in the exact ZCA basis (ExactZCAWTransform2d, dwt_whiten_eigh_*).

CPU: the float64 closed-form backward of S^-1/2 (tests/support/eigh_reference.py) against autograd through
torch.linalg.eigh and against central finite differences where eigenvalues repeat; the module surface; the refusals of
the C ABI (argument checks run before any device call, so fake pointers do).

GPU: the tensor-core kernels against the float64 reference -- outputs and input gradients within 1e-3 norm-wise (max
element within 5x that), statistics and running buffers within 1e-4, as in test_zca_whitening.py -- and against
themselves (layouts, dtypes, reruns, graphs, the fused site), at condition numbers where the Newton-Schulz basis
cannot whiten.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import eigh_reference as E  # noqa: E402
import zca_reference as Z  # noqa: E402

BOUND, STAT_BOUND = 1e-3, 1e-4
gpu = pytest.mark.gpu


# =========================================================================== CPU: the float64 reference
@pytest.mark.parametrize("gs", [8, 16, 32, 64])
@pytest.mark.parametrize("cond", [3.0, 100.0])
def test_closed_form_backward_matches_autograd_eigh(gs, cond):
    """Well-separated spectra (log-spaced from 1 to 1/cond): the Daleckii-Krein backward equals autograd through eigh."""
    rng = np.random.default_rng(gs + int(cond))
    x = Z.conditioned_input(rng, 8, 2 * gs, (4, 5), gs, cond, shift=0.5)
    dy = torch.tensor(rng.standard_normal(x.shape))
    out = []
    for via in (False, True):
        xt = torch.tensor(x, requires_grad=True)
        y, *_ = E.exact_torch(xt, gs, autograd_eigh=via)
        (dx,) = torch.autograd.grad(y, xt, dy)
        out.append((y.detach(), dx))
    (y0, dx0), (y1, dx1) = out
    assert torch.allclose(y0, y1, rtol=1e-14, atol=0)
    assert (dx0 - dx1).abs().max() <= 1e-10 * dx1.abs().max()


@pytest.mark.parametrize("gs", [8, 64])
def test_closed_form_backward_at_repeated_eigenvalues(gs):
    """S = I (condition number 1: every eigenvalue repeated), where eigh's own backward divides by zero: the closed
    form stays finite and matches central finite differences of <dy, y(x)>."""
    rng = np.random.default_rng(gs)
    x = torch.tensor(Z.conditioned_input(rng, 8, gs, (4, 5), gs, 1.0, shift=0.5))
    dy = torch.tensor(rng.standard_normal(tuple(x.shape)))
    xt = x.clone().requires_grad_(True)
    y, _, cov, _ = E.exact_torch(xt, gs, eps=0.0)
    assert torch.allclose(cov, torch.eye(gs, dtype=cov.dtype), atol=1e-12)
    (dx,) = torch.autograd.grad(y, xt, dy)
    assert torch.isfinite(dx).all()
    h = 1e-6
    for k in range(3):
        v = torch.tensor(rng.standard_normal(tuple(x.shape)))
        lp = (dy * E.exact_torch(x + h * v, gs, eps=0.0)[0]).sum()
        lm = (dy * E.exact_torch(x - h * v, gs, eps=0.0)[0]).sum()
        fd, an = float((lp - lm) / (2 * h)), float((dx * v).sum())
        assert abs(fd - an) <= 1e-6 * max(abs(an), 1.0), (k, fd, an)


def test_reference_output_is_white():
    rng = np.random.default_rng(1)
    x = torch.tensor(Z.conditioned_input(rng, 16, 64, (8, 8), 64, 1e3, shift=2.0))
    y, *_ = E.exact_torch(x, 64, eps=0.0)
    yg = y.transpose(0, 1).reshape(64, -1)
    assert torch.allclose(yg @ yg.T / yg.shape[-1], torch.eye(64, dtype=y.dtype), atol=1e-9)


# =========================================================================== CPU: module surface
def test_module_surface_and_state_dicts():
    import inspect
    import dwt_b200
    assert "ExactZCAWTransform2d" in dwt_b200.__all__
    assert inspect.signature(dwt_b200.ExactZCAWTransform2d.__init__) == inspect.signature(dwt_b200.WTransform2d.__init__)
    e, w, z = dwt_b200.ExactZCAWTransform2d(64, 16), dwt_b200.WTransform2d(64, 16), dwt_b200.ZCAWTransform2d(64, 16)
    assert set(e.state_dict()) == set(w.state_dict()) == {"running_mean", "running_variance"}
    assert all(e.state_dict()[k].shape == w.state_dict()[k].shape for k in w.state_dict())
    with torch.no_grad():
        w.running_mean.normal_()
        w.running_variance.normal_()
    e.load_state_dict(w.state_dict())
    z.load_state_dict(e.state_dict())
    assert torch.equal(z.running_variance, w.running_variance) and torch.equal(e.running_mean, w.running_mean)
    assert (e.group_size, e.num_groups, e.eps, e.momentum, e.alpha) == (16, 4, 1e-3, 0.1, 1)
    assert dwt_b200.ExactZCAWTransform2d(8, 16).group_size == 8
    rm, rv = torch.zeros(1, 64, 1, 1), torch.ones(4, 16, 16)
    b = dwt_b200.ExactZCAWTransform2d(64, 16, running_m=rm, running_var=rv)
    assert b.running_mean.data_ptr() == rm.data_ptr() and b.running_variance.data_ptr() == rv.data_ptr()


def test_cpu_tensors_and_bad_inputs_are_refused():
    import dwt_b200
    m = dwt_b200.ExactZCAWTransform2d(64, 16)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(torch.zeros(2, 64, 8, 8))
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(2, 64, 8))
    with pytest.raises(ValueError, match="expected number of channels divisible by group_size"):
        dwt_b200.ExactZCAWTransform2d(48, 32)(torch.zeros(2, 48, 3, 3))


def test_domain_site_refuses_mixed_bases():
    import dwt_b200
    site = dwt_b200.DomainTripleNorm("whiten", 64, 16)
    for other in (dwt_b200.ZCAWTransform2d(64, 16), dwt_b200.WTransform2d(64, 16)):
        mods = [dwt_b200.ExactZCAWTransform2d(64, 16), dwt_b200.ExactZCAWTransform2d(64, 16), other]
        with pytest.raises(ValueError, match="share one basis"):
            site(torch.zeros(6, 64, 8, 8), mods, None, None)
        with pytest.raises(ValueError, match="share one basis"):
            site(torch.zeros(2, 64, 8, 8), mods, None, None, replicated=True)
    for gs in (1, 2, 4):
        with pytest.raises(dwt_b200._native.NativeError, match="tensor-core"):
            dwt_b200.DomainTripleNorm("whiten", 64, gs)(torch.zeros(6, 64, 8, 8), [dwt_b200.ExactZCAWTransform2d(64, gs)] * 3,
                                                        None, None)


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _eigh_fwd(lib, N=8, C=128, HW=3136, gs=64, D=1, mode=0, save_e=_FAKE):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_eigh_fwd(p, p, N, C, HW, gs, D, mode, 1e-3, 0.1, 0, None, None, p, p,
                                   None if save_e is None else ctypes.c_void_p(save_e), p, 1 << 40, None)


def _eigh_bwd(lib, N=8, C=128, HW=3136, gs=64, D=1, mode=0, save_e=_FAKE):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_eigh_bwd(p, p, p, N, C, HW, gs, D, mode, 1e-3, p, p,
                                   None if save_e is None else ctypes.c_void_p(save_e), p, 1 << 40, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


_EXACT = b"exact ZCA basis"


@pytest.mark.parametrize("call", [_eigh_fwd, _eigh_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(gs=1), -4, _EXACT), (dict(gs=2), -4, _EXACT), (dict(gs=4), -4, _EXACT),
    (dict(gs=128), -4, _EXACT), (dict(C=128, gs=256), -4, b"group_size"),
    (dict(HW=16, N=512), -4, _EXACT),                                       # HW < 32: the tiled family
    (dict(HW=36, N=64), -4, _EXACT),                                        # N*HW < 4096 per domain
    (dict(HW=34, N=512), -4, _EXACT),                                       # HW % 4 != 0
    (dict(HW=36, N=512, mode=0x200), -4, b"HW >= 32 and a multiple of 8"),   # NCHW bf16: HW % 8 != 0
    (dict(C=64, gs=4, mode=0x100), -4, _EXACT),                             # channels-last group size 4
    (dict(save_e=None), -1, b"null pointer argument (save_e)"),
    (dict(save_e=_FAKE + 4), -1, b"save_e must be 16-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


def test_c_abi_keeps_the_newton_schulz_texts(lib):
    p = ctypes.c_void_p(_FAKE)
    assert lib.dwt_whiten_zca_fwd(p, p, 8, 128, 3136, 4, 1, 0, 1e-3, 0.1, 0, None, None, 5, p, p, p, p, 1 << 40, None) == -4
    err = lib.dwt_last_error()
    assert err.startswith(b"the ZCA basis is built for the tensor-core kernels only") and _EXACT not in err


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nexact ZCA basis, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-34s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b, bound=BOUND):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= bound and m <= 5 * bound, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def iid(shape, dev, seed=0, shift=1.5):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, device=dev, generator=g) + shift


def mixed(shape, dev, seed=0, shift=2.0):
    """bench.py's microbench input: x = mix . randn + 2, mix = randn / sqrt(C) + I over all channels."""
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    mix = torch.randn(c, c, device=dev, generator=g) / c ** 0.5 + torch.eye(c, device=dev)
    return (torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, h, w, device=dev, generator=g)) + shift).contiguous()


def conditioned(dev, n, c, hw, gs, cond, seed=0, shift=1.0):
    return torch.tensor(Z.conditioned_input(np.random.default_rng(seed), n, c, hw, gs, cond, shift=shift),
                        dtype=torch.float32, device=dev)


def families(prof):
    return {k.split("|")[0] for k in prof}


def run_case(dev, worst, label, x, gs, d=1, mode="train", layout="shared", via="module", check_profile=False):
    """x [d*N, C, H, W] through d ExactZCAWTransform2d modules (via='module': d sequential calls) or one DomainTripleNorm
    site (via='site'), forward + backward, against float64 per domain; running buffers through the ordered EMA."""
    import dwt_b200
    from dwt_b200 import _native as nv
    c = x.shape[1]
    n = x.shape[0] // d
    gen = torch.Generator(device=dev).manual_seed(1)
    dy = torch.randn(x.shape, device=dev, generator=gen)
    sfx = "_nhwc" if x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous() else ""
    default = mode == "default"
    pairs = []
    for k in range({"shared": 1, "distinct": d, "mixed": 2}[layout]):
        rm = torch.randn(1, c, 1, 1, device=dev, generator=gen) * 0.1
        a = torch.randn(c // gs, gs, 2 * gs, device=dev, generator=gen)
        rc = 0.25 * torch.bmm(a, a.transpose(1, 2)) / (2 * gs) + torch.eye(gs, device=dev)
        pairs.append((rm, rc))
    which = {"shared": [0] * d, "distinct": list(range(d)), "mixed": [0, 1, 0, 1][:d]}[layout]
    mods = []
    for k in range(d):
        rm, rc = pairs[which[k]]
        m = (dwt_b200.ExactZCAWTransform2d(c, gs) if default else
             dwt_b200.ExactZCAWTransform2d(c, gs, running_m=rm, running_var=rc)).to(dev)
        mods.append(m.train(mode in ("train", "nograd", "default")))
    before = [(m.running_mean.clone(), m.running_variance.clone()) for m in mods]
    xg = x.clone().requires_grad_(mode != "nograd")
    nv.profile_begin()
    with torch.set_grad_enabled(mode != "nograd"):
        if via == "site":
            y = dwt_b200.DomainTripleNorm("whiten", c, gs, n_domains=d)(xg, mods, None, None)
        else:
            y = torch.cat([mods[k](xg[k * n:(k + 1) * n]) for k in range(d)])
        dx = torch.autograd.grad(y, xg, dy)[0] if mode != "nograd" else None
    prof = nv.profile_end()
    if check_profile:
        fam = families(prof)
        want = {"dense_fwd_eigh", "tc_apply" + sfx}
        if dx is not None:
            want |= {"dense_bwd_eigh", "tc_bwd_apply" + sfx}
        if mode != "eval":
            want.add("tc_stats" + sfx)
        assert want <= fam, fam
        assert not any(f.startswith(("dense_fwd_finalize", "dense_bwd_finalize", "dense_fwd_zca", "dense_bwd_zca", "tiled", "small"))
                       for f in fam), fam
    train = mode != "eval"
    ref_buf = {}
    for k in range(d):
        key = which[k] if not default else k
        rm0, rc0 = ref_buf.get(key, tuple(t.double() for t in before[k]))
        xd = x[k * n:(k + 1) * n].double().requires_grad_(True)
        yr, mean, cov, _ = E.exact_torch(xd, gs, eps=1e-3, running_mean=rm0, running_cov=rc0, train=train)
        tag = f"{label} d{k}"
        check(worst, tag, "y", y[k * n:(k + 1) * n].detach(), yr.detach())
        if dx is not None:
            (dxr,) = torch.autograd.grad(yr, xd, dy[k * n:(k + 1) * n].double())
            check(worst, tag, "dx", dx[k * n:(k + 1) * n], dxr)
        if train:
            m = 0.1
            ref_buf[key] = ((1 - m) * rm0 + m * mean.detach().reshape(rm0.shape),
                            (1 - m) * rc0 + m * cov.detach().reshape(rc0.shape))
    for k in range(d):
        if train:
            key = which[k] if not default else k
            check(worst, f"{label} d{k}", "running_mean", mods[k].running_mean, ref_buf[key][0], STAT_BOUND)
            check(worst, f"{label} d{k}", "running_var", mods[k].running_variance, ref_buf[key][1], STAT_BOUND)
        else:
            assert torch.equal(mods[k].running_mean, before[k][0]) and torch.equal(mods[k].running_variance, before[k][1])
    return y


@gpu
def test_config2_full_size(dev, worst):
    """N=256 C=256 56^2 at group size 64, the microbench input, default-constructed buffers; the profile shows the
    eigh families beside unchanged tc_* ones."""
    run_case(dev, worst, "config2 gs64", mixed((256, 256, 56, 56), dev), 64, mode="default", check_profile=True)


EDGES = [
    # label, (N, C, H, W), gs, domains, mode, buffer layout, via, channels-last
    ("gs8 c64 hw32", (128, 64, 4, 8), 8, 1, "train", "shared", "module", False),
    ("gs16 c96 partial-sb", (16, 96, 16, 16), 16, 1, "train", "shared", "module", False),
    ("gs32 c96 partial-sb nhwc", (16, 96, 16, 16), 32, 1, "train", "shared", "module", True),
    ("gs64 c512", (8, 512, 24, 24), 64, 1, "train", "shared", "module", False),
    ("gs64 hw36 d2 distinct", (2 * 114, 128, 6, 6), 64, 2, "train", "distinct", "site", False),
    ("gs32 hw40 d3 mixed nhwc", (3 * 103, 64, 5, 8), 32, 3, "train", "mixed", "site", True),
    ("gs16 hw3136 d4 shared", (4 * 2, 64, 56, 56), 16, 4, "train", "shared", "site", False),
    ("gs8 hw3136 d4 distinct nhwc", (4 * 2, 64, 56, 56), 8, 4, "train", "distinct", "site", True),
    ("gs64 m4096 nograd", (128, 128, 4, 8), 64, 1, "nograd", "shared", "module", False),
    ("gs64 m4096 d1", (128, 64, 4, 8), 64, 1, "train", "shared", "module", False),
    ("gs64 eval", (16, 128, 16, 16), 64, 1, "eval", "shared", "module", False),
    ("gs8 eval d3 site nhwc", (3 * 16, 64, 16, 16), 8, 3, "eval", "distinct", "site", True),
    ("gs32 default d3 site", (3 * 16, 128, 16, 16), 32, 3, "default", "shared", "site", False),
]


@gpu
@pytest.mark.parametrize("case", EDGES, ids=[e[0] for e in EDGES])
def test_edges(case, dev, worst):
    label, shape, gs, d, mode, layout, via, cl = case
    x = iid(shape, dev, seed=len(label))
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    run_case(dev, worst, label, x, gs, d, mode, layout, via, check_profile=True)


@gpu
@pytest.mark.parametrize("gs", [8, 64])
@pytest.mark.parametrize("cond", [1.0, 10.0, 100.0, 1e3])
def test_conditioning(gs, cond, dev, worst):
    """Every group's batch covariance has condition number `cond` exactly: the Newton-Schulz basis whitens these only
    partly (T <= 5) or not at all (T = 16); the exact basis matches float64."""
    run_case(dev, worst, f"cond{cond:g} gs{gs}", conditioned(dev, 64, 128, (8, 8), gs, cond, seed=gs), gs)


@gpu
@pytest.mark.parametrize("gs", [16, 64])
@pytest.mark.parametrize("cond", [1.0, 100.0, 1e3])
def test_output_is_white_with_tiny_eps(gs, cond, dev):
    import dwt_b200
    x = conditioned(dev, 64, 128, (8, 8), gs, cond, seed=5, shift=3.0)
    y = dwt_b200.ExactZCAWTransform2d(128, gs, eps=1e-7).to(dev)(x).double()
    yg = y.transpose(0, 1).reshape(128 // gs, gs, -1)
    cov = yg @ yg.transpose(1, 2) / yg.shape[-1]
    err = float((cov - torch.eye(gs, dtype=cov.dtype, device=dev)).abs().max())
    assert err < 2e-3, err


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_statistics_equal_cholesky(layout, dev):
    """Running buffers and save_mean bit for bit those of WTransform2d (the shared prologue and EMA); W is symmetric."""
    import dwt_b200
    from dwt_b200 import functional as F
    x = mixed((32, 128, 16, 16), dev)
    if layout == "nhwc":
        x = x.contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    em, wm = dwt_b200.ExactZCAWTransform2d(128, 32).to(dev), dwt_b200.WTransform2d(128, 32).to(dev)
    ye, yw = em(x), wm(x)
    assert torch.equal(em.running_mean, wm.running_mean) and torch.equal(em.running_variance, wm.running_variance)
    assert torch.equal(ye.grad_fn.saved_tensors[1], yw.grad_fn.saved_tensors[1])          # save_mean
    w = ye.grad_fn.saved_tensors[2]
    assert torch.equal(w, w.transpose(-1, -2))
    bufs = [(torch.zeros(1, 128, 1, 1, device=dev), torch.eye(32, device=dev).repeat(4, 1, 1)) for _ in range(2)]
    for it, (rm, rc) in zip(("eigh", 0), bufs):
        F.norm(x.detach().repeat(3, 1, 1, 1), None, None, kind="whiten", group_size=32, n_domains=3, training_stats=True,
               eps=1e-3, momentum=0.1, update_running=True, running=[(rm, rc)] * 3, iterations=it)
    assert torch.equal(bufs[0][0], bufs[1][0]) and torch.equal(bufs[0][1], bufs[1][1])


def _fwd_bwd(m, x, dy):
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    (dx,) = torch.autograd.grad(y, xg, dy)
    return y.detach(), dx


@gpu
@pytest.mark.parametrize("gs", [16, 64])
def test_channels_last_equals_nchw(gs, dev):
    import dwt_b200
    x, dy = mixed((16, 128, 16, 16), dev), iid((16, 128, 16, 16), dev, seed=5, shift=0.0)
    a, b = dwt_b200.ExactZCAWTransform2d(128, gs).to(dev), dwt_b200.ExactZCAWTransform2d(128, gs).to(dev)
    y0, dx0 = _fwd_bwd(a, x, dy)
    cl = torch.channels_last
    y1, dx1 = _fwd_bwd(b, x.contiguous(memory_format=cl), dy.contiguous(memory_format=cl))
    assert y1.is_contiguous(memory_format=cl) and dx1.is_contiguous(memory_format=cl)
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    assert torch.equal(a.running_variance, b.running_variance)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_bf16_equals_float32_on_widened_input(layout, dev):
    import dwt_b200
    from dwt_b200 import _native as nv
    x, dy = mixed((16, 128, 16, 16), dev).bfloat16(), iid((16, 128, 16, 16), dev, seed=5, shift=0.0).bfloat16()
    if layout == "nhwc":
        x, dy = x.contiguous(memory_format=torch.channels_last), dy.contiguous(memory_format=torch.channels_last)
    a, b = dwt_b200.ExactZCAWTransform2d(128, 32).to(dev), dwt_b200.ExactZCAWTransform2d(128, 32).to(dev)
    nv.profile_begin()
    y16, dx16 = _fwd_bwd(a, x, dy)
    fam = families(nv.profile_end())
    assert {"dense_fwd_eigh_bf16", "dense_bwd_eigh_bf16"} <= fam, fam
    y32, dx32 = _fwd_bwd(b, x.float(), dy.float())
    assert y16.dtype == torch.bfloat16 and torch.equal(y16, y32.bfloat16()) and torch.equal(dx16, dx32.bfloat16())
    assert torch.equal(a.running_variance, b.running_variance)


@gpu
def test_reruns_and_graph_replay_are_bit_identical(dev):
    import dwt_b200
    x, dy = conditioned(dev, 16, 128, (16, 16), 64, 1e3, seed=2), iid((16, 128, 16, 16), dev, seed=5, shift=0.0)
    m = dwt_b200.ExactZCAWTransform2d(128, 64).to(dev)
    outs = []
    for _ in range(2):
        m.running_mean.zero_()
        m.running_variance.fill_(1.0)
        outs.append(_fwd_bwd(m, x, dy) + (m.running_variance.clone(),))
    assert all(torch.equal(p, q) for p, q in zip(*outs))
    m, m_eager = dwt_b200.ExactZCAWTransform2d(128, 64).to(dev), dwt_b200.ExactZCAWTransform2d(128, 64).to(dev)
    leaf = x.clone().requires_grad_(True)

    def step(mod):
        y = mod(leaf)
        (dx,) = torch.autograd.grad(y, leaf, dy)
        return y, dx

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(m)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        step(m_eager)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y_g, dx_g = step(m)
    g.replay()
    torch.cuda.synchronize()
    y_e, dx_e = step(m_eager)
    assert torch.equal(y_g, y_e) and torch.equal(dx_g, dx_e)
    assert torch.equal(m.running_variance, m_eager.running_variance) and torch.equal(m.running_mean, m_eager.running_mean)


@gpu
def test_nan_group_sets_status_and_skips_ema(dev):
    import dwt_b200
    from dwt_b200 import _native as nv
    x = mixed((16, 128, 16, 16), dev)
    x[3, 70] = float("nan")                                                   # group 1 of 2 at group size 64
    m = dwt_b200.ExactZCAWTransform2d(128, 64).to(dev)
    rv0 = m.running_variance.clone()
    nv.clear_status(dev)
    y = m(x)
    torch.cuda.synchronize()
    assert nv.status(dev) & nv.STATUS_NOT_PD
    assert torch.equal(m.running_variance[1], rv0[1]) and not torch.equal(m.running_variance[0], rv0[0])
    assert torch.isfinite(y[:, :64]).all()
    with pytest.raises(dwt_b200.NotPositiveDefiniteError):
        nv.check_status(dev)
    nv.raise_on_status(1)
    try:
        with pytest.raises(dwt_b200.NotPositiveDefiniteError):
            m(x)
    finally:
        nv.raise_on_status(0)
        nv.clear_status(dev)


@gpu
def test_eval_indefinite_running_buffer_sets_status(dev):
    """Eval mode on running buffers: a positive definite group normalises as the float64 reference, an indefinite one
    (an eigenvalue of S below zero) sets the status -- which the Newton-Schulz basis cannot detect."""
    import dwt_b200
    from dwt_b200 import _native as nv
    gs = 32
    x = mixed((16, 64, 16, 16), dev)
    q, _ = torch.linalg.qr(torch.randn(gs, gs, device=dev, dtype=torch.float64))
    good = torch.eye(gs, device=dev) * 2.0
    bad = (q @ torch.diag(torch.linspace(-0.5, 2.0, gs, device=dev, dtype=torch.float64)) @ q.T).float()
    rv = torch.stack([good, bad])
    m = dwt_b200.ExactZCAWTransform2d(64, gs, running_m=torch.zeros(1, 64, 1, 1, device=dev), running_var=rv).to(dev).eval()
    nv.clear_status(dev)
    y = m(x)
    torch.cuda.synchronize()
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    yr, *_ = E.exact_torch(x.double(), gs, running_mean=torch.zeros(64, device=dev, dtype=torch.float64),
                           running_cov=good.double().expand(2, gs, gs), train=False)
    assert rel(y[:, :gs], yr[:, :gs])[0] < BOUND
    m.running_variance[1] = good
    m(x)
    torch.cuda.synchronize()
    assert not nv.status(dev) & nv.STATUS_NOT_PD


@gpu
@pytest.mark.parametrize("layout", ["shared", "distinct"])
def test_domain_site_equals_three_module_calls(layout, dev, worst):
    import dwt_b200
    x = mixed((3 * 16, 128, 16, 16), dev)
    dy = iid(x.shape, dev, seed=9, shift=0.0)
    ra = (torch.zeros(1, 128, 1, 1, device=dev), torch.eye(32, device=dev).repeat(4, 1, 1))
    bufs = {"shared": [ra] * 3, "distinct": [(ra[0].clone(), ra[1].clone()) for _ in range(3)]}[layout]
    clone = {id(b): (b[0].clone(), b[1].clone()) for b in bufs}
    mk = lambda rs: [dwt_b200.ExactZCAWTransform2d(128, 32, running_m=a, running_var=b).to(dev) for a, b in rs]   # noqa: E731
    site_mods, seq_mods = mk(bufs), mk([clone[id(b)] for b in bufs])
    xs = x.clone().requires_grad_(True)
    ys = dwt_b200.DomainTripleNorm("whiten", 128, 32)(xs, site_mods, None, None)
    (dxs,) = torch.autograd.grad(ys, xs, dy)
    xq = x.clone().requires_grad_(True)
    yq = torch.cat([seq_mods[k](xq[16 * k:16 * (k + 1)]) for k in range(3)])
    (dxq,) = torch.autograd.grad(yq, xq, dy)
    check(worst, f"site vs modules {layout}", "y", ys.detach(), yq.detach(), 1e-5)
    check(worst, f"site vs modules {layout}", "dx", dxs, dxq, 1e-5)
    for a, b in zip(site_mods, seq_mods):
        check(worst, f"site vs modules {layout}", "running_var", a.running_variance, b.running_variance, 1e-6)


@gpu
def test_domain_site_replicated_and_fork(dev):
    import dwt_b200
    from dwt_b200 import _native as nv
    x = mixed((16, 128, 16, 16), dev)
    site = dwt_b200.DomainTripleNorm("whiten", 128, 32)
    mods = [dwt_b200.ExactZCAWTransform2d(128, 32).to(dev) for _ in range(3)]
    ref = [dwt_b200.ExactZCAWTransform2d(128, 32).to(dev) for _ in range(3)]
    nv.profile_begin()
    with torch.no_grad():
        site(x, mods, None, None, replicated=True)
    assert "dense_fwd_eigh" in families(nv.profile_end())
    with torch.no_grad():
        for m in ref:
            m(x)
    for a, b in zip(mods, ref):
        assert torch.allclose(a.running_variance, b.running_variance, rtol=1e-5, atol=1e-6)
    xg = mixed((48, 128, 16, 16), dev).requires_grad_(True)
    y = site(xg, mods, None, None)
    a, b = dwt_b200.fork_for_sum(y)
    (g1,) = torch.autograd.grad((a * 2 + b).sum(), xg)
    y = site(xg, mods, None, None)
    (g2,) = torch.autograd.grad((y * 3).sum(), xg)
    assert torch.allclose(g1, g2, rtol=1e-4, atol=1e-5)


@gpu
def test_conv_exact_zca_conv_training_step(dev, worst):
    """conv(64 -> 256, 3x3) -> ExactZCAWTransform2d(256, 64) -> conv(256 -> 32, 1x1): loss and both weight gradients of
    one training step against the same network in float64."""
    import dwt_b200
    torch.manual_seed(0)
    c1 = torch.nn.Conv2d(64, 256, 3, padding=1, bias=False).to(dev)
    c2 = torch.nn.Conv2d(256, 32, 1, bias=False).to(dev)
    norm = dwt_b200.ExactZCAWTransform2d(256, 64).to(dev)
    x = torch.randn(32, 64, 16, 16, device=dev)
    target = torch.randn(32, 32, 16, 16, device=dev)
    loss = ((c2(norm(c1(x))) - target) ** 2).mean()
    g = torch.autograd.grad(loss, [c1.weight, c2.weight])
    w1, w2 = c1.weight.detach().double().requires_grad_(True), c2.weight.detach().double().requires_grad_(True)
    h, *_ = E.exact_torch(torch.nn.functional.conv2d(x.double(), w1, padding=1), 64)
    loss_r = ((torch.nn.functional.conv2d(h, w2) - target.double()) ** 2).mean()
    gr = torch.autograd.grad(loss_r, [w1, w2])
    check(worst, "conv-exact-conv", "loss", loss.detach().reshape(1), loss_r.detach().reshape(1))
    check(worst, "conv-exact-conv", "dconv1", g[0], gr[0])
    check(worst, "conv-exact-conv", "dconv2", g[1], gr[1])
