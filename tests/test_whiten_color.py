"""Whitening followed by a learnable colouring (WCTransform2d, dwt_whiten_color_*, DomainTripleNorm with a matrix gamma).

CPU: the float64 closed-form backward (tests/support/wc_reference.py) against autograd through torch.linalg.cholesky /
inverse and against central finite differences for dcolor and dbias; the module surface; the refusals of the C ABI
(argument checks run before any device call, so fake pointers do).

GPU: the tensor-core kernels against the float64 reference -- y, dx, dcolor and dbias within 1e-3 norm-wise (max element
within 5x that), statistics and running buffers within 1e-4, as in test_zca_exact.py -- and against themselves and
WTransform2d bit for bit (identity colouring, layouts, dtypes, reruns, graphs).
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import wc_reference as R  # noqa: E402

BOUND, STAT_BOUND = 1e-3, 1e-4
gpu = pytest.mark.gpu


def _cpu_case(gs, seed, n=6, c=None, hw=(3, 4)):
    c = c or 2 * gs
    g = torch.Generator().manual_seed(seed)
    mix = torch.eye(c, dtype=torch.float64) + 0.3 * torch.randn(c, c, generator=g, dtype=torch.float64) / c ** 0.5
    x = torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, *hw, generator=g, dtype=torch.float64)) + 0.5
    color = torch.eye(gs, dtype=torch.float64) + 0.3 * torch.randn(c // gs, gs, gs, generator=g, dtype=torch.float64) / gs ** 0.5
    bias = torch.randn(c, generator=g, dtype=torch.float64)
    dout = torch.randn(x.shape, generator=g, dtype=torch.float64) + 0.2
    return x, color, bias, dout


def _eval_stats(x, gs, seed):
    g = torch.Generator().manual_seed(seed)
    c = x.shape[1]
    a = torch.randn(c // gs, gs, 2 * gs, generator=g, dtype=torch.float64)
    return 0.3 * torch.randn(c, generator=g, dtype=torch.float64), a @ a.transpose(1, 2) / (2 * gs) + 0.5 * torch.eye(gs, dtype=torch.float64)


# =========================================================================== CPU: the float64 reference
@pytest.mark.parametrize("gs", [8, 16, 64])
@pytest.mark.parametrize("train", [True, False])
def test_closed_form_backward_matches_autograd(gs, train):
    x, color, bias, dout = _cpu_case(gs, gs)
    mean, cov = (None, None) if train else _eval_stats(x, gs, gs)
    xt, ct, bt = (t.clone().requires_grad_(True) for t in (x, color, bias))
    y, *_ = R.wc_torch(xt, gs, ct, bt, mean=mean, cov=cov)
    dx, dc, db = torch.autograd.grad(y, (xt, ct, bt), dout)
    fx, fc, fb = R.closed_form_backward(x, gs, color, dout, mean=mean, cov=cov)
    for a, b in ((fx, dx), (fc, dc), (fb, db)):
        assert (a - b).abs().max() <= 1e-10 * b.abs().max(), float((a - b).abs().max())


@pytest.mark.parametrize("train", [True, False])
def test_closed_form_parameter_gradients_match_finite_differences(train):
    gs = 8
    x, color, bias, dout = _cpu_case(gs, 3)
    mean, cov = (None, None) if train else _eval_stats(x, gs, 3)
    _, dc, db = R.closed_form_backward(x, gs, color, dout, mean=mean, cov=cov)
    loss = lambda c, b: float((dout * R.wc_torch(x, gs, c, b, mean=mean, cov=cov)[0]).sum())
    h = 1e-6
    rng = np.random.default_rng(0)
    for _ in range(3):
        v = torch.tensor(rng.standard_normal(tuple(color.shape)))
        fd = (loss(color + h * v, bias) - loss(color - h * v, bias)) / (2 * h)
        assert abs(fd - float((dc * v).sum())) <= 1e-6 * max(abs(fd), 1.0)
        u = torch.tensor(rng.standard_normal(tuple(bias.shape)))
        fd = (loss(color, bias + h * u) - loss(color, bias - h * u)) / (2 * h)
        assert abs(fd - float((db * u).sum())) <= 1e-6 * max(abs(fd), 1.0)


def test_identity_colouring_is_whitening():
    x, color, bias, _ = _cpu_case(16, 1)
    eye = torch.eye(16, dtype=torch.float64).expand_as(color)
    y, mu, cov, w = R.wc_torch(x, 16, eye, torch.zeros_like(bias), eps=0.0)
    yg = y.transpose(0, 1).reshape(2, 16, -1)
    assert torch.allclose(yg @ yg.transpose(1, 2) / yg.shape[-1], torch.eye(16, dtype=y.dtype).expand(2, 16, 16), atol=1e-9)


# =========================================================================== CPU: module surface
def test_module_surface_and_state_dicts():
    import inspect
    import dwt_b200
    assert "WCTransform2d" in dwt_b200.__all__
    assert inspect.signature(dwt_b200.WCTransform2d.__init__) == inspect.signature(dwt_b200.WTransform2d.__init__)
    m, w = dwt_b200.WCTransform2d(64, 16), dwt_b200.WTransform2d(64, 16)
    assert set(m.state_dict()) == {"running_mean", "running_variance", "weight", "bias"}
    assert [n for n, _ in m.named_parameters()] == ["weight", "bias"]
    assert m.weight.shape == (4, 16, 16) and m.bias.shape == (64,)
    assert torch.equal(m.weight, torch.eye(16).expand(4, 16, 16)) and torch.equal(m.bias, torch.zeros(64))
    with torch.no_grad():
        w.running_mean.normal_()
        w.running_variance.normal_()
        m.weight.normal_()
        m.bias.normal_()
    res = m.load_state_dict(w.state_dict(), strict=False)
    assert set(res.missing_keys) == {"weight", "bias"} and not res.unexpected_keys
    assert torch.equal(m.running_variance, w.running_variance) and torch.equal(m.running_mean, w.running_mean)
    m.reset_parameters()
    assert torch.equal(m.weight, torch.eye(16).expand(4, 16, 16)) and torch.equal(m.bias, torch.zeros(64))
    assert (m.group_size, m.num_groups, m.eps, m.momentum, m.alpha) == (16, 4, 1e-3, 0.1, 1)
    assert dwt_b200.WCTransform2d(8, 16).weight.shape == (1, 8, 8)
    rm, rv = torch.zeros(1, 64, 1, 1), torch.ones(4, 16, 16)
    b = dwt_b200.WCTransform2d(64, 16, running_m=rm, running_var=rv)
    assert b.running_mean.data_ptr() == rm.data_ptr() and b.running_variance.data_ptr() == rv.data_ptr()


def test_cpu_tensors_and_bad_inputs_are_refused():
    import dwt_b200
    m = dwt_b200.WCTransform2d(64, 16)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(torch.zeros(2, 64, 8, 8))
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(2, 64, 8))
    with pytest.raises(ValueError, match="expected number of channels divisible by group_size"):
        dwt_b200.WCTransform2d(48, 32)(torch.zeros(2, 48, 3, 3))


def test_domain_site_refuses_matrix_gamma_off_the_cholesky_tensor_core_path():
    import dwt_b200
    x = torch.zeros(6, 64, 8, 8)
    for gs in (2, 4):                               # at group size 1 a [C, 1, 1] gamma is the per-channel one
        site = dwt_b200.DomainTripleNorm("whiten", 64, gs)
        with pytest.raises(dwt_b200._native.NativeError, match="matrix gamma"):
            site(x, [dwt_b200.WTransform2d(64, gs)] * 3, torch.zeros(64 // gs, gs, gs), torch.zeros(64))
    site = dwt_b200.DomainTripleNorm("whiten", 64, 16)
    for mod in (dwt_b200.ZCAWTransform2d(64, 16), dwt_b200.ExactZCAWTransform2d(64, 16)):
        with pytest.raises(dwt_b200._native.NativeError, match="Cholesky basis"):
            site(x, [mod] * 3, torch.zeros(4, 16, 16), torch.zeros(64))
    with pytest.raises(ValueError, match="matrix gamma has shape"):
        site(x, [dwt_b200.WTransform2d(64, 16)] * 3, torch.zeros(4, 8, 8), torch.zeros(64))


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _fp(v):
    return None if v is None else ctypes.c_void_p(v)


def _color_fwd(lib, N=8, C=128, HW=3136, gs=64, D=1, mode=0, color=_FAKE, bias=_FAKE):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_color_fwd(p, p, N, C, HW, gs, D, mode, 1e-3, 0.1, 0, None, None, _fp(color), _fp(bias), p, p, p,
                                    1 << 40, None)


def _color_bwd(lib, N=8, C=128, HW=3136, gs=64, D=1, mode=0, color=_FAKE, dcolor=_FAKE, dbias=_FAKE):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_color_bwd(p, p, p, N, C, HW, gs, D, mode, 1e-3, p, p, _fp(color), _fp(dcolor), _fp(dbias), p,
                                    1 << 40, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


_COLOR = b"colouring transform is built for the tensor-core kernels only"


@pytest.mark.parametrize("call", [_color_fwd, _color_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(gs=1), -4, _COLOR), (dict(gs=2), -4, _COLOR), (dict(gs=4), -4, _COLOR),
    (dict(gs=128), -4, _COLOR), (dict(C=128, gs=256), -4, _COLOR),
    (dict(HW=16, N=512), -4, _COLOR),                                       # HW < 32: the tiled shapes
    (dict(HW=36, N=64), -4, _COLOR),                                        # N*HW < 4096 per domain
    (dict(HW=34, N=512), -4, _COLOR),                                       # HW % 4 != 0
    (dict(HW=36, N=512, mode=0x200), -4, _COLOR),                           # NCHW bf16: HW % 8 != 0
    (dict(C=64, gs=4, mode=0x100), -4, _COLOR),                             # channels-last group size 4
    (dict(color=None), -1, b"null pointer argument (color)"),
    (dict(color=_FAKE + 4), -1, b"color must be 16-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


@pytest.mark.parametrize("kw, text", [
    (dict(bias=None), b"null pointer argument (bias)"), (dict(bias=_FAKE + 8), b"bias must be 16-byte aligned")])
def test_c_abi_refuses_bad_bias(lib, kw, text):
    assert _color_fwd(lib, **kw) == -1
    assert text in lib.dwt_last_error()


@pytest.mark.parametrize("kw, text", [
    (dict(dcolor=None), b"dcolor and dbias go together"), (dict(dbias=None), b"dcolor and dbias go together"),
    (dict(dcolor=_FAKE + 4), b"dcolor must be 16-byte aligned"), (dict(dbias=_FAKE + 4), b"dbias must be 16-byte aligned")])
def test_c_abi_refuses_bad_gradients(lib, kw, text):
    assert _color_bwd(lib, **kw) == -1
    assert text in lib.dwt_last_error()


def test_c_abi_keeps_the_other_bases_texts(lib):
    p = ctypes.c_void_p(_FAKE)
    assert lib.dwt_whiten_eigh_fwd(p, p, 8, 128, 3136, 4, 1, 0, 1e-3, 0.1, 0, None, None, p, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_last_error().startswith(b"the exact ZCA basis (eigendecomposition) is built for the tensor-core")
    assert lib.dwt_whiten_eigh_fwd(p, p, 512, 128, 36, 64, 1, 0x200, 1e-3, 0.1, 0, None, None, p, p, p, p, 1 << 40, None) == -4
    assert b"HW >= 32 and a multiple of 8" in lib.dwt_last_error() and b"colouring" not in lib.dwt_last_error()


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\ncolouring transform, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-40s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b, bound=BOUND):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= bound and m <= 5 * bound, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def mixed(shape, dev, seed=0, shift=1.5):
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    mix = torch.randn(c, c, device=dev, generator=g) / c ** 0.5 + torch.eye(c, device=dev)
    return (torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, h, w, device=dev, generator=g)) + shift).contiguous()


def params(c, gs, dev, seed=5, identity=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    eye = torch.eye(gs, device=dev).expand(c // gs, gs, gs)
    if identity:
        return eye.clone(), torch.zeros(c, device=dev)
    return eye + 0.3 * torch.randn(c // gs, gs, gs, device=dev, generator=g) / gs ** 0.5, torch.randn(c, device=dev, generator=g)


def running_pair(c, gs, dev, seed=7):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(c // gs, gs, 2 * gs, device=dev, generator=g)
    return (torch.randn(1, c, 1, 1, device=dev, generator=g) * 0.1,
            0.25 * torch.bmm(a, a.transpose(1, 2)) / (2 * gs) + torch.eye(gs, device=dev))


def families(prof):
    return {k.split("|")[0] for k in prof}


def reference(x, dy, gs, color, bias, d, train, running, momentum=0.1, eps=1e-3):
    """float64 per domain: y, dx, dcolor, dbias (summed over domains), running buffers after the ordered EMA."""
    n = x.shape[0] // d
    rm, rc = (t.double().cpu().clone() for t in running)
    ys, dxs, dc, db = [], [], 0, 0
    for k in range(d):
        xk, dk = x[k * n:(k + 1) * n].double().cpu(), dy[k * n:(k + 1) * n].double().cpu()
        mean, cov = (None, None) if train else (rm.reshape(-1), rc)
        y, mu, cv, _ = R.wc_torch(xk, gs, color.double().cpu(), bias.double().cpu(), eps, mean, cov)
        dx, c_, b_ = R.closed_form_backward(xk, gs, color.double().cpu(), dk, eps, mean, cov)
        ys.append(y)
        dxs.append(dx)
        dc, db = dc + c_, db + b_
        if train:
            rm = (1 - momentum) * rm + momentum * mu.reshape(rm.shape)
            rc = (1 - momentum) * rc + momentum * cv
    return torch.cat(ys), torch.cat(dxs), dc, db, rm, rc


CASES = [(8, 64), (16, 96), (32, 96), (64, 128)]


@gpu
@pytest.mark.parametrize("gs, c", CASES)
@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_against_float64(dev, worst, gs, c, d, mode, layout):
    """WCTransform2d (d = 1) or a DomainTripleNorm site of d domains sharing gamma / beta, forward + backward, against
    float64; offset inputs and gradients; eval normalises with running buffers that differ from the batch statistics
    (the eval dcolor needs R without the pilot shift of dy)."""
    import dwt_b200
    from dwt_b200 import _native as nv
    n = 8
    x = mixed((d * n, c, 32, 32), dev, seed=gs + d, shift=1.5)
    g = torch.Generator(device=dev).manual_seed(2)
    dy = torch.randn(x.shape, device=dev, generator=g) + 0.5
    if layout == "nhwc":
        x, dy = x.contiguous(memory_format=torch.channels_last), dy.contiguous(memory_format=torch.channels_last)
    color, bias = params(c, gs, dev)
    rm, rc = running_pair(c, gs, dev)
    running0 = (rm.clone(), rc.clone())
    train = mode == "train"
    xg = x.clone().requires_grad_(True)
    nv.profile_begin()
    if d == 1:
        m = dwt_b200.WCTransform2d(c, gs, running_m=rm, running_var=rc).to(dev).train(train)
        with torch.no_grad():
            m.weight.copy_(color)
            m.bias.copy_(bias)
        y = m(xg)
        dx, dc, db = torch.autograd.grad(y, (xg, m.weight, m.bias), dy)
    else:
        mods = [dwt_b200.WTransform2d(c, gs, running_m=rm, running_var=rc).to(dev).train(train) for _ in range(d)]
        cg, bg = color.clone().requires_grad_(True), bias.view(c, 1, 1).clone().requires_grad_(True)
        y = dwt_b200.DomainTripleNorm("whiten", c, gs, n_domains=d)(xg, mods, cg, bg)
        dx, dc, db = torch.autograd.grad(y, (xg, cg, bg), dy)
        db = db.reshape(-1)
    prof = nv.profile_end()
    sfx = "_nhwc" if layout == "nhwc" else ""
    fam = families(prof)
    assert {"dense_fwd_color", "tc_apply" + sfx, "tc_bwd_reduce" + sfx, "dense_bwd_color", "tc_bwd_apply" + sfx} <= fam
    assert fam <= {"tc_stats" + sfx, "dense_fwd_color", "tc_apply" + sfx, "tc_bwd_reduce" + sfx, "dense_bwd_color",
                   "tc_bwd_apply" + sfx}, fam
    assert ("tc_stats" + sfx in fam) == train
    ry, rdx, rdc, rdb, rrm, rrc = reference(x, dy, gs, color, bias, d, train, running0)
    label = f"gs{gs} C{c} D{d} {mode} {layout}"
    check(worst, label, "y", y, ry)
    check(worst, label, "dx", dx, rdx)
    check(worst, label, "dcolor", dc, rdc)
    check(worst, label, "dbias", db, rdb)
    check(worst, label, "running_mean", rm, rrm, STAT_BOUND)
    check(worst, label, "running_cov", rc, rrc, STAT_BOUND)
    assert nv.status(dev) == 0


@gpu
@pytest.mark.parametrize("mode", ["nograd", "untracked"])
def test_nograd_and_untracked_statistics(dev, worst, mode):
    import dwt_b200
    c, gs = 128, 64
    x = mixed((8, c, 32, 32), dev, seed=3)
    color, bias = params(c, gs, dev)
    rm, rc = running_pair(c, gs, dev)
    running0 = (rm.clone(), rc.clone())
    m = dwt_b200.WCTransform2d(c, gs, running_m=rm, running_var=rc, track_running_stats=mode != "untracked").to(dev)
    m.train(mode == "nograd")
    with torch.no_grad():
        m.weight.copy_(color)
        m.bias.copy_(bias)
        y = m(x)
    ry, _, _, _, rrm, rrc = reference(x, torch.zeros_like(x), gs, color, bias, 1, True, running0)
    check(worst, mode, "y", y, ry)
    if mode == "nograd":
        check(worst, mode, "running_mean", m.running_mean, rrm, STAT_BOUND)
        check(worst, mode, "running_cov", m.running_variance, rrc, STAT_BOUND)
    else:
        assert torch.equal(rm, running0[0]) and torch.equal(rc, running0[1])


@gpu
@pytest.mark.parametrize("gs, c", CASES)
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_identity_colouring_equals_wtransform_bit_for_bit(dev, gs, c, mode):
    import dwt_b200
    x = mixed((8, c, 32, 32), dev, seed=gs)
    dy = torch.randn(x.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    outs = []
    for cls in (dwt_b200.WTransform2d, dwt_b200.WCTransform2d):
        rm, rc = running_pair(c, gs, dev)
        m = cls(c, gs, running_m=rm, running_var=rc).to(dev).train(mode == "train")
        xg = x.clone().requires_grad_(True)
        y = m(xg)
        (dx,) = torch.autograd.grad(y, xg, dy)
        outs.append((y, dx, rm, rc))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _run_module(m, x, dy):
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    dx, dc, db = torch.autograd.grad(y, (xg, m.weight, m.bias), dy)
    return y, dx, dc, db


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_layouts_dtypes_and_reruns_agree_bit_for_bit(dev, mode):
    """channels-last = NCHW; bf16 = the fp32 kernels on the widened bf16 values, rounded (dcolor / dbias equal that fp32
    call's); two reruns are identical."""
    import dwt_b200
    c, gs = 96, 32
    xb = mixed((8, c, 32, 32), dev, seed=9).bfloat16()
    dyb = torch.randn(xb.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(4)).bfloat16()
    color, bias = params(c, gs, dev)

    def module():
        rm, rc = running_pair(c, gs, dev)
        m = dwt_b200.WCTransform2d(c, gs, running_m=rm, running_var=rc).to(dev).train(mode == "train")
        with torch.no_grad():
            m.weight.copy_(color)
            m.bias.copy_(bias)
        return m
    ref = _run_module(module(), xb.float(), dyb.float())
    again = _run_module(module(), xb.float(), dyb.float())
    assert all(torch.equal(a, b) for a, b in zip(ref, again))
    cl = _run_module(module(), xb.float().contiguous(memory_format=torch.channels_last),
                     dyb.float().contiguous(memory_format=torch.channels_last))
    assert all(torch.equal(a, b) for a, b in zip(ref, cl))
    for fmt in (torch.contiguous_format, torch.channels_last):
        y, dx, dc, db = _run_module(module(), xb.contiguous(memory_format=fmt), dyb.contiguous(memory_format=fmt))
        assert y.dtype == torch.bfloat16 and dx.dtype == torch.bfloat16
        assert torch.equal(y, ref[0].bfloat16()) and torch.equal(dx, ref[1].bfloat16())
        assert torch.equal(dc, ref[2]) and torch.equal(db, ref[3])


@gpu
def test_graph_replay_equals_eager(dev):
    import dwt_b200
    c, gs = 128, 64
    x = mixed((8, c, 32, 32), dev, seed=11)
    dy = torch.randn(x.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    color, bias = params(c, gs, dev)

    def module():
        m = dwt_b200.WCTransform2d(c, gs).to(dev)
        with torch.no_grad():
            m.weight.copy_(color)
            m.bias.copy_(bias)
        return m
    eager = module()
    ref = _run_module(eager, x, dy)
    m = module()
    sx, sdy = x.clone(), dy.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _run_module(m, sx, sdy)                      # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    with torch.no_grad():
        m.running_mean.zero_()
        m.running_variance.fill_(1.0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _run_module(m, sx, sdy)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(out, ref))


@gpu
def test_not_positive_definite_group_sets_status_and_skips_its_ema(dev):
    import dwt_b200
    from dwt_b200 import _native as nv
    c, gs, d, n = 64, 16, 3, 8
    x = mixed((d * n, c, 32, 32), dev, seed=12)
    x[n:2 * n, 16] = float("nan")                   # domain 1, group 1
    pairs = [running_pair(c, gs, dev, seed=20 + k) for k in range(d)]
    before = [(a.clone(), b.clone()) for a, b in pairs]
    mods = [dwt_b200.WTransform2d(c, gs, running_m=a, running_var=b).to(dev) for a, b in pairs]
    color, bias = params(c, gs, dev)
    nv.clear_status(dev)
    with torch.no_grad():
        dwt_b200.DomainTripleNorm("whiten", c, gs, n_domains=d)(x, mods, color, bias)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    assert torch.equal(pairs[1][1][1], before[1][1][1]) and torch.equal(pairs[1][0][:, 16:32], before[1][0][:, 16:32])
    assert not torch.equal(pairs[1][1][0], before[1][1][0])          # the other groups of that domain update
    for k in (0, 2):
        assert not torch.equal(pairs[k][1][1], before[k][1][1])


@gpu
@pytest.mark.parametrize("replicated", [False, True])
def test_domain_site_matrix_gamma_with_relu_and_residual(dev, worst, replicated):
    """The matrix-gamma site equals three module calls followed by the colouring, ReLU and residual in float64 (the
    gradient through the kernel's ReLU mask)."""
    import dwt_b200
    c, gs, d, n = 128, 64, 3, 8
    x = mixed(((1 if replicated else d) * n, c, 32, 32), dev, seed=13)
    res = torch.randn(x.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(6))
    dy = torch.randn(x.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    color, bias = params(c, gs, dev)
    rm, rc = running_pair(c, gs, dev)
    running0 = (rm.clone(), rc.clone())
    mods = [dwt_b200.WTransform2d(c, gs, running_m=rm, running_var=rc).to(dev) for _ in range(d)]
    xg, cg, bg = x.clone().requires_grad_(True), color.clone().requires_grad_(True), bias.view(c, 1, 1).clone().requires_grad_(True)
    y = dwt_b200.DomainTripleNorm("whiten", c, gs, n_domains=d)(xg, mods, cg, bg, relu=True, residual=res,
                                                                replicated=replicated)
    dx, dc, db = torch.autograd.grad(y, (xg, cg, bg), dy)
    xd, cd, bd = (t.detach().double().cpu().requires_grad_(True) for t in (x, color, bias))
    outs = []
    for k in range(1 if replicated else d):
        z, *_ = R.wc_torch(xd[k * n:(k + 1) * n], gs, cd, bd)
        outs.append(z)
    zr = torch.cat(outs) + res.double().cpu()
    yr = torch.relu(zr)
    # the ReLU mask from the kernel's output: where float32 and float64 disagree about the sign of a value near zero, the
    # two masks differ and so would the gradient of that element, whatever the accuracy of the kernels
    rdx, rdc, rdb = torch.autograd.grad(zr, (xd, cd, bd), (dy * (y > 0)).double().cpu())
    label = f"site relu+residual{' replicated' if replicated else ''}"
    check(worst, label, "y", y, yr)
    check(worst, label, "dx", dx, rdx)
    check(worst, label, "dcolor", dc, rdc)
    check(worst, label, "dbias", db.reshape(-1), rdb)
    if replicated:                                  # one buffer shared by three branches: the 3-fold EMA
        _, mu, cv, _ = R.wc_torch(x.double().cpu(), gs, cd.detach(), bd.detach())
        k = 0.9 ** 3
        check(worst, label, "running_mean", rm, k * running0[0].double().cpu() + (1 - k) * mu.reshape(rm.shape), STAT_BOUND)
        check(worst, label, "running_cov", rc, k * running0[1].double().cpu() + (1 - k) * cv, STAT_BOUND)
