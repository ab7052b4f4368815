"""Instance whitening (InstanceWTransform2d, functional.instance_whiten, dwt_whiten_instance_*).

CPU: the float64 closed-form backward (tests/support/iw_reference.py) against autograd through torch.linalg.cholesky /
inverse and against central finite differences; the module surface; the refusals of the C ABI (argument checks run before
any device call, so fake pointers do), and that the other entry points keep theirs.

GPU: the tensor-core kernels against the float64 reference -- y and dx within 1e-4 norm-wise, max element within 1e-3 of
the largest -- at the production shapes and the launch edges, and against themselves bit for bit (layouts, dtypes,
reruns, graphs, images that do not depend on each other).
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import iw_reference as R  # noqa: E402

BOUND, MAX_BOUND = 1e-4, 1e-3
gpu = pytest.mark.gpu


def _cpu_case(gs, seed, n=3, c=None, hw=(4, 5)):
    c = c or 2 * gs
    g = torch.Generator().manual_seed(seed)
    mix = torch.eye(c, dtype=torch.float64) + 0.3 * torch.randn(c, c, generator=g, dtype=torch.float64) / c ** 0.5
    x = torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, *hw, generator=g, dtype=torch.float64)) + 0.5
    x = x + torch.randn(n, c, 1, 1, generator=g, dtype=torch.float64)          # a different mean per image
    dout = torch.randn(x.shape, generator=g, dtype=torch.float64) + 0.2
    return x, dout


# =========================================================================== CPU: the float64 reference
@pytest.mark.parametrize("gs", [8, 16, 64])
def test_closed_form_backward_matches_autograd(gs):
    x, dout = _cpu_case(gs, gs, hw=(9, 9) if gs == 64 else (4, 5))
    xt = x.clone().requires_grad_(True)
    y, *_ = R.iw_torch(xt, gs)
    (dx,) = torch.autograd.grad(y, xt, dout)
    fx = R.closed_form_backward(x, gs, dout)
    assert (fx - dx).abs().max() <= 1e-10 * dx.abs().max(), float((fx - dx).abs().max())


def test_closed_form_backward_matches_finite_differences():
    gs = 8
    x, dout = _cpu_case(gs, 3)
    dx = R.closed_form_backward(x, gs, dout)
    loss = lambda t: float((dout * R.iw_torch(t, gs)[0]).sum())
    h = 1e-6
    rng = np.random.default_rng(0)
    for _ in range(4):
        v = torch.tensor(rng.standard_normal(tuple(x.shape)))
        fd = (loss(x + h * v) - loss(x - h * v)) / (2 * h)
        assert abs(fd - float((dx * v).sum())) <= 1e-6 * max(abs(fd), 1.0)


def test_images_are_independent_and_white():
    x, _ = _cpu_case(16, 1, n=4)
    y, *_ = R.iw_torch(x, 16, eps=0.0)
    yg = y.reshape(4, 2, 16, -1)
    assert torch.allclose(yg @ yg.transpose(-1, -2) / yg.shape[-1], torch.eye(16, dtype=y.dtype).expand(4, 2, 16, 16), atol=1e-9)
    y2, *_ = R.iw_torch(torch.cat([x[:2], 3 * x[2:] + 1]), 16, eps=0.0)
    assert torch.allclose(y2[:2], y[:2], atol=0) and torch.allclose(y2[2:], y[2:], atol=1e-9)


# =========================================================================== CPU: module surface
def test_module_surface():
    import inspect
    import dwt_b200
    assert "InstanceWTransform2d" in dwt_b200.__all__
    assert list(inspect.signature(dwt_b200.InstanceWTransform2d.__init__).parameters) == ["self", "num_features", "group_size", "eps"]
    m = dwt_b200.InstanceWTransform2d(64, 16)
    assert m.state_dict() == {} and list(m.buffers()) == [] and list(m.parameters()) == []
    assert (m.num_features, m.group_size, m.num_groups, m.eps) == (64, 16, 4, 1e-3)
    assert dwt_b200.InstanceWTransform2d(8, 16).group_size == 8                  # min(C, gs), as WTransform2d
    m.load_state_dict({})
    assert "group_size=16" in repr(m)


def test_cpu_tensors_and_bad_inputs_are_refused():
    import dwt_b200
    from dwt_b200 import functional as F
    m = dwt_b200.InstanceWTransform2d(64, 16)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(torch.zeros(2, 64, 16, 16))
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        F.instance_whiten(torch.zeros(2, 64, 16, 16), group_size=16, eps=1e-3)
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(2, 64, 8))
    with pytest.raises(ValueError, match="expected number of channels divisible by group_size"):
        dwt_b200.InstanceWTransform2d(48, 32)(torch.zeros(2, 48, 16, 16))


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _fp(v):
    return None if v is None else ctypes.c_void_p(v)


def _iw_fwd(lib, N=8, C=128, HW=3136, gs=64, flags=0, x=_FAKE, y=_FAKE, save_w=_FAKE, ws_bytes=1 << 40):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_instance_fwd(_fp(x), _fp(y), N, C, HW, gs, flags, 1e-3, p, _fp(save_w), p, ws_bytes, None)


def _iw_bwd(lib, N=8, C=128, HW=3136, gs=64, flags=0, x=_FAKE, y=_FAKE, save_w=_FAKE, ws_bytes=1 << 40):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_instance_bwd(_fp(x), p, _fp(y), N, C, HW, gs, flags, 1e-3, p, _fp(save_w), p, ws_bytes, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


_IW = b"instance whitening is built for the tensor-core kernels only"


@pytest.mark.parametrize("call", [_iw_fwd, _iw_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(gs=1), -4, _IW), (dict(gs=2), -4, _IW), (dict(gs=4), -4, _IW), (dict(gs=128), -4, _IW),
    (dict(C=96, gs=24), -4, _IW),                                           # not a power of two dividing 64
    (dict(C=96, gs=64), -4, _IW),                                           # C not a multiple of gs
    (dict(HW=196), -4, _IW), (dict(HW=252), -4, _IW),                       # HW < 256 (14 x 14)
    (dict(HW=258), -4, _IW), (dict(HW=258, flags=0x100), -4, _IW),          # HW % 4 != 0
    (dict(HW=260, flags=0x200), -4, _IW),                                   # NCHW bf16: HW % 8 != 0
    (dict(N=65536, C=64, HW=256), -4, _IW),                                 # more images than grid.z
    (dict(N=1024, C=256, HW=8192), -4, _IW),                                # N*C*HW >= 2^31
    (dict(flags=0x1), -1, b"bad flags"), (dict(flags=0x400), -1, b"bad flags"),
    (dict(N=0), -1, b"empty tensor"), (dict(HW=0), -1, b"empty tensor"),
    (dict(x=None), -1, b"null pointer argument"), (dict(y=None), -1, b"null pointer argument"),
    (dict(save_w=None), -1, b"null pointer argument"),
    (dict(x=_FAKE + 4), -1, b"must be 16-byte aligned"), (dict(y=_FAKE + 8), -1, b"must be 16-byte aligned"),
    (dict(save_w=_FAKE + 4), -1, b"must be 16-byte aligned"),
    (dict(flags=0x300, x=_FAKE + 8), -1, b"must be 16-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


@pytest.mark.parametrize("call", [_iw_fwd, _iw_bwd])
@pytest.mark.parametrize("kw", [dict(N=1, C=64, HW=256, gs=64), dict(N=3, C=96, HW=784, gs=32, flags=0x300),
                                dict(N=2, C=64, HW=1024, gs=8, flags=0x200)])
def test_small_batches_pass_every_check_up_to_the_workspace(lib, call, kw):
    """No per-batch sample floor: N*HW < 4096 passes the argument checks and stops at a too-small workspace."""
    need = lib.dwt_instance_workspace_bytes(kw["N"], kw["C"], kw["HW"], kw["gs"])
    assert need > 0
    assert call(lib, ws_bytes=need - 1, **kw) == -2
    assert b"workspace too small" in lib.dwt_last_error()


def test_workspace_query(lib):
    assert lib.dwt_instance_workspace_bytes(8, 128, 3136, 64) > 0
    for args in ((8, 128, 3136, 4), (8, 128, 196, 64), (0, 128, 3136, 64), (8, 96, 3136, 64), (8, 128, 3136, 128)):
        assert lib.dwt_instance_workspace_bytes(*args) == 0
    a = lib.dwt_instance_workspace_bytes(192, 256, 3136, 64)
    assert a >= 4 * 192 * (256 // 64) * (2 * 64 * 64 + 64)                  # the backward coefficients at least


def test_other_entry_points_keep_their_refusals(lib):
    """Five domains stay refused by the domain entry points, with their text (the images of an instance call are not
    domains)."""
    p = ctypes.c_void_p(_FAKE)
    assert lib.dwt_whiten_fwd(p, p, 8, 128, 3136, 64, 5, 0, 1e-3, 0.1, 0, None, None, None, None, None, None, 0, p, p, p,
                              1 << 40, None) == -1
    assert lib.dwt_last_error() == b"n_domains 5 outside [1,4]"
    assert lib.dwt_workspace_bytes(8, 128, 3136, 64, 5) == 0


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\ninstance whitening, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-44s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= BOUND and m <= MAX_BOUND, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def images(shape, dev, seed=0, cond=None):
    """[N, C, H, W] float32: per image its own channel mixing I + 0.5 G / sqrt(C) (group covariances conditioned to a few
    tens) and mean.  cond: the covariance of every group of every image has that condition number instead (eigenvalues
    log-spaced from 1 down to 1/cond, a random basis per image and group)."""
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    z = torch.randn(n, c, h * w, device=dev, generator=g)
    if cond is None:
        mix = torch.eye(c, device=dev) + 0.5 * torch.randn(n, c, c, device=dev, generator=g) / c ** 0.5
        x = mix @ z
    else:
        gs = 64 if c % 64 == 0 else 32
        q, _ = torch.linalg.qr(torch.randn(n, c // gs, gs, gs, device=dev, generator=g, dtype=torch.float64))
        sv = torch.logspace(0, -0.5 * np.log10(cond), gs, device=dev, dtype=torch.float64)
        x = ((q * sv) @ z.double().reshape(n, c // gs, gs, -1)).float().reshape(n, c, -1)
    x = x + 2.0 * torch.randn(n, c, 1, device=dev, generator=g) + 1.0
    return x.reshape(n, c, h, w).contiguous()


def grad(shape, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, device=dev, generator=g) + 0.5


def run(x, dy, gs, eps=1e-3):
    from dwt_b200 import functional as F
    xg = x.detach().clone().requires_grad_(True)
    y = F.instance_whiten(xg, group_size=gs, eps=eps)
    (dx,) = torch.autograd.grad(y, xg, dy)
    return y.detach(), dx


def against_float64(worst, label, x, dy, gs):
    y, dx = run(x, dy, gs)
    xd, dyd = x.double(), dy.double()
    check(worst, label, "y", y, R.iw_torch(xd, gs)[0])
    check(worst, label, "dx", dx, R.closed_form_backward(xd, gs, dyd))


@gpu
@pytest.mark.parametrize("shape, gs", [
    ((192, 256, 56, 56), 16), ((192, 256, 56, 56), 64),       # many short problems: a CTA owns a whole image
    ((8, 64, 112, 112), 64),                                  # few long ones: an image split across CTAs
    ((16, 64, 16, 16), 64), ((16, 64, 16, 16), 8),            # the smallest accepted HW
    ((24, 128, 28, 28), 32),                                  # 28 x 28
    ((8, 96, 32, 32), 32), ((8, 96, 32, 32), 16),             # a partial 64-channel super-block
])
def test_against_float64(dev, worst, shape, gs):
    x = images(shape, dev, seed=gs)
    against_float64(worst, f"{list(shape)} gs {gs}", x, grad(shape, dev), gs)


@gpu
@pytest.mark.parametrize("cond", [1.0, 10.0, 100.0, 1000.0])
@pytest.mark.parametrize("shape", [(16, 128, 28, 28), (8, 64, 56, 56)])
def test_conditioning_against_float64(dev, worst, cond, shape):
    x = images(shape, dev, seed=3, cond=cond)
    against_float64(worst, f"{list(shape)} gs 64 cond {cond:g}", x, grad(shape, dev), 64)


@gpu
@pytest.mark.parametrize("shape, gs", [((192, 256, 56, 56), 64), ((8, 64, 112, 112), 16), ((16, 96, 16, 16), 32)])
def test_channels_last_is_bitwise_nchw(dev, shape, gs):
    x, dy = images(shape, dev, seed=4), grad(shape, dev)
    y, dx = run(x, dy, gs)
    cl = torch.channels_last
    yc, dxc = run(x.contiguous(memory_format=cl), dy.contiguous(memory_format=cl), gs)
    assert yc.is_contiguous(memory_format=cl) and dxc.is_contiguous(memory_format=cl)
    assert torch.equal(yc, y) and torch.equal(dxc, dx)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("shape, gs", [((32, 128, 56, 56), 64), ((16, 64, 28, 28), 16)])
def test_bf16_is_the_fp32_kernels_rounded(dev, layout, shape, gs):
    fmt = torch.channels_last if layout == "nhwc" else torch.contiguous_format
    x = images(shape, dev, seed=5).bfloat16().contiguous(memory_format=fmt)
    dy = grad(shape, dev).bfloat16().contiguous(memory_format=fmt)
    y, dx = run(x, dy, gs)
    assert y.dtype == torch.bfloat16 and dx.dtype == torch.bfloat16
    yf, dxf = run(x.float(), dy.float(), gs)
    assert torch.equal(y, yf.bfloat16()) and torch.equal(dx, dxf.bfloat16())


@gpu
def test_bf16_nchw_off_the_bf16_rows_runs_the_fp32_kernels(dev):
    shape = (4, 64, 18, 18)                                   # HW = 324: a multiple of 4, not of 8
    x, dy = images(shape, dev, seed=6).bfloat16(), grad(shape, dev).bfloat16()
    y, dx = run(x, dy, 16)
    yf, dxf = run(x.float(), dy.float(), 16)
    assert y.dtype == torch.bfloat16 and torch.equal(y, yf.bfloat16()) and torch.equal(dx, dxf.bfloat16())


@gpu
def test_reruns_are_bit_identical(dev):
    for shape, gs in (((192, 256, 56, 56), 64), ((8, 64, 112, 112), 64)):
        x, dy = images(shape, dev, seed=7), grad(shape, dev)
        a, b = run(x, dy, gs), run(x, dy, gs)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@gpu
def test_cuda_graph_capture_and_replay(dev):
    import dwt_b200
    shape, gs = (16, 128, 28, 28), 32
    m = dwt_b200.InstanceWTransform2d(128, gs)
    x, dy = images(shape, dev, seed=8), grad(shape, dev)
    sx, sdy = x.clone(), dy.clone()

    def step():
        xg = sx.detach().requires_grad_(True)
        y = m(xg)
        (dx,) = torch.autograd.grad(y, xg, sdy)
        return y.detach(), dx

    ref = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                        # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])
    sx.copy_(images(shape, dev, seed=9))
    graph.replay()
    torch.cuda.synchronize()
    fresh = run(sx, sdy, gs)
    assert torch.equal(out[0], fresh[0]) and torch.equal(out[1], fresh[1])


@gpu
def test_nan_image_and_indefinite_group_set_status_and_stay_local(dev):
    from dwt_b200 import _native as nv
    shape, gs, eps = (8, 64, 32, 32), 16, -1e-3       # eps < 0: a constant group's S = eps I is indefinite
    x, dy = images(shape, dev, seed=10), grad(shape, dev)
    y0, dx0 = run(x, dy, gs, eps)
    bad = x.clone()
    bad[3, 5, 7, 9] = float("nan")                    # image 3, group 0
    bad[6, 16:32] = 0.25                              # image 6, group 1: zero covariance
    nv.clear_status(dev)
    y, dx = run(bad, dy, gs, eps)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    assert torch.isnan(y[3, :16]).all() and torch.isnan(y[6, 16:32]).all()
    # the NaN pixel reaches its whole image (the apply multiplies a super-block's zero entries by it); the indefinite
    # group stays in its group
    keep = torch.ones(shape[:2], dtype=torch.bool, device=dev)
    keep[3] = keep[6, 16:32] = False
    assert torch.equal(y[keep], y0[keep])
    assert torch.isnan(dx[3, :16]).all() and torch.isnan(dx[6, 16:32]).all()
    assert torch.equal(dx[keep], dx0[keep])
    run(x, dy, gs, eps)
    assert nv.status(dev) == 0


@gpu
def test_one_image_agrees_with_the_domain_layer(dev):
    """N = 1 with HW >= 4096: the domain layer without running statistics whitens that image by the same statistics."""
    import dwt_b200
    shape, gs = (1, 128, 64, 64), 32
    x, dy = images(shape, dev, seed=11), grad(shape, dev)
    y, dx = run(x, dy, gs)
    w = dwt_b200.WTransform2d(128, gs, track_running_stats=False).to(dev)
    xg = x.clone().requires_grad_(True)
    yw = w(xg)
    (dxw,) = torch.autograd.grad(yw, xg, dy)
    for a, b in ((y, yw), (dx, dxw)):
        r, m = rel(a, b)
        assert r <= 1e-6 and m <= 1e-5, (r, m)


@gpu
def test_training_step_decreases_the_loss(dev):
    import dwt_b200
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Conv2d(3, 64, 3, padding=1), dwt_b200.InstanceWTransform2d(64, 16),
                              torch.nn.ReLU(), torch.nn.Conv2d(64, 8, 3, padding=1)).to(dev)
    x = torch.randn(8, 3, 32, 32, device=dev)
    target = torch.randn(8, 8, 32, 32, device=dev)
    opt = torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        loss = torch.nn.functional.mse_loss(net(x), target)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert all(np.isfinite(losses)) and losses[-1] < 0.95 * losses[0], losses
