"""Switchable whitening (SwitchableWTransform2d, functional.switchable_whiten, dwt_whiten_switch_*).

CPU: the float64 closed-form backward (tests/support/sw_reference.py) -- dx and the six mix gradients -- against autograd
through torch.linalg.cholesky / inverse and against central finite differences, in train and eval; the module surface;
the refusals of the C ABI (argument checks run before any device call, so fake pointers do), and that the other entry
points keep theirs.

GPU: the tensor-core kernels against the float64 reference -- y, dx, dmix, the mixed mean and the updated running buffers
within 1e-4 norm-wise, max element within 1e-3 of the largest -- at the production shapes, the launch edges, conditioning
up to 1e3 and per-image mean offsets of ~100; against themselves bit for bit (layouts, dtypes, reruns, graphs); and at the
mixtures where they reduce to InstanceWTransform2d and WTransform2d.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import sw_reference as R  # noqa: E402

BOUND, MAX_BOUND = 1e-4, 1e-3
gpu = pytest.mark.gpu

SWA = (0.5, 0.5, 0.5, 0.5, 0.0, 0.0)          # softmax(ones) of ("bw", "iw")
SWB = (0.5, 0.5, 0.25, 0.25, 0.25, 0.25)      # softmax(ones) of all four
MIXES = {"swa": SWA, "swb": SWB, "skew": (0.8, 0.2, 0.1, 0.6, 0.2, 0.1)}


def _cpu_case(gs, seed, n=3, c=None, hw=(4, 5)):
    c = c or 2 * gs
    g = torch.Generator().manual_seed(seed)
    mix = torch.eye(c, dtype=torch.float64) + 0.3 * torch.randn(c, c, generator=g, dtype=torch.float64) / c ** 0.5
    x = torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, *hw, generator=g, dtype=torch.float64)) + 0.5
    x = x + torch.randn(n, c, 1, 1, generator=g, dtype=torch.float64)          # a different mean per image
    dout = torch.randn(x.shape, generator=g, dtype=torch.float64) + 0.2
    return x, dout


def _running(x, gs, seed):
    """Running buffers near the batch statistics of x (positive definite, not equal to them)."""
    f = R.sw_torch(x, gs, torch.tensor(SWA, dtype=x.dtype))
    g = torch.Generator(device=x.device).manual_seed(seed)
    rm = f["mu_b"].reshape(-1) + 0.1 * torch.randn(f["mu_b"].numel(), generator=g, device=x.device, dtype=x.dtype)
    return rm, 0.9 * f["cov_b"] + 0.1 * torch.eye(gs, dtype=x.dtype, device=x.device)


# =========================================================================== CPU: the float64 reference
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("mix", ["swa", "swb", "skew", "random0", "random1"])
@pytest.mark.parametrize("gs", [8, 16])
def test_closed_form_backward_matches_autograd(gs, mix, train):
    x, dout = _cpu_case(gs, gs, hw=(5, 6))
    if mix.startswith("random"):
        m = torch.rand(6, generator=torch.Generator().manual_seed(int(mix[-1])), dtype=torch.float64)
        m[2:] += 0.1                                        # keep cov_hat positive definite
    else:
        m = torch.tensor(MIXES[mix], dtype=torch.float64)
    running = None if train else _running(x, gs, 1)
    xt, mt = x.clone().requires_grad_(True), m.clone().requires_grad_(True)
    y = R.sw_torch(xt, gs, mt, running=running)["y"]
    dx, dm = torch.autograd.grad(y, (xt, mt), dout)
    fx, fm = R.closed_form_backward(x, gs, dout, m, running=running)
    assert (fx - dx).abs().max() <= 1e-10 * dx.abs().max(), float((fx - dx).abs().max())
    assert (fm - dm).abs().max() <= 1e-10 * dm.abs().max(), (fm, dm)


@pytest.mark.parametrize("train", [True, False])
def test_closed_form_backward_matches_finite_differences(train):
    gs = 8
    x, dout = _cpu_case(gs, 3)
    m = torch.tensor(MIXES["skew"], dtype=torch.float64)
    running = None if train else _running(x, gs, 2)
    dx, dm = R.closed_form_backward(x, gs, dout, m, running=running)
    loss = lambda t, mm: float((dout * R.sw_torch(t, gs, mm, running=running)["y"]).sum())
    h = 1e-6
    rng = np.random.default_rng(0)
    for _ in range(4):
        v = torch.tensor(rng.standard_normal(tuple(x.shape)))
        fd = (loss(x + h * v, m) - loss(x - h * v, m)) / (2 * h)
        assert abs(fd - float((dx * v).sum())) <= 1e-6 * max(abs(fd), 1.0)
    for k in range(6):
        e = torch.zeros(6, dtype=torch.float64)
        e[k] = h
        fd = (loss(x, m + e) - loss(x, m - e)) / (2 * h)
        assert abs(fd - float(dm[k])) <= 1e-6 * max(abs(fd), 1.0), (k, fd, float(dm[k]))


def test_mixtures_reduce_to_instance_and_batch_whitening():
    import iw_reference as IW
    x, _ = _cpu_case(16, 4)
    y_i = R.sw_torch(x, 16, torch.tensor([0.0, 1, 0, 1, 0, 0], dtype=torch.float64))["y"]
    assert torch.allclose(y_i, IW.iw_torch(x, 16)[0], atol=1e-12)
    f = R.sw_torch(x, 16, torch.tensor([1.0, 0, 1, 0, 0, 0], dtype=torch.float64), eps=0.0)
    assert torch.allclose(f["w"], f["w"][:1].expand_as(f["w"])) and torch.allclose(f["m"], f["m"][:1].expand_as(f["m"]))
    yg = f["y"].reshape(3, 2, 16, -1).permute(1, 2, 0, 3).reshape(2, 16, -1)   # the whole batch is white
    yc = yg - yg.mean(-1, keepdim=True)
    assert torch.allclose(yc @ yc.transpose(-1, -2) / yg.shape[-1], torch.eye(16, dtype=x.dtype).expand(2, 16, 16), atol=1e-9)


# =========================================================================== CPU: module surface
def test_module_surface():
    import inspect
    import dwt_b200
    assert "SwitchableWTransform2d" in dwt_b200.__all__
    assert list(inspect.signature(dwt_b200.SwitchableWTransform2d.__init__).parameters) == [
        "self", "num_features", "group_size", "components", "running_m", "running_var", "momentum", "track_running_stats", "eps"]
    m = dwt_b200.SwitchableWTransform2d(64, 16)
    assert (m.num_features, m.group_size, m.num_groups, m.eps, m.momentum, m.components) == (64, 16, 4, 1e-3, 0.1, ("bw", "iw"))
    assert dwt_b200.SwitchableWTransform2d(8, 16).group_size == 8                 # min(C, gs), as WTransform2d
    assert [n for n, _ in m.named_parameters()] == ["mean_weight", "var_weight"]
    assert torch.equal(m.mean_weight.detach(), torch.ones(2)) and torch.equal(m.var_weight.detach(), torch.ones(2))
    assert sorted(m.state_dict()) == ["mean_weight", "running_mean", "running_variance", "var_weight"]
    assert m.running_mean.shape == (1, 64, 1, 1) and m.running_variance.shape == (4, 16, 16)
    assert torch.allclose(m.mix(), torch.tensor(SWA))
    assert torch.allclose(dwt_b200.SwitchableWTransform2d(64, 16, ("bw", "iw", "bn", "in")).mix(), torch.tensor(SWB))
    assert torch.allclose(dwt_b200.SwitchableWTransform2d(64, 16, ("in",)).mix(), torch.tensor([0.0, 1, 0, 0, 0, 1]))
    m.mean_weight.data = torch.tensor([0.0, 1.0])
    m.mix().sum().backward()                                                       # differentiable
    assert m.mean_weight.grad is not None and "components=('bw', 'iw')" in repr(m)


def test_state_dict_loads_from_a_wtransform():
    import dwt_b200
    w = dwt_b200.WTransform2d(64, 16)
    w.running_mean.normal_()
    w.running_variance.normal_()
    m = dwt_b200.SwitchableWTransform2d(64, 16)
    res = m.load_state_dict(w.state_dict(), strict=False)
    assert sorted(res.missing_keys) == ["mean_weight", "var_weight"] and res.unexpected_keys == []
    assert torch.equal(m.running_mean, w.running_mean) and torch.equal(m.running_variance, w.running_variance)
    rm, rv = torch.zeros(1, 64, 1, 1), torch.ones(4, 16, 16)                       # borrowed buffers, as WTransform2d
    b = dwt_b200.SwitchableWTransform2d(64, 16, running_m=rm, running_var=rv)
    assert b.running_mean is rm and b.running_variance is rv


@pytest.mark.parametrize("components", [(), ("bw", "bw"), ("ln",), ("bw", "iw", "xx"), []])
def test_bad_components_are_refused(components):
    import dwt_b200
    with pytest.raises(ValueError, match="components must be a non-empty subset"):
        dwt_b200.SwitchableWTransform2d(64, 16, components)


def test_cpu_tensors_and_bad_inputs_are_refused():
    import dwt_b200
    from dwt_b200 import functional as F
    m = dwt_b200.SwitchableWTransform2d(64, 16)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(torch.zeros(2, 64, 16, 16))
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        F.switchable_whiten(torch.zeros(2, 64, 16, 16), torch.tensor(SWA), group_size=16, training_stats=True, eps=1e-3,
                            momentum=0.1, update_running=False, running=(m.running_mean, m.running_variance))
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(2, 64, 8))
    with pytest.raises(ValueError, match="expected number of channels divisible by group_size"):
        dwt_b200.SwitchableWTransform2d(48, 32)(torch.zeros(2, 48, 16, 16))


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _fp(v):
    return None if v is None else ctypes.c_void_p(v)


def _sw_fwd(lib, N=8, C=128, HW=3136, gs=64, mode=0, x=_FAKE, y=_FAKE, mix=_FAKE, save_w=_FAKE, save_stats=_FAKE,
            running=_FAKE, update=1, ws_bytes=1 << 40):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_switch_fwd(_fp(x), _fp(y), N, C, HW, gs, mode, 1e-3, 0.1, update, _fp(running), _fp(running),
                                     _fp(mix), p, _fp(save_w), _fp(save_stats), p, ws_bytes, None)


def _sw_bwd(lib, N=8, C=128, HW=3136, gs=64, mode=0, x=_FAKE, y=_FAKE, mix=_FAKE, save_w=_FAKE, save_stats=_FAKE,
            running=_FAKE, update=1, ws_bytes=1 << 40):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_switch_bwd(_fp(x), p, _fp(y), N, C, HW, gs, mode, 1e-3, _fp(mix), p, _fp(save_w), _fp(save_stats),
                                     None, p, ws_bytes, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


_SW = b"switchable whitening is built for the tensor-core kernels only"


@pytest.mark.parametrize("call", [_sw_fwd, _sw_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(gs=1), -4, _SW), (dict(gs=2), -4, _SW), (dict(gs=4), -4, _SW), (dict(gs=128), -4, _SW),
    (dict(C=96, gs=24), -4, _SW), (dict(C=96, gs=64), -4, _SW),
    (dict(HW=196), -4, _SW), (dict(HW=252), -4, _SW),                       # HW < 256
    (dict(HW=258), -4, _SW), (dict(HW=258, mode=0x101), -4, _SW),           # HW % 4 != 0
    (dict(HW=260, mode=0x200), -4, _SW), (dict(HW=260, mode=0x201), -4, _SW),   # NCHW bf16: HW % 8 != 0
    (dict(N=65536, C=64, HW=256), -4, _SW), (dict(N=1024, C=256, HW=8192), -4, _SW),
    (dict(mode=0x2), -1, b"bad mode"), (dict(mode=0x400), -1, b"bad mode"), (dict(mode=0x3), -1, b"bad mode"),
    (dict(N=0), -1, b"empty tensor"), (dict(HW=0), -1, b"empty tensor"),
    (dict(x=None), -1, b"null pointer argument"), (dict(y=None), -1, b"null pointer argument"),
    (dict(mix=None), -1, b"null pointer argument"), (dict(save_w=None), -1, b"null pointer argument"),
    (dict(save_stats=None), -1, b"null pointer argument"),
    (dict(x=_FAKE + 4), -1, b"must be 16-byte aligned"), (dict(y=_FAKE + 8), -1, b"must be 16-byte aligned"),
    (dict(mix=_FAKE + 4), -1, b"must be 16-byte aligned"), (dict(mix=_FAKE + 8), -1, b"must be 16-byte aligned"),
    (dict(save_w=_FAKE + 4), -1, b"must be 16-byte aligned"), (dict(save_stats=_FAKE + 4), -1, b"must be 16-byte aligned"),
    (dict(mode=0x300, x=_FAKE + 8), -1, b"must be 16-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


@pytest.mark.parametrize("kw", [dict(mode=1), dict(mode=0, update=1)])
def test_missing_running_buffers_are_refused(lib, kw):
    assert _sw_fwd(lib, running=None, **kw) == -1
    assert b"running buffer is null" in lib.dwt_last_error()


@pytest.mark.parametrize("call", [_sw_fwd, _sw_bwd])
@pytest.mark.parametrize("kw", [dict(N=1, C=64, HW=256, gs=64), dict(N=3, C=96, HW=784, gs=32, mode=0x301),
                                dict(N=2, C=64, HW=1024, gs=8, mode=0x200), dict(N=2, C=64, HW=1024, gs=8, running=None, update=0)])
def test_small_batches_pass_every_check_up_to_the_workspace(lib, call, kw):
    need = lib.dwt_switch_workspace_bytes(kw["N"], kw["C"], kw["HW"], kw["gs"])
    assert need > lib.dwt_instance_workspace_bytes(kw["N"], kw["C"], kw["HW"], kw["gs"]) > 0
    assert call(lib, ws_bytes=need - 1, **kw) == -2
    assert b"workspace too small" in lib.dwt_last_error()


def test_workspace_query(lib):
    assert lib.dwt_switch_workspace_bytes(8, 128, 3136, 64) > 0
    for args in ((8, 128, 3136, 1), (8, 128, 3136, 2), (8, 128, 3136, 4), (8, 128, 196, 64), (0, 128, 3136, 64),
                 (8, 96, 3136, 64), (8, 128, 3136, 128), (65536, 64, 256, 64)):
        assert lib.dwt_switch_workspace_bytes(*args) == 0


def test_other_entry_points_keep_their_refusals(lib):
    p = ctypes.c_void_p(_FAKE)
    assert lib.dwt_whiten_fwd(p, p, 8, 128, 3136, 64, 5, 0, 1e-3, 0.1, 0, None, None, None, None, None, None, 0, p, p, p,
                              1 << 40, None) == -1
    assert lib.dwt_last_error() == b"n_domains 5 outside [1,4]"
    assert lib.dwt_whiten_instance_fwd(p, p, 8, 128, 3136, 4, 0, 1e-3, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_last_error().startswith(b"instance whitening is built for the tensor-core kernels only")
    assert lib.dwt_whiten_instance_fwd(p, p, 8, 128, 3136, 64, 0x1, 1e-3, p, p, p, 1 << 40, None) == -1
    assert lib.dwt_last_error().startswith(b"bad flags")


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nswitchable whitening, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-52s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= BOUND and m <= MAX_BOUND, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def images(shape, dev, seed=0, cond=None, offset=2.0):
    """[N, C, H, W] float32 as test_instance_whitening.images: per image its own channel mixing (or covariances of
    condition number cond) and a per-image, per-channel mean of spread `offset`."""
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
    x = x + offset * torch.randn(n, c, 1, device=dev, generator=g) + 1.0
    return x.reshape(n, c, h, w).contiguous()


def grad(shape, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, device=dev, generator=g) + 0.5


def fresh_running(x, gs, seed=3):
    rm, rv = _running(x.double(), gs, seed)
    return rm.float().reshape(1, -1, 1, 1).contiguous(), rv.float().contiguous()


def run(x, dy, gs, mix, mode="train", running=None, eps=1e-3, momentum=0.1):
    """(y, dx, dmix, save_mean) of one forward + backward.  mode: train (batch statistics, running updated in place),
    eval (running), notrack (batch statistics, running untouched)."""
    from dwt_b200 import functional as F
    xg = x.detach().clone().requires_grad_(True)
    mg = torch.as_tensor(mix, dtype=torch.float32, device=x.device).clone().requires_grad_(True)
    if running is None:
        c = x.shape[1]
        running = (torch.zeros(1, c, 1, 1, device=x.device), torch.ones(c // gs, gs, gs, device=x.device))
    y = F.switchable_whiten(xg, mg, group_size=gs, training_stats=mode != "eval", eps=eps, momentum=momentum,
                            update_running=mode == "train", running=running)
    save_mean = y.grad_fn.saved_tensors[2].clone() if y.grad_fn is not None and hasattr(y.grad_fn, "saved_tensors") else None
    dx, dmix = torch.autograd.grad(y, (xg, mg), dy)
    return y.detach(), dx, dmix, save_mean


def against_float64(worst, label, x, dy, gs, mix, mode="train"):
    running = fresh_running(x, gs)
    old = (running[0].clone(), running[1].clone())
    y, dx, dmix, save_mean = run(x, dy, gs, mix, mode, running)
    xd, dyd = x.double(), dy.double()
    md = torch.tensor(mix, dtype=torch.float64, device=x.device)
    ref_run = None if mode != "eval" else (old[0].double(), old[1].double())
    f = R.sw_torch(xd, gs, md, running=ref_run)
    rdx, rdmix = R.closed_form_backward(xd, gs, dyd, md, running=ref_run)
    check(worst, label, "y", y, f["y"])
    check(worst, label, "dx", dx, rdx)
    check(worst, label, "dmix", dmix, rdmix)
    check(worst, label, "mean", save_mean, f["m"].reshape(x.shape[0], -1))
    if mode == "train":
        check(worst, label, "rmean", running[0].reshape(-1), 0.9 * old[0].reshape(-1).double() + 0.1 * f["mu_b"].reshape(-1))
        check(worst, label, "rcov", running[1], 0.9 * old[1].double() + 0.1 * f["cov_b"])
    else:
        assert torch.equal(running[0], old[0]) and torch.equal(running[1], old[1])


@gpu
@pytest.mark.parametrize("mix", ["swa", "swb"])
@pytest.mark.parametrize("shape, gs", [
    ((192, 256, 56, 56), 16), ((192, 256, 56, 56), 64), ((192, 64, 112, 112), 64),
    ((8, 64, 112, 112), 64),                                  # few long images: split across CTAs
    ((16, 64, 16, 16), 64), ((16, 64, 16, 16), 8),            # the smallest accepted HW
    ((8, 96, 32, 32), 32), ((8, 96, 32, 32), 16),             # a partial 64-channel super-block
])
def test_against_float64(dev, worst, shape, gs, mix):
    x = images(shape, dev, seed=gs)
    against_float64(worst, f"{list(shape)} gs {gs} {mix}", x, grad(shape, dev), gs, MIXES[mix])


@gpu
@pytest.mark.parametrize("mode", ["train", "eval", "notrack"])
@pytest.mark.parametrize("shape, gs", [((32, 128, 28, 28), 32), ((8, 96, 32, 32), 16)])
def test_modes_against_float64(dev, worst, shape, gs, mode):
    x = images(shape, dev, seed=5)
    against_float64(worst, f"{list(shape)} gs {gs} skew {mode}", x, grad(shape, dev), gs, MIXES["skew"], mode)


@gpu
@pytest.mark.parametrize("cond", [1.0, 10.0, 100.0, 1000.0])
@pytest.mark.parametrize("shape", [(16, 128, 28, 28), (8, 64, 56, 56)])
def test_conditioning_against_float64(dev, worst, cond, shape):
    x = images(shape, dev, seed=3, cond=cond)
    against_float64(worst, f"{list(shape)} gs 64 cond {cond:g} swa", x, grad(shape, dev), 64, SWA)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape, gs", [((64, 128, 28, 28), 64), ((16, 64, 16, 16), 16)])
def test_large_per_image_offsets_against_float64(dev, worst, shape, gs, mode):
    """Per-image means ~100 apart: the batch covariance is mostly cov(mu_n), formed without cancellation."""
    x = images(shape, dev, seed=12, offset=100.0)
    against_float64(worst, f"{list(shape)} gs {gs} offset 100 {mode}", x, grad(shape, dev), gs, MIXES["skew"], mode)


@gpu
@pytest.mark.parametrize("shape, gs", [((192, 256, 56, 56), 64), ((8, 64, 112, 112), 16), ((16, 96, 16, 16), 32)])
def test_channels_last_is_bitwise_nchw(dev, shape, gs):
    x, dy = images(shape, dev, seed=4), grad(shape, dev)
    y, dx, dmix, _ = run(x, dy, gs, SWB)
    cl = torch.channels_last
    yc, dxc, dmixc, _ = run(x.contiguous(memory_format=cl), dy.contiguous(memory_format=cl), gs, SWB)
    assert yc.is_contiguous(memory_format=cl) and dxc.is_contiguous(memory_format=cl)
    assert torch.equal(yc, y) and torch.equal(dxc, dx) and torch.equal(dmixc, dmix)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("shape, gs", [((32, 128, 56, 56), 64), ((16, 64, 28, 28), 16)])
def test_bf16_is_the_fp32_kernels_rounded(dev, layout, shape, gs):
    fmt = torch.channels_last if layout == "nhwc" else torch.contiguous_format
    x = images(shape, dev, seed=5).bfloat16().contiguous(memory_format=fmt)
    dy = grad(shape, dev).bfloat16().contiguous(memory_format=fmt)
    y, dx, dmix, _ = run(x, dy, gs, SWA)
    assert y.dtype == torch.bfloat16 and dx.dtype == torch.bfloat16 and dmix.dtype == torch.float32
    yf, dxf, dmixf, _ = run(x.float(), dy.float(), gs, SWA)
    assert torch.equal(y, yf.bfloat16()) and torch.equal(dx, dxf.bfloat16()) and torch.equal(dmix, dmixf)


@gpu
def test_bf16_nchw_off_the_bf16_rows_runs_the_fp32_kernels(dev):
    shape = (4, 64, 18, 18)                                   # HW = 324: a multiple of 4, not of 8
    x, dy = images(shape, dev, seed=6).bfloat16(), grad(shape, dev).bfloat16()
    y, dx, _, _ = run(x, dy, 16, SWA)
    yf, dxf, _, _ = run(x.float(), dy.float(), 16, SWA)
    assert y.dtype == torch.bfloat16 and torch.equal(y, yf.bfloat16()) and torch.equal(dx, dxf.bfloat16())


@gpu
def test_reruns_are_bit_identical(dev):
    for shape, gs in (((192, 256, 56, 56), 64), ((8, 64, 112, 112), 64)):
        x, dy = images(shape, dev, seed=7), grad(shape, dev)
        ra, rb = fresh_running(x, gs), fresh_running(x, gs)
        a, b = run(x, dy, gs, SWB, running=ra), run(x, dy, gs, SWB, running=rb)
        for u, v in zip(a + ra, b + rb):
            assert torch.equal(u, v)


@gpu
def test_cuda_graph_capture_and_replay(dev):
    import dwt_b200
    shape, gs = (16, 128, 28, 28), 32
    m = dwt_b200.SwitchableWTransform2d(128, gs, ("bw", "iw", "bn", "in")).to(dev)
    x, dy = images(shape, dev, seed=8), grad(shape, dev)
    sx, sdy = x.clone(), dy.clone()
    start = [t.clone() for t in (m.running_mean, m.running_variance)]

    def step():
        xg = sx.detach().requires_grad_(True)
        y = m(xg)
        dx, dmw, dvw = torch.autograd.grad(y, (xg, m.mean_weight, m.var_weight), sdy)
        return y.detach(), dx, dmw, dvw

    def reset():
        m.running_mean.copy_(start[0])
        m.running_variance.copy_(start[1])

    ref = step()
    ref_run = [m.running_mean.clone(), m.running_variance.clone()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                        # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        reset()
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(out, ref))
        assert torch.equal(m.running_mean, ref_run[0]) and torch.equal(m.running_variance, ref_run[1])
    sx.copy_(images(shape, dev, seed=9))
    reset()
    graph.replay()
    torch.cuda.synchronize()
    reset()
    fresh = step()
    assert all(torch.equal(a, b) for a, b in zip(out, fresh))


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_instance_mixture_agrees_with_instance_whitening(dev, mode):
    import dwt_b200
    shape, gs = (32, 128, 28, 28), 32
    x, dy = images(shape, dev, seed=13), grad(shape, dev)
    y, dx, _, _ = run(x, dy, gs, (0.0, 1.0, 0.0, 1.0, 0.0, 0.0), mode, fresh_running(x, gs))
    xg = x.clone().requires_grad_(True)
    yi = dwt_b200.InstanceWTransform2d(128, gs)(xg)
    (dxi,) = torch.autograd.grad(yi, xg, dy)
    for a, b in ((y, yi), (dx, dxi)):
        r, m = rel(a, b)
        assert r <= 1e-6 and m <= 1e-6, (r, m)


@gpu
def test_batch_mixture_agrees_with_the_domain_layer(dev, worst):
    import dwt_b200
    shape, gs = (32, 128, 28, 28), 32
    x, dy = images(shape, dev, seed=14), grad(shape, dev)
    w = dwt_b200.WTransform2d(128, gs).to(dev)
    w.running_variance.copy_(torch.eye(gs).expand(4, gs, gs))
    w.running_mean.normal_()
    running = (w.running_mean.clone(), w.running_variance.clone())
    y, dx, _, _ = run(x, dy, gs, (1.0, 0.0, 1.0, 0.0, 0.0, 0.0), "train", running)
    xg = x.clone().requires_grad_(True)
    yw = w(xg)
    (dxw,) = torch.autograd.grad(yw, xg, dy)
    nt = dwt_b200.WTransform2d(128, gs, track_running_stats=False).to(dev)
    xn = x.clone().requires_grad_(True)
    yn = nt(xn)
    (dxn,) = torch.autograd.grad(yn, xn, dy)
    check(worst, "batch mixture vs WTransform2d(track_running_stats=False)", "y", y, yn)
    check(worst, "batch mixture vs WTransform2d(track_running_stats=False)", "dx", dx, dxn)
    check(worst, "batch mixture vs WTransform2d", "rmean", running[0], w.running_mean)
    check(worst, "batch mixture vs WTransform2d", "rcov", running[1], w.running_variance)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_indefinite_group_sets_status_and_stays_local(dev, mode):
    """eps < 0 and a constant group of one image: with w_iw = 1 that (image, group)'s S = eps I is indefinite.  The
    forward keeps the NaN in that (image, group).  In eval so does the backward.  In training the batch terms of the
    backward carry it to that group's dx in every image, and to dmix; every other group stays finite."""
    from dwt_b200 import _native as nv
    shape, gs, eps, mix = (8, 128, 32, 32), 16, -1e-3, (0.5, 0.5, 0.0, 1.0, 0.0, 0.0)
    x, dy = images(shape, dev, seed=10), grad(shape, dev)
    running = fresh_running(x, gs)
    mode_r = "notrack" if mode == "train" else "eval"
    y0, dx0, _, _ = run(x, dy, gs, mix, mode_r, running, eps=eps)
    bad = x.clone()
    bad[6, 16:32] = 0.25                              # image 6, group 1 (super-block 0): zero covariance
    nv.clear_status(dev)
    y, dx, dmix, _ = run(bad, dy, gs, mix, mode_r, running, eps=eps)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    keep = torch.ones(shape[:2], dtype=torch.bool, device=dev)
    keep[6, 16:32] = False
    assert torch.isnan(y[6, 16:32]).all() and not torch.isnan(y[keep]).any()
    assert torch.isnan(dx[6, 16:32]).all()
    if mode == "eval":                                # nothing couples the images: the rest is the clean call's
        assert not torch.isnan(dx[keep]).any()
        assert torch.equal(y[:6], y0[:6]) and torch.equal(dx[:6], dx0[:6])
    else:
        other = torch.ones(shape[1], dtype=torch.bool, device=dev)
        other[16:32] = False
        assert torch.isnan(dx[:, 16:32]).all(), "the group's dx in every image"
        assert not torch.isnan(dx[:, other]).any(), "every other group"
    assert torch.isnan(dmix).any()
    run(x, dy, gs, mix, mode_r, running, eps=eps)
    assert nv.status(dev) == 0


@gpu
def test_non_finite_mix_gives_nan_and_status(dev):
    from dwt_b200 import _native as nv
    shape, gs = (8, 64, 32, 32), 16
    x, dy = images(shape, dev, seed=15), grad(shape, dev)
    running = fresh_running(x, gs)
    before = (running[0].clone(), running[1].clone())
    nv.clear_status(dev)
    y, _, _, _ = run(x, dy, gs, (0.5, 0.5, float("nan"), 0.5, 0.0, 0.0), "train", running)
    assert nv.status(dev) & nv.STATUS_NOT_PD and torch.isnan(y).all()
    nv.clear_status(dev)
    # the batch moments are finite: the EMA still runs (it does not depend on mix)
    assert not torch.equal(running[1], before[1]) and torch.isfinite(running[1]).all()
    y, _, _, _ = run(x, dy, gs, (float("inf"), 0.5, 0.5, 0.5, 0.0, 0.0), "eval", running)
    assert nv.status(dev) & nv.STATUS_NOT_PD and torch.isnan(y).all()
    nv.clear_status(dev)
    run(x, dy, gs, SWA, "train", running)
    assert nv.status(dev) == 0


@gpu
def test_non_finite_batch_moments_skip_the_ema(dev):
    from dwt_b200 import _native as nv
    shape, gs = (8, 64, 32, 32), 16
    x = images(shape, dev, seed=16)
    x[3, 5, 7, 9] = float("inf")                      # image 3, group 0: the batch moments of group 0 are not finite
    running = fresh_running(x[:2], gs)
    before = (running[0].clone(), running[1].clone())
    nv.clear_status(dev)
    run(x, grad(shape, dev), gs, SWA, "train", running)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    assert torch.equal(running[0][0, :16], before[0][0, :16]) and torch.equal(running[1][0], before[1][0])
    assert not torch.equal(running[1][1:], before[1][1:]) and torch.isfinite(running[1]).all()


@gpu
def test_training_step_decreases_the_loss(dev):
    import dwt_b200
    torch.manual_seed(0)
    sw = dwt_b200.SwitchableWTransform2d(64, 16, ("bw", "iw", "bn", "in"))
    net = torch.nn.Sequential(torch.nn.Conv2d(3, 64, 3, padding=1), sw, torch.nn.ReLU(),
                              torch.nn.Conv2d(64, 8, 3, padding=1)).to(dev)
    x = torch.randn(8, 3, 32, 32, device=dev)
    target = torch.randn(8, 8, 32, 32, device=dev)
    opt = torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9)
    losses = []
    for it in range(20):
        opt.zero_grad()
        loss = torch.nn.functional.mse_loss(net(x), target)
        loss.backward()
        if it == 0:
            for p in (sw.mean_weight, sw.var_weight):
                assert torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, p.grad
        opt.step()
        losses.append(float(loss.detach()))
    assert all(np.isfinite(losses)) and losses[-1] < 0.95 * losses[0], losses
    net.eval()
    with torch.no_grad():
        assert torch.isfinite(net(x)).all()
