"""Latent-domain whitening (LatentDomainWTransform2d, functional.latent_domain_whiten, dwt_whiten_latent_*).

CPU: the float64 closed-form backward (tests/support/ld_reference.py) -- dx and dweights -- against autograd through
torch.linalg.cholesky / inverse and against central finite differences, in train and eval, for 1, 3 and 8 domains under
softmax, one-hot and zero-mass weights; the module surface; the refusals of the C ABI (argument checks run before any
device call, so fake pointers do), and that the other entry points keep theirs.

GPU: the tensor-core kernels against the float64 reference -- y, dx and the running buffers within 1e-4 norm-wise,
dweights within 1e-3 -- at the production shapes, the launch edges, conditioning up to 1e3 and per-image mean offsets of
~100, in train, eval and untracked modes; against themselves bit for bit (layouts, dtypes, reruns, graphs, a zero-mass
domain); and at the weights where they reduce to WTransform2d on contiguous or gathered subsets of the batch.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import ld_reference as R  # noqa: E402

BOUND, DW_BOUND = 1e-4, 1e-3
gpu = pytest.mark.gpu


def _cpu_case(gs, seed, n=6, c=None, hw=(5, 6)):
    c = c or 2 * gs
    g = torch.Generator().manual_seed(seed)
    mix = torch.eye(c, dtype=torch.float64) + 0.3 * torch.randn(c, c, generator=g, dtype=torch.float64) / c ** 0.5
    x = torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, *hw, generator=g, dtype=torch.float64)) + 0.5
    x = x + torch.randn(n, c, 1, 1, generator=g, dtype=torch.float64)          # a different mean per image
    dout = torch.randn(x.shape, generator=g, dtype=torch.float64) + 0.2
    return x, dout


def _weights(kind, n, d, seed=0, dtype=torch.float64, device="cpu"):
    """softmax: random soft assignments; onehot: image i in domain i % d; zero: onehot with the last domain's column 0
    (its images moved to domain 0)."""
    g = torch.Generator(device=device).manual_seed(seed)
    if kind == "softmax":
        return torch.softmax(2.0 * torch.randn(n, d, generator=g, dtype=dtype, device=device), 1)
    w = torch.zeros(n, d, dtype=dtype, device=device)
    lab = torch.arange(n, device=device) % d
    if kind == "zero" and d > 1:
        lab[lab == d - 1] = 0
    w[torch.arange(n, device=device), lab] = 1.0
    return w


def _running(x, gs, w, seed):
    """Running buffers near the weighted statistics of x (positive definite, not equal to them)."""
    f = R.ld_torch(x, gs, w)
    g = torch.Generator(device=x.device).manual_seed(seed)
    c, d = x.shape[1], w.shape[1]
    eye = torch.eye(gs, dtype=x.dtype, device=x.device)
    rm = torch.stack([f["mu"][k].reshape(-1) if f["mu"][k] is not None else torch.zeros(c, dtype=x.dtype, device=x.device)
                      for k in range(d)])
    rm = rm + 0.1 * torch.randn(rm.shape, generator=g, device=x.device, dtype=x.dtype)
    rv = torch.stack([0.9 * f["sigma"][k] + 0.1 * eye if f["sigma"][k] is not None else eye.expand(c // gs, gs, gs)
                      for k in range(d)])
    return rm, rv


# =========================================================================== CPU: the float64 reference
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("kind", ["softmax", "onehot", "zero"])
@pytest.mark.parametrize("d", [1, 3, 8])
def test_closed_form_backward_matches_autograd(d, kind, train):
    gs = 8
    x, dout = _cpu_case(gs, d, n=9)
    w = _weights(kind, 9, d, seed=d)
    running = None if train else _running(x, gs, w, 1)
    xt, wt = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = R.ld_torch(xt, gs, wt, running=running)["y"]
    dx, dw = torch.autograd.grad(y, (xt, wt), dout)
    fx, fw = R.closed_form_backward(x, gs, dout, w, running=running)
    assert (fx - dx).abs().max() <= 1e-10 * dx.abs().max(), float((fx - dx).abs().max())
    assert (fw - dw).abs().max() <= 1e-10 * dw.abs().max(), (fw, dw)
    if kind == "zero" and d > 1:
        assert torch.equal(fw[:, -1], torch.zeros(9, dtype=fw.dtype))


@pytest.mark.parametrize("train", [True, False])
def test_closed_form_backward_matches_finite_differences(train):
    gs, d = 8, 3
    x, dout = _cpu_case(gs, 3)
    w = _weights("softmax", 6, d, seed=5)
    running = None if train else _running(x, gs, w, 2)
    dx, dw = R.closed_form_backward(x, gs, dout, w, running=running)
    loss = lambda t, ww: float((dout * R.ld_torch(t, gs, ww, running=running)["y"]).sum())
    h = 1e-6
    rng = np.random.default_rng(0)
    for _ in range(4):
        v = torch.tensor(rng.standard_normal(tuple(x.shape)))
        fd = (loss(x + h * v, w) - loss(x - h * v, w)) / (2 * h)
        assert abs(fd - float((dx * v).sum())) <= 1e-6 * max(abs(fd), 1.0)
    for n in range(6):
        for k in range(d):
            e = torch.zeros_like(w)
            e[n, k] = h
            fd = (loss(x, w + e) - loss(x, w - e)) / (2 * h)
            assert abs(fd - float(dw[n, k])) <= 1e-6 * max(abs(fd), 1.0), (n, k, fd, float(dw[n, k]))


def test_one_hot_weights_reduce_to_whitening_each_subset():
    gs = 8
    x, _ = _cpu_case(gs, 4, n=7)
    lab = torch.tensor([2, 0, 0, 1, 2, 0, 1])
    w = torch.nn.functional.one_hot(lab, 3).double()
    y = R.ld_torch(x, gs, w, eps=0.0)["y"]
    for d in range(3):
        yd = y[lab == d].reshape(-1, 2, gs, 30).permute(1, 2, 0, 3).reshape(2, gs, -1)    # each subset is white
        yc = yd - yd.mean(-1, keepdim=True)
        assert torch.allclose(yc @ yc.transpose(-1, -2) / yd.shape[-1], torch.eye(gs, dtype=x.dtype).expand(2, gs, gs), atol=1e-9)


# =========================================================================== CPU: module surface
def test_module_surface():
    import inspect
    import dwt_b200
    assert "LatentDomainWTransform2d" in dwt_b200.__all__
    assert list(inspect.signature(dwt_b200.LatentDomainWTransform2d.__init__).parameters) == [
        "self", "num_features", "group_size", "num_domains", "momentum", "track_running_stats", "eps"]
    m = dwt_b200.LatentDomainWTransform2d(64, 16, 3)
    assert (m.num_features, m.group_size, m.num_groups, m.num_domains, m.eps, m.momentum, m.track_running_stats) == (
        64, 16, 4, 3, 1e-3, 0.1, True)
    assert dwt_b200.LatentDomainWTransform2d(8, 16, 2).group_size == 8              # min(C, gs), as WTransform2d
    assert list(m.named_parameters()) == []
    assert sorted(m.state_dict()) == ["running_mean", "running_variance"]
    assert torch.equal(m.running_mean, torch.zeros(3, 64)) and torch.equal(m.running_variance, torch.ones(3, 4, 16, 16))
    assert "num_domains=3" in repr(m)
    m2 = dwt_b200.LatentDomainWTransform2d(64, 16, 3)
    m2.load_state_dict(m.state_dict())


def test_bad_inputs_and_cpu_tensors_are_refused():
    import dwt_b200
    from dwt_b200 import functional as F
    m = dwt_b200.LatentDomainWTransform2d(64, 16, 3)
    x = torch.zeros(4, 64, 16, 16)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(x, torch.full((4, 3), 1 / 3))
    with pytest.raises(ValueError, match=r"expected weights of shape \[4, 3\] \(got \[4, 2\]\)"):
        m(x, torch.ones(4, 2))
    with pytest.raises(ValueError, match=r"expected weights of shape \[4, 3\] \(got \[12\]\)"):
        m(x, torch.ones(12))
    with pytest.raises(ValueError, match=r"expected weights of shape \[4, 3\] \(got \[3, 3\]\)"):
        m(x, torch.ones(3, 3))
    with pytest.raises(TypeError, match="floating-point weights"):
        m(x, torch.ones(4, 3, dtype=torch.int64))
    with pytest.raises(ValueError, match="weights on x's device"):
        m(x, torch.ones(4, 3, device="meta"))
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(4, 64, 8), torch.ones(4, 3))
    with pytest.raises(ValueError, match="expected number of channels divisible by group_size"):
        dwt_b200.LatentDomainWTransform2d(48, 32, 2)(torch.zeros(2, 48, 16, 16), torch.ones(2, 2))
    with pytest.raises(ValueError, match="expected 64 channels"):
        m(torch.zeros(4, 32, 16, 16), torch.ones(4, 3))
    run = (m.running_mean, m.running_variance)
    with pytest.raises(ValueError, match=r"weights of shape \[N, n_domains\] with N = 4"):
        F.latent_domain_whiten(x, torch.ones(5, 3), group_size=16, training_stats=True, eps=1e-3, momentum=0.1,
                               update_running=False, running=run)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        F.latent_domain_whiten(x, torch.ones(4, 3), group_size=16, training_stats=True, eps=1e-3, momentum=0.1,
                               update_running=False, running=run)


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _fp(v):
    return None if v is None else ctypes.c_void_p(v)


def _ld_fwd(lib, N=8, C=128, HW=3136, gs=64, D=3, mode=0, x=_FAKE, y=_FAKE, w=_FAKE, save_w=_FAKE, save_stats=_FAKE,
            running=_FAKE, update=1, ws_bytes=1 << 40):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_latent_fwd(_fp(x), _fp(y), N, C, HW, gs, D, mode, 1e-3, 0.1, update, _fp(running), _fp(running),
                                     _fp(w), p, _fp(save_w), _fp(save_stats), p, ws_bytes, None)


def _ld_bwd(lib, N=8, C=128, HW=3136, gs=64, D=3, mode=0, x=_FAKE, y=_FAKE, w=_FAKE, save_w=_FAKE, save_stats=_FAKE,
            running=_FAKE, update=1, ws_bytes=1 << 40):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_latent_bwd(_fp(x), p, _fp(y), N, C, HW, gs, D, mode, 1e-3, _fp(w), p, _fp(save_w),
                                     _fp(save_stats), None, p, ws_bytes, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


_LD = b"latent-domain whitening is built for the tensor-core kernels only"


@pytest.mark.parametrize("call", [_ld_fwd, _ld_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(gs=1), -4, _LD), (dict(gs=2), -4, _LD), (dict(gs=4), -4, _LD), (dict(gs=128), -4, _LD),
    (dict(C=96, gs=24), -4, _LD), (dict(C=96, gs=64), -4, _LD),
    (dict(HW=196), -4, _LD), (dict(HW=252), -4, _LD),                       # HW < 256
    (dict(HW=258), -4, _LD), (dict(HW=258, mode=0x101), -4, _LD),           # HW % 4 != 0
    (dict(HW=260, mode=0x200), -4, _LD), (dict(HW=260, mode=0x201), -4, _LD),   # NCHW bf16: HW % 8 != 0
    (dict(N=65536, C=64, HW=256), -4, _LD), (dict(N=1024, C=256, HW=8192), -4, _LD),
    (dict(D=0), -1, b"n_domains 0 outside [1,8] (latent-domain whitening)"),
    (dict(D=9), -1, b"n_domains 9 outside [1,8] (latent-domain whitening)"),
    (dict(D=-1), -1, b"n_domains -1 outside [1,8]"),
    (dict(mode=0x2), -1, b"bad mode"), (dict(mode=0x400), -1, b"bad mode"), (dict(mode=0x3), -1, b"bad mode"),
    (dict(N=0), -1, b"empty tensor"), (dict(HW=0), -1, b"empty tensor"),
    (dict(x=None), -1, b"null pointer argument"), (dict(y=None), -1, b"null pointer argument"),
    (dict(w=None), -1, b"null pointer argument"), (dict(save_w=None), -1, b"null pointer argument"),
    (dict(save_stats=None), -1, b"null pointer argument"),
    (dict(x=_FAKE + 4), -1, b"must be 16-byte aligned (latent-domain whitening)"),
    (dict(y=_FAKE + 8), -1, b"must be 16-byte aligned (latent-domain whitening)"),
    (dict(w=_FAKE + 4), -1, b"must be 16-byte aligned"), (dict(w=_FAKE + 8), -1, b"must be 16-byte aligned"),
    (dict(save_w=_FAKE + 4), -1, b"must be 16-byte aligned"), (dict(save_stats=_FAKE + 4), -1, b"must be 16-byte aligned"),
    (dict(mode=0x300, x=_FAKE + 8), -1, b"must be 16-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


@pytest.mark.parametrize("kw", [dict(mode=1), dict(mode=0, update=1)])
def test_missing_running_buffers_are_refused(lib, kw):
    assert _ld_fwd(lib, running=None, **kw) == -1
    assert b"running buffer is null" in lib.dwt_last_error()


@pytest.mark.parametrize("call", [_ld_fwd, _ld_bwd])
@pytest.mark.parametrize("kw", [dict(N=1, C=64, HW=256, gs=64, D=1), dict(N=3, C=96, HW=784, gs=32, D=8, mode=0x301),
                                dict(N=2, C=64, HW=1024, gs=8, D=2, mode=0x200),
                                dict(N=2, C=64, HW=1024, gs=8, D=3, running=None, update=0)])
def test_small_batches_pass_every_check_up_to_the_workspace(lib, call, kw):
    need = lib.dwt_latent_workspace_bytes(kw["N"], kw["C"], kw["HW"], kw["gs"], kw["D"])
    assert need > lib.dwt_instance_workspace_bytes(kw["N"], kw["C"], kw["HW"], kw["gs"]) > 0
    assert call(lib, ws_bytes=need - 1, **kw) == -2
    assert b"workspace too small" in lib.dwt_last_error()


def test_workspace_query(lib):
    assert lib.dwt_latent_workspace_bytes(8, 128, 3136, 64, 3) > 0
    assert lib.dwt_latent_workspace_bytes(8, 128, 3136, 64, 8) > lib.dwt_latent_workspace_bytes(8, 128, 3136, 64, 1)
    for args in ((8, 128, 3136, 1, 3), (8, 128, 3136, 2, 3), (8, 128, 3136, 4, 3), (8, 128, 196, 64, 3),
                 (0, 128, 3136, 64, 3), (8, 96, 3136, 64, 3), (8, 128, 3136, 128, 3), (65536, 64, 256, 64, 3),
                 (8, 128, 3136, 64, 0), (8, 128, 3136, 64, 9)):
        assert lib.dwt_latent_workspace_bytes(*args) == 0
    lib.dwt_whiten_latent_fwd(None, None, 8, 128, 3136, 64, 3, 0, 1e-3, 0.1, 0, None, None, None, None, None, None, None,
                              0, None)
    err = lib.dwt_last_error()
    lib.dwt_latent_workspace_bytes(8, 128, 3136, 64, 9)
    assert lib.dwt_last_error() == err                                           # a size query leaves the text alone


def test_other_entry_points_keep_their_refusals(lib):
    p = ctypes.c_void_p(_FAKE)
    assert lib.dwt_whiten_fwd(p, p, 8, 128, 3136, 64, 5, 0, 1e-3, 0.1, 0, None, None, None, None, None, None, 0, p, p, p,
                              1 << 40, None) == -1
    assert lib.dwt_last_error() == b"n_domains 5 outside [1,4]"
    assert lib.dwt_workspace_bytes(8, 128, 3136, 64, 5) == 0
    assert lib.dwt_whiten_instance_fwd(p, p, 8, 128, 3136, 4, 0, 1e-3, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_last_error().startswith(b"instance whitening is built for the tensor-core kernels only")
    assert lib.dwt_whiten_instance_fwd(p, p, 8, 128, 3136, 64, 0x1, 1e-3, p, p, p, 1 << 40, None) == -1
    assert lib.dwt_last_error().startswith(b"bad flags")
    assert lib.dwt_whiten_switch_fwd(p, p, 8, 128, 3136, 4, 0, 1e-3, 0.1, 1, p, p, p, p, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_last_error().startswith(b"switchable whitening is built for the tensor-core kernels only")
    assert lib.dwt_whiten_switch_fwd(p, p, 8, 128, 3136, 64, 0, 1e-3, 0.1, 1, p, p, ctypes.c_void_p(_FAKE + 4), p, p, p, p,
                                     1 << 40, None) == -1
    assert b"(switchable whitening)" in lib.dwt_last_error()


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nlatent-domain whitening, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-56s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b, bound=BOUND):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= bound, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def images(shape, dev, seed=0, cond=None, offset=2.0):
    """[N, C, H, W] float32 as test_switchable_whitening.images: per image its own channel mixing (or covariances of
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


def fresh_running(x, gs, w, seed=3):
    rm, rv = _running(x.double(), gs, w.double(), seed)
    return rm.float().contiguous(), rv.float().contiguous()


def default_running(c, gs, d, dev):
    return torch.zeros(d, c, device=dev), torch.ones(d, c // gs, gs, gs, device=dev)


def run(x, dy, gs, w, mode="train", running=None, eps=1e-3, momentum=0.1, wgrad=True):
    """(y, dx, dweights) of one forward + backward.  mode: train (weighted statistics, running updated in place), eval
    (running), notrack (weighted statistics, running untouched).  wgrad False: weights without grad (labels), so the
    backward passes no dweights buffer and dweights is None."""
    from dwt_b200 import functional as F
    xg = x.detach().clone().requires_grad_(True)
    wg = w.detach().float().clone().requires_grad_(wgrad)
    if running is None:
        running = default_running(x.shape[1], gs, w.shape[1], x.device)
    y = F.latent_domain_whiten(xg, wg, group_size=gs, training_stats=mode != "eval", eps=eps, momentum=momentum,
                               update_running=mode == "train", running=running)
    if not wgrad:
        (dx,) = torch.autograd.grad(y, xg, dy)
        return y.detach(), dx, None
    dx, dw = torch.autograd.grad(y, (xg, wg), dy)
    return y.detach(), dx, dw


def against_float64(worst, label, x, dy, gs, w, mode="train"):
    running = fresh_running(x, gs, w)
    old = (running[0].clone(), running[1].clone())
    y, dx, dw = run(x, dy, gs, w, mode, running)
    xd, dyd, wd = x.double(), dy.double(), w.double()
    ref_run = None if mode != "eval" else (old[0].double(), old[1].double())
    f = R.ld_torch(xd, gs, wd, running=ref_run)
    rdx, rdw = R.closed_form_backward(xd, gs, dyd, wd, running=ref_run)
    check(worst, label, "y", y, f["y"])
    check(worst, label, "dx", dx, rdx)
    check(worst, label, "dweights", dw, rdw, DW_BOUND)
    if mode == "train":
        for k in range(w.shape[1]):
            check(worst, label, f"rmean{k}", running[0][k], 0.9 * old[0][k].double() + 0.1 * f["mu"][k].reshape(-1))
            check(worst, label, f"rcov{k}", running[1][k], 0.9 * old[1][k].double() + 0.1 * f["sigma"][k])
    else:
        assert torch.equal(running[0], old[0]) and torch.equal(running[1], old[1])


@gpu
@pytest.mark.parametrize("shape, gs, d", [
    ((192, 256, 56, 56), 64, 3), ((192, 256, 56, 56), 64, 8), ((192, 64, 112, 112), 16, 3),
    ((8, 64, 112, 112), 64, 2),                               # few long images: split across CTAs
    ((16, 64, 16, 16), 64, 3), ((16, 64, 16, 16), 8, 8),      # the smallest accepted HW
    ((8, 96, 32, 32), 32, 3), ((8, 96, 32, 32), 16, 1),       # a partial 64-channel super-block
])
def test_against_float64(dev, worst, shape, gs, d):
    x = images(shape, dev, seed=gs + d)
    w = _weights("softmax", shape[0], d, seed=d, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs {gs} D {d} softmax", x, grad(shape, dev), gs, w)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval", "notrack"])
@pytest.mark.parametrize("kind", ["softmax", "onehot"])
@pytest.mark.parametrize("shape, gs", [((32, 128, 28, 28), 32), ((8, 96, 32, 32), 16)])
def test_modes_against_float64(dev, worst, shape, gs, kind, mode):
    x = images(shape, dev, seed=5)
    w = _weights(kind, shape[0], 3, seed=2, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs {gs} D 3 {kind} {mode}", x, grad(shape, dev), gs, w, mode)


@gpu
@pytest.mark.parametrize("cond", [1.0, 10.0, 100.0, 1000.0])
def test_conditioning_against_float64(dev, worst, cond):
    shape = (16, 128, 28, 28)
    x = images(shape, dev, seed=3, cond=cond)
    w = _weights("softmax", shape[0], 3, seed=4, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs 64 D 3 cond {cond:g}", x, grad(shape, dev), 64, w)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape, gs", [((192, 128, 28, 28), 64), ((16, 64, 16, 16), 16)])
def test_large_per_image_offsets_against_float64(dev, worst, shape, gs, mode):
    """Per-image means ~100 apart: Sigma_d is mostly the weighted covariance of the image means.  At group size 64 the
    batch has 192 images: with about as many images per domain as channels per group (64 images, 3 domains) that
    covariance is close to singular (condition ~1e4), and dx's float32 error reaches 1.3e-4."""
    x = images(shape, dev, seed=12, offset=100.0)
    w = _weights("softmax", shape[0], 3, seed=6, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs {gs} D 3 offset 100 {mode}", x, grad(shape, dev), gs, w, mode)


def _wtransform(x, dy, gs, running, dev):
    """y, dx and the updated buffers of a WTransform2d in train mode on x (buffers copied from running)."""
    import dwt_b200
    m = dwt_b200.WTransform2d(x.shape[1], gs).to(dev)
    m.running_mean.copy_(running[0].reshape(m.running_mean.shape))
    m.running_variance.copy_(running[1].reshape(m.running_variance.shape))
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    (dx,) = torch.autograd.grad(y, xg, dy)
    return y.detach(), dx, m.running_mean.reshape(-1), m.running_variance


@gpu
def test_one_domain_of_unit_weights_agrees_with_wtransform(dev, worst):
    shape, gs = (32, 128, 28, 28), 32
    x, dy = images(shape, dev, seed=13), grad(shape, dev)
    w = torch.ones(shape[0], 1, device=dev)
    running = fresh_running(x, gs, w)
    yw, dxw, rmw, rvw = _wtransform(x, dy, gs, (running[0][0], running[1][0]), dev)
    y, dx, _ = run(x, dy, gs, w, "train", running)
    label = "D 1, unit weights vs WTransform2d"
    for name, a, b in (("y", y, yw), ("dx", dx, dxw), ("rmean", running[0][0], rmw), ("rcov", running[1][0], rvw)):
        check(worst, label, name, a, b)


@gpu
@pytest.mark.parametrize("layout", ["contiguous", "interleaved"])
def test_one_hot_weights_agree_with_wtransform_per_domain(dev, worst, layout):
    """contiguous: three equal slices (a DomainTripleNorm site); interleaved: uneven 100 / 60 / 32 labels in random order,
    against WTransform2d on each gathered subset."""
    shape, gs = (192, 128, 28, 28), 32
    x, dy = images(shape, dev, seed=17), grad(shape, dev)
    if layout == "contiguous":
        lab = torch.arange(192, device=dev) // 64
    else:
        lab = torch.cat([torch.full((n,), d) for d, n in enumerate((100, 60, 32))])
        lab = lab[torch.randperm(192, generator=torch.Generator().manual_seed(0))].to(dev)
    w = torch.nn.functional.one_hot(lab, 3).float()
    running = fresh_running(x, gs, w)
    start = (running[0].clone(), running[1].clone())
    y, dx, _ = run(x, dy, gs, w, "train", running)
    for d in range(3):
        idx = (lab == d).nonzero().squeeze(1)
        yw, dxw, rmw, rvw = _wtransform(x[idx], dy[idx], gs, (start[0][d], start[1][d]), dev)
        label = f"one-hot {layout} vs WTransform2d, domain {d}"
        for name, a, b in (("y", y[idx], yw), ("dx", dx[idx], dxw), ("rmean", running[0][d], rmw),
                           ("rcov", running[1][d], rvw)):
            check(worst, label, name, a, b)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_zero_mass_domain_is_bitwise_absent(dev, mode):
    from dwt_b200 import _native as nv
    shape, gs = (24, 128, 28, 28), 32
    x, dy = images(shape, dev, seed=18), grad(shape, dev)
    w3 = _weights("softmax", shape[0], 3, seed=7, dtype=torch.float32, device=dev)
    w4 = torch.cat([w3[:, :1], torch.zeros(shape[0], 1, device=dev), w3[:, 1:]], 1)
    r3 = fresh_running(x, gs, w3)
    r4 = (torch.cat([r3[0][:1], torch.randn(1, 128, device=dev), r3[0][1:]]),
          torch.cat([r3[1][:1], torch.eye(gs, device=dev).expand(1, 4, gs, gs) * 2, r3[1][1:]]))
    before = (r4[0][1].clone(), r4[1][1].clone())
    nv.clear_status(dev)
    y3, dx3, dw3 = run(x, dy, gs, w3, mode, r3)
    y4, dx4, dw4 = run(x, dy, gs, w4, mode, r4)
    assert nv.status(dev) == 0, "a zero-mass domain is skipped, not an error"
    assert torch.equal(y3, y4) and torch.equal(dx3, dx4)
    assert torch.equal(dw4[:, 1], torch.zeros_like(dw4[:, 1])) and torch.equal(dw4[:, [0, 2, 3]], dw3)
    assert torch.equal(r4[0][1], before[0]) and torch.equal(r4[1][1], before[1])
    assert torch.equal(r4[0][[0, 2, 3]], r3[0]) and torch.equal(r4[1][[0, 2, 3]], r3[1])


@gpu
def test_labels_without_grad_pass_no_dweights(dev):
    """Weights that do not require grad (plain one-hot labels): the backward passes dweights = NULL and skips its sum;
    y, dx and the running buffers are bit for bit those of the call that returns dweights."""
    shape, gs = (48, 128, 28, 28), 32
    x, dy = images(shape, dev, seed=19), grad(shape, dev)
    lab = torch.randint(0, 3, (shape[0],), generator=torch.Generator().manual_seed(1)).to(dev)
    w = torch.nn.functional.one_hot(lab, 3).float()
    ra, rb = fresh_running(x, gs, w), fresh_running(x, gs, w)
    y, dx, dw = run(x, dy, gs, w, "train", ra)
    yl, dxl, dwl = run(x, dy, gs, w, "train", rb, wgrad=False)
    assert dw is not None and dwl is None
    assert torch.equal(y, yl) and torch.equal(dx, dxl)
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1])


@gpu
def test_negative_mass_domain_sets_status_and_skips_its_ema(dev):
    """Domain 2's weights are -1 (s_2 = -4 < 0): W_2 is NaN, the status is set and domain 2's buffers stay untouched bit
    for bit.  Its images read NaN; every image whose weight on it is exactly 0 stays finite in y and dx, and the other
    domains' buffers are updated."""
    from dwt_b200 import _native as nv
    shape, gs = (12, 64, 32, 32), 16
    x, dy = images(shape, dev, seed=20), grad(shape, dev)
    lab = torch.arange(12, device=dev) % 3
    w = torch.nn.functional.one_hot(lab, 3).float()
    w[:, 2] = -w[:, 2]
    running = fresh_running(x, gs, torch.nn.functional.one_hot(lab, 3).float())
    before = (running[0].clone(), running[1].clone())
    nv.clear_status(dev)
    y, dx, dw = run(x, dy, gs, w, "train", running)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    bad = lab == 2
    assert torch.isnan(y[bad]).all() and torch.isnan(dx[bad]).all()
    assert torch.isfinite(y[~bad]).all() and torch.isfinite(dx[~bad]).all() and torch.isfinite(dw[~bad][:, :2]).all()
    assert torch.equal(running[0][2], before[0][2]) and torch.equal(running[1][2], before[1][2])
    assert not torch.equal(running[1][:2], before[1][:2]) and torch.isfinite(running[0]).all() and torch.isfinite(running[1]).all()


@gpu
@pytest.mark.parametrize("case", ["zero_row_train", "zero_row_eval", "negative_weight_eval"])
def test_image_without_a_positive_mix_sets_status_and_stays_local(dev, case):
    """Image 4 has no weight on any domain (A_4 = 0), or -1 on its own domain (eval: the domain's statistics are the
    running buffers and s_1 = 2 > 0, so A_4 = -W_1 has a negative diagonal).  A_4 is NaN in every group and the status is
    set; every other image is finite in y and dx, and train still updates every domain's buffers."""
    from dwt_b200 import _native as nv
    shape, gs = (12, 64, 32, 32), 16
    x, dy = images(shape, dev, seed=21), grad(shape, dev)
    lab = torch.arange(12, device=dev) % 3
    onehot = torch.nn.functional.one_hot(lab, 3).float()
    w = onehot.clone()
    w[4] = 0.0
    if case.startswith("negative"):
        w[4, lab[4]] = -1.0
    mode = "eval" if case.endswith("eval") else "train"
    running = fresh_running(x, gs, onehot)
    before = (running[0].clone(), running[1].clone())
    nv.clear_status(dev)
    y, dx, _ = run(x, dy, gs, w, mode, running)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    other = torch.arange(12, device=dev) != 4
    assert torch.isnan(y[4]).all() and torch.isnan(dx[4]).all()
    assert torch.isfinite(y[other]).all() and torch.isfinite(dx[other]).all()
    if mode == "train":
        assert all(not torch.equal(running[1][k], before[1][k]) for k in range(3)) and torch.isfinite(running[1]).all()
    else:
        assert torch.equal(running[0], before[0]) and torch.equal(running[1], before[1])
    run(x, dy, gs, onehot, mode, running)
    assert nv.status(dev) == 0


@gpu
def test_nan_weight_sets_status_and_stays_in_its_domain(dev):
    from dwt_b200 import _native as nv
    shape, gs = (12, 64, 32, 32), 16
    x, dy = images(shape, dev, seed=10), grad(shape, dev)
    lab = torch.arange(12, device=dev) % 3
    w = torch.nn.functional.one_hot(lab, 3).float()
    w[3, 0] = float("nan")                            # image 3 is in domain 0
    running = fresh_running(x, gs, torch.nn.functional.one_hot(lab, 3).float())
    before = (running[0].clone(), running[1].clone())
    nv.clear_status(dev)
    y, dx, dw = run(x, dy, gs, w, "train", running)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    bad = lab == 0
    assert torch.isnan(y[bad]).all() and torch.isnan(dx[bad]).all()
    assert torch.isfinite(y[~bad]).all() and torch.isfinite(dx[~bad]).all() and torch.isfinite(dw[~bad][:, 1:]).all()
    assert torch.equal(running[0][0], before[0][0]) and torch.equal(running[1][0], before[1][0])
    assert not torch.equal(running[1][1:], before[1][1:]) and torch.isfinite(running[1]).all()
    run(x, dy, gs, torch.nn.functional.one_hot(lab, 3).float(), "train", running)
    assert nv.status(dev) == 0


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_indefinite_group_sets_status_and_stays_local(dev, mode):
    """eps < 0 and a group that is constant over every image of domain 1: S_1 = eps I is indefinite there, W_1 is NaN in
    that group, and only domain 1's images read NaN, only in that group (one-hot weights couple nothing else)."""
    from dwt_b200 import _native as nv
    shape, gs, eps = (12, 64, 32, 32), 16, -1e-3
    x, dy = images(shape, dev, seed=11), grad(shape, dev)
    lab = torch.arange(12, device=dev) % 3
    w = torch.nn.functional.one_hot(lab, 3).float()
    x[lab == 1, 16:32] = 0.25
    running = fresh_running(images(shape, dev, seed=11), gs, w)
    if mode == "eval":
        running[1][1, 1] = 0.0                        # domain 1, group 1: zero covariance
    nv.clear_status(dev)
    y, dx, _ = run(x, dy, gs, w, "notrack" if mode == "train" else "eval", running, eps=eps)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    keep = torch.ones(shape[:2], dtype=torch.bool, device=dev)
    keep[lab == 1, 16:32] = False
    assert torch.isnan(y[lab == 1][:, 16:32]).all() and not torch.isnan(y[keep]).any()
    assert torch.isnan(dx[lab == 1][:, 16:32]).all() and not torch.isnan(dx[keep]).any()


@gpu
@pytest.mark.parametrize("shape, gs, d", [((192, 256, 56, 56), 64, 3), ((8, 64, 112, 112), 16, 8), ((16, 96, 16, 16), 32, 2)])
def test_channels_last_is_bitwise_nchw(dev, shape, gs, d):
    x, dy = images(shape, dev, seed=4), grad(shape, dev)
    w = _weights("softmax", shape[0], d, seed=1, dtype=torch.float32, device=dev)
    y, dx, dw = run(x, dy, gs, w)
    cl = torch.channels_last
    yc, dxc, dwc = run(x.contiguous(memory_format=cl), dy.contiguous(memory_format=cl), gs, w)
    assert yc.is_contiguous(memory_format=cl) and dxc.is_contiguous(memory_format=cl)
    assert torch.equal(yc, y) and torch.equal(dxc, dx) and torch.equal(dwc, dw)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("shape, gs", [((32, 128, 56, 56), 64), ((16, 64, 28, 28), 16)])
def test_bf16_is_the_fp32_kernels_rounded(dev, layout, shape, gs):
    fmt = torch.channels_last if layout == "nhwc" else torch.contiguous_format
    x = images(shape, dev, seed=5).bfloat16().contiguous(memory_format=fmt)
    dy = grad(shape, dev).bfloat16().contiguous(memory_format=fmt)
    w = _weights("softmax", shape[0], 3, seed=2, dtype=torch.float32, device=dev)
    y, dx, dw = run(x, dy, gs, w)
    assert y.dtype == torch.bfloat16 and dx.dtype == torch.bfloat16 and dw.dtype == torch.float32
    yf, dxf, dwf = run(x.float(), dy.float(), gs, w)
    assert torch.equal(y, yf.bfloat16()) and torch.equal(dx, dxf.bfloat16()) and torch.equal(dw, dwf)


@gpu
def test_reruns_are_bit_identical(dev):
    for shape, gs, d in (((192, 256, 56, 56), 64, 8), ((8, 64, 112, 112), 64, 3)):
        x, dy = images(shape, dev, seed=7), grad(shape, dev)
        w = _weights("softmax", shape[0], d, seed=3, dtype=torch.float32, device=dev)
        ra, rb = fresh_running(x, gs, w), fresh_running(x, gs, w)
        a, b = run(x, dy, gs, w, running=ra), run(x, dy, gs, w, running=rb)
        for u, v in zip(a + ra, b + rb):
            assert torch.equal(u, v)


@gpu
def test_cuda_graph_capture_and_replay(dev):
    import dwt_b200
    shape, gs = (16, 128, 28, 28), 32
    m = dwt_b200.LatentDomainWTransform2d(128, gs, 3).to(dev)
    x, dy = images(shape, dev, seed=8), grad(shape, dev)
    logits = torch.randn(shape[0], 3, device=dev)
    sx, sdy, sl = x.clone(), dy.clone(), logits.clone()
    start = [t.clone() for t in (m.running_mean, m.running_variance)]

    def step():
        xg = sx.detach().requires_grad_(True)
        lg = sl.detach().requires_grad_(True)
        y = m(xg, torch.softmax(lg, 1))
        dx, dl = torch.autograd.grad(y, (xg, lg), sdy)
        return y.detach(), dx, dl

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
def test_training_step_through_a_softmax_branch_decreases_the_loss(dev):
    import dwt_b200
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(3, 64, 3, padding=1)
    branch = torch.nn.Sequential(torch.nn.AdaptiveAvgPool2d(1), torch.nn.Flatten(), torch.nn.Linear(3, 3))
    ld = dwt_b200.LatentDomainWTransform2d(64, 16, 3)
    head = torch.nn.Conv2d(64, 8, 3, padding=1)
    mods = torch.nn.ModuleList([conv, branch, ld, head]).to(dev)
    x = torch.randn(8, 3, 32, 32, device=dev)
    x[:4] += 1.5                                      # two latent sources
    target = torch.randn(8, 8, 32, 32, device=dev)
    opt = torch.optim.SGD(mods.parameters(), lr=0.05, momentum=0.9)
    losses = []
    for it in range(20):
        opt.zero_grad()
        w = torch.softmax(branch(x), 1)
        loss = torch.nn.functional.mse_loss(head(torch.relu(ld(conv(x), w))), target)
        loss.backward()
        if it == 0:
            g = branch[2].weight.grad
            assert torch.isfinite(g).all() and g.abs().max() > 0, g
        opt.step()
        losses.append(float(loss.detach()))
    assert all(np.isfinite(losses)) and losses[-1] < 0.95 * losses[0], losses
    mods.eval()
    with torch.no_grad():
        assert torch.isfinite(head(ld(conv(x), torch.softmax(branch(x), 1)))).all()
