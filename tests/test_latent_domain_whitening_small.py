"""Latent-domain whitening at group sizes 1, 2, 4 (dwt_whiten_latent_small_*, functional.latent_domain_whiten's route for
group sizes up to 4, LatentDomainWTransform2d at ResNet-50-DWT's and the digits LeNet's whitening sites).

CPU: the float64 closed-form backward (tests/support/ld_reference.py) against autograd at group sizes 1, 2, 4 for 1, 3
and 8 domains under softmax, one-hot and zero-mass weights, in train and eval, at H*W = 1 and 7x7; the refusals of the new
C ABI pair (argument checks run before any device call, so fake pointers do) and its workspace query; the module's
buffers at group size 4.

GPU: the register-resident kernels against the float64 reference -- y, dx and every domain's running buffers within 1e-4
norm-wise, dweights within 1e-3 -- at the model sites and the launch edges, under conditioning up to 1e3 and per-image
mean offsets of ~100, in train, eval and untracked modes and both layouts; against WTransform2d where the layer reduces to
it; against themselves bit for bit (bf16, reruns, graphs, labels without a gradient); and every edge rule of the header.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import ld_reference as R  # noqa: E402

BOUND, DW_BOUND, WT_BOUND = 1e-4, 1e-3, 1e-5
gpu = pytest.mark.gpu


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
@pytest.mark.parametrize("hw", [(1, 1), (7, 7)])
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("kind", ["softmax", "onehot", "zero"])
@pytest.mark.parametrize("d", [1, 3, 8])
@pytest.mark.parametrize("gs", [1, 2, 4])
def test_closed_form_backward_matches_autograd(gs, d, kind, train, hw):
    n, c = 11, 2 * gs
    g = torch.Generator().manual_seed(100 * gs + d)
    mix = torch.eye(c, dtype=torch.float64) + 0.3 * torch.randn(c, c, generator=g, dtype=torch.float64) / c ** 0.5
    x = torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, *hw, generator=g, dtype=torch.float64)) + 0.5
    x = x + torch.randn(n, c, 1, 1, generator=g, dtype=torch.float64)        # a different mean per image
    dout = torch.randn(x.shape, generator=g, dtype=torch.float64) + 0.2
    w = _weights(kind, n, d, seed=d)
    running = None if train else _running(x, gs, w, 1)
    xt, wt = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = R.ld_torch(xt, gs, wt, running=running)["y"]
    dx, dw = torch.autograd.grad(y, (xt, wt), dout)
    fx, fw = R.closed_form_backward(x, gs, dout, w, running=running)
    assert (fx - dx).abs().max() <= 1e-9 * dx.abs().max(), float((fx - dx).abs().max())
    assert (fw - dw).abs().max() <= 1e-9 * dw.abs().max(), (fw, dw)
    if kind == "zero" and d > 1:
        assert torch.equal(fw[:, -1], torch.zeros(n, dtype=fw.dtype))


# =========================================================================== CPU: module surface
def test_module_buffers_at_group_size_4_and_cpu_tensors_are_refused():
    import dwt_b200
    from dwt_b200 import functional as F
    m = dwt_b200.LatentDomainWTransform2d(64, 4, 3)
    assert (m.group_size, m.num_groups) == (4, 16)
    assert torch.equal(m.running_mean, torch.zeros(3, 64)) and torch.equal(m.running_variance, torch.ones(3, 16, 4, 4))
    assert dwt_b200.LatentDomainWTransform2d(2, 4, 3).group_size == 2                # min(C, gs), as WTransform2d
    x = torch.zeros(4, 64, 7, 7)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(x, torch.full((4, 3), 1 / 3))
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        F.latent_domain_whiten(x, torch.ones(4, 3), group_size=4, training_stats=True, eps=1e-3, momentum=0.1,
                               update_running=False, running=(m.running_mean, m.running_variance))


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _fp(v):
    return None if v is None else ctypes.c_void_p(v)


def _lds_fwd(lib, N=8, C=64, HW=3136, gs=4, D=3, mode=0, x=_FAKE, y=_FAKE, w=_FAKE, save_mean=_FAKE, save_w=_FAKE,
             save_stats=_FAKE, running=_FAKE, update=1, ws_bytes=1 << 40):
    return lib.dwt_whiten_latent_small_fwd(_fp(x), _fp(y), N, C, HW, gs, D, mode, 1e-3, 0.1, update, _fp(running),
                                           _fp(running), _fp(w), _fp(save_mean), _fp(save_w), _fp(save_stats),
                                           ctypes.c_void_p(_FAKE), ws_bytes, None)


def _lds_bwd(lib, N=8, C=64, HW=3136, gs=4, D=3, mode=0, x=_FAKE, y=_FAKE, w=_FAKE, save_mean=_FAKE, save_w=_FAKE,
             save_stats=_FAKE, running=_FAKE, update=1, ws_bytes=1 << 40):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_latent_small_bwd(_fp(x), p, _fp(y), N, C, HW, gs, D, mode, 1e-3, _fp(w), _fp(save_mean),
                                           _fp(save_w), _fp(save_stats), None, p, ws_bytes, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


_LDS = b"latent-domain whitening at group sizes 1, 2, 4"


@pytest.mark.parametrize("call", [_lds_fwd, _lds_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(gs=3, C=96), -4, _LDS), (dict(gs=8), -4, _LDS), (dict(gs=128, C=128), -4, _LDS), (dict(gs=0), -4, _LDS),
    (dict(C=6, gs=4), -4, _LDS + b" needs group_size 1, 2 or 4 dividing C"),
    (dict(C=6, gs=2, mode=0x100), -4, _LDS + b" runs channels-last at C % 4 == 0 only"),
    (dict(C=6, gs=2, mode=0x101), -4, b"channels-last at C % 4 == 0 only"),
    (dict(HW=49, mode=0x200), -4, _LDS + b" runs NCHW bf16 at HW % 4 == 0 only"),
    (dict(N=1024, C=256, HW=8192), -4, _LDS + b" needs N*C*HW < 2^31"),
    (dict(N=2, C=1 << 20, HW=1 << 10), -4, b"N*C*HW < 2^31"),
    (dict(D=0), -1, b"n_domains 0 outside [1,8] (latent-domain whitening)"),
    (dict(D=9), -1, b"n_domains 9 outside [1,8] (latent-domain whitening)"),
    (dict(mode=0x2), -1, b"bad mode"), (dict(mode=0x400), -1, b"bad mode"),
    (dict(N=0), -1, b"empty tensor"), (dict(C=0), -1, b"empty tensor"), (dict(HW=0), -1, b"empty tensor"),
    (dict(x=None), -1, b"null pointer argument"), (dict(y=None), -1, b"null pointer argument"),
    (dict(w=None), -1, b"null pointer argument"), (dict(save_mean=None), -1, b"null pointer argument"),
    (dict(save_w=None), -1, b"null pointer argument"), (dict(save_stats=None), -1, b"null pointer argument"),
    (dict(x=_FAKE + 4), -1, b"activation tensors must be 16-byte aligned (latent-domain whitening)"),
    (dict(y=_FAKE + 8), -1, b"activation tensors must be 16-byte aligned"),
    (dict(mode=0x200, x=_FAKE + 4), -1, b"activation tensors must be 8-byte aligned"),
    (dict(w=_FAKE + 8), -1, b"weights, save_w and save_stats must be 16-byte"),
    (dict(save_w=_FAKE + 4), -1, b"must be 16-byte"), (dict(save_stats=_FAKE + 8), -1, b"must be 16-byte"),
    (dict(save_mean=_FAKE + 2), -1, b"save_mean 4-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


@pytest.mark.parametrize("kw", [dict(mode=1), dict(mode=0, update=1), dict(mode=0x301)])
def test_missing_running_buffers_are_refused(lib, kw):
    assert _lds_fwd(lib, running=None, **kw) == -1
    assert b"running buffer is null" in lib.dwt_last_error()


@pytest.mark.parametrize("call", [_lds_fwd, _lds_bwd])
@pytest.mark.parametrize("kw", [dict(N=1, C=4, HW=1, gs=4, D=1), dict(N=3, C=6, HW=49, gs=2, D=8),
                                dict(N=2, C=64, HW=3136, gs=1, D=2, mode=0x301),
                                dict(N=2, C=64, HW=3136, gs=4, D=3, mode=0x200, x=_FAKE + 8),
                                dict(N=2, C=48, HW=196, gs=4, D=3, running=None, update=0)])
def test_small_batches_pass_every_check_up_to_the_workspace(lib, call, kw):
    # the query sizes the larger of the two layouts' plans, so only a workspace short of every plan is refused for sure
    assert lib.dwt_latent_small_workspace_bytes(kw["N"], kw["C"], kw["HW"], kw["gs"], kw["D"]) > 256
    assert call(lib, ws_bytes=256, **kw) == -2
    assert b"workspace too small" in lib.dwt_last_error()


def test_workspace_query(lib):
    q = lib.dwt_latent_small_workspace_bytes
    assert q(192, 64, 12544, 4, 3) > 0 and q(1, 1, 1, 1, 1) > 0
    assert q(192, 256, 3136, 4, 8) > q(192, 256, 3136, 4, 1)
    assert q(8, 6, 49, 2, 3) > 0                                     # channels-last refused, NCHW taken
    for args in ((8, 64, 3136, 3, 3), (8, 64, 3136, 8, 3), (8, 64, 3136, 128, 3), (8, 6, 3136, 4, 3),
                 (0, 64, 3136, 4, 3), (8, 64, 0, 4, 3), (1024, 256, 8192, 4, 3), (8, 64, 3136, 4, 0),
                 (8, 64, 3136, 4, 9)):
        assert q(*args) == 0, args
    _lds_fwd(lib, gs=3, C=96)
    err = lib.dwt_last_error()
    q(8, 64, 3136, 4, 9)
    assert lib.dwt_last_error() == err                                           # a size query leaves the text alone


def test_tensor_core_entry_points_keep_their_refusals(lib):
    p = ctypes.c_void_p(_FAKE)
    assert lib.dwt_whiten_latent_fwd(p, p, 8, 64, 3136, 4, 3, 0, 1e-3, 0.1, 1, p, p, p, p, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_last_error().startswith(b"latent-domain whitening is built for the tensor-core kernels only")
    assert lib.dwt_latent_workspace_bytes(8, 64, 3136, 4, 3) == 0


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nlatent-domain whitening at group sizes 1, 2, 4, worst errors (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-60s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b, bound=BOUND):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= bound, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def images(shape, dev, gs, seed=0, cond=None, offset=2.0):
    """[N, C, H, W] float32: per image and group its own channel mixing (or, cond given, a covariance of condition number
    cond in a random basis) and a per-image, per-channel mean of spread `offset`."""
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    z = torch.randn(n, c // gs, gs, h * w, device=dev, generator=g)
    if cond is None:
        mix = torch.eye(gs, device=dev) + 0.5 * torch.randn(n, c // gs, gs, gs, device=dev, generator=g) / gs ** 0.5
    else:
        q, _ = torch.linalg.qr(torch.randn(n, c // gs, gs, gs, device=dev, generator=g, dtype=torch.float64))
        mix = (q * torch.logspace(0, -0.5 * np.log10(cond), gs, device=dev, dtype=torch.float64)).float()
    x = (mix @ z).reshape(n, c, h * w)
    x = x + offset * torch.randn(n, c, 1, device=dev, generator=g) + 1.0
    return x.reshape(n, c, h, w).contiguous()


def grad(shape, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, device=dev, generator=g) + 0.5


def fresh_running(x, gs, w, seed=3):
    rm, rv = _running(x.double(), gs, w.double(), seed)
    return rm.float().contiguous(), rv.float().contiguous()


def run(x, dy, gs, w, mode="train", running=None, eps=1e-3, momentum=0.1, wgrad=True):
    """(y, dx, dweights) of one forward + backward.  mode: train (weighted statistics, running updated in place), eval
    (running), notrack (weighted statistics, running untouched).  wgrad False: weights without grad, so the backward
    passes no dweights buffer and dweights is None."""
    from dwt_b200 import functional as F
    xg = x.detach().clone().requires_grad_(True)
    wg = w.detach().float().clone().requires_grad_(wgrad)
    if running is None:
        running = (torch.zeros(w.shape[1], x.shape[1], device=x.device),
                   torch.ones(w.shape[1], x.shape[1] // gs, gs, gs, device=x.device))
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
            if k not in f["live"]:
                assert torch.equal(running[0][k], old[0][k]) and torch.equal(running[1][k], old[1][k])
                continue
            check(worst, label, f"rmean{k}", running[0][k], 0.9 * old[0][k].double() + 0.1 * f["mu"][k].reshape(-1))
            check(worst, label, f"rcov{k}", running[1][k], 0.9 * old[1][k].double() + 0.1 * f["sigma"][k])
    else:
        assert torch.equal(running[0], old[0]) and torch.equal(running[1], old[1])


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("shape, gs, d", [
    ((192, 64, 112, 112), 4, 3),                             # ResNet-50-DWT stem
    ((192, 256, 56, 56), 4, 3), ((192, 256, 56, 56), 4, 8), ((192, 64, 56, 56), 4, 3),   # layer1
    ((128, 32, 28, 28), 4, 3), ((128, 48, 14, 14), 4, 3),   # digits LeNet
    ((32, 64, 56, 56), 1, 3), ((32, 64, 56, 56), 2, 3),
])
def test_model_sites_against_float64(dev, worst, shape, gs, d, layout):
    x, dy = images(shape, dev, gs, seed=gs + d), grad(shape, dev)
    if layout == "nhwc":
        x, dy = _cl(x), _cl(dy)
    w = _weights("softmax", shape[0], d, seed=d, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs {gs} D {d} softmax {layout}", x, dy, gs, w)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("shape, gs", [
    ((1, 64, 56, 56), 4), ((32, 4, 28, 28), 4), ((64, 64, 1, 1), 4), ((64, 64, 1, 1), 1), ((64, 64, 7, 7), 4),
    ((64, 8, 7, 7), 2), ((16, 16, 5, 5), 4),
    ((2, 8, 257, 1), 4),                                     # NCHW: one pixel past 256, two segments of 132 + 125
    ((2, 4, 1025, 1), 4),                                    # channels-last: one pixel past 1024, segments of 513 + 512
])
def test_edges_against_float64(dev, worst, shape, gs, layout):
    x, dy = images(shape, dev, gs, seed=7), grad(shape, dev)
    if layout == "nhwc":
        x, dy = _cl(x), _cl(dy)
    w = _weights("softmax", shape[0], 3, seed=2, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs {gs} D 3 {layout}", x, dy, gs, w)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("mode", ["train", "eval", "notrack"])
@pytest.mark.parametrize("kind", ["softmax", "onehot", "zero"])
@pytest.mark.parametrize("d", [1, 3, 8])
def test_modes_and_weights_against_float64(dev, worst, d, kind, mode, layout):
    shape, gs = (32, 64, 28, 28), 4
    x, dy = images(shape, dev, gs, seed=5), grad(shape, dev)
    if layout == "nhwc":
        x, dy = _cl(x), _cl(dy)
    w = _weights(kind, shape[0], d, seed=2, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs 4 D {d} {kind} {mode} {layout}", x, dy, gs, w, mode)


@gpu
@pytest.mark.parametrize("gs", [2, 4])
@pytest.mark.parametrize("cond", [1.0, 10.0, 100.0, 1000.0])
def test_conditioning_against_float64(dev, worst, cond, gs):
    shape = (32, 64, 28, 28)
    x = images(shape, dev, gs, seed=3, cond=cond)
    w = _weights("softmax", shape[0], 3, seed=4, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs {gs} D 3 cond {cond:g}", x, grad(shape, dev), gs, w)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", [(192, 64, 56, 56), (16, 64, 14, 14)])
def test_large_per_image_offsets_against_float64(dev, worst, shape, mode):
    x = images(shape, dev, 4, seed=12, offset=100.0)
    w = _weights("softmax", shape[0], 3, seed=6, dtype=torch.float32, device=dev)
    against_float64(worst, f"{list(shape)} gs 4 D 3 offset 100 {mode}", x, grad(shape, dev), 4, w, mode)


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
@pytest.mark.parametrize("gs", [1, 2, 4])
def test_one_domain_of_unit_weights_agrees_with_wtransform(dev, worst, gs):
    shape = (32, 64, 28, 28)
    x, dy = images(shape, dev, gs, seed=13), grad(shape, dev)
    w = torch.ones(shape[0], 1, device=dev)
    running = fresh_running(x, gs, w)
    yw, dxw, rmw, rvw = _wtransform(x, dy, gs, (running[0][0], running[1][0]), dev)
    y, dx, _ = run(x, dy, gs, w, "train", running)
    label = f"gs {gs} D 1, unit weights vs WTransform2d"
    for name, a, b in (("y", y, yw), ("dx", dx, dxw), ("rmean", running[0][0], rmw), ("rcov", running[1][0], rvw)):
        check(worst, label, name, a, b, WT_BOUND)


@gpu
@pytest.mark.parametrize("gs", [1, 2, 4])
def test_interleaved_one_hot_labels_agree_with_wtransform_per_domain(dev, worst, gs):
    """Uneven 100 / 60 / 32 labels in random order, against WTransform2d on each gathered subset."""
    shape = (192, 64, 28, 28)
    x, dy = images(shape, dev, gs, seed=17), grad(shape, dev)
    lab = torch.cat([torch.full((n,), d) for d, n in enumerate((100, 60, 32))])
    lab = lab[torch.randperm(192, generator=torch.Generator().manual_seed(0))].to(dev)
    w = torch.nn.functional.one_hot(lab, 3).float()
    running = fresh_running(x, gs, w)
    start = (running[0].clone(), running[1].clone())
    y, dx, _ = run(x, dy, gs, w, "train", running)
    for d in range(3):
        idx = (lab == d).nonzero().squeeze(1)
        yw, dxw, rmw, rvw = _wtransform(x[idx], dy[idx], gs, (start[0][d], start[1][d]), dev)
        label = f"gs {gs} one-hot interleaved vs WTransform2d, domain {d}"
        for name, a, b in (("y", y[idx], yw), ("dx", dx[idx], dxw), ("rmean", running[0][d], rmw),
                           ("rcov", running[1][d], rvw)):
            check(worst, label, name, a, b, WT_BOUND)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("shape", [(32, 64, 56, 56), (16, 48, 14, 14), (16, 64, 7, 7)])
def test_bf16_is_the_fp32_kernels_rounded(dev, layout, shape):
    """7x7 NCHW (H*W % 4 != 0) runs the fp32 kernels on an upcast copy; the rest run the bf16 kernels."""
    fmt = torch.channels_last if layout == "nhwc" else torch.contiguous_format
    x = images(shape, dev, 4, seed=5).bfloat16().contiguous(memory_format=fmt)
    dy = grad(shape, dev).bfloat16().contiguous(memory_format=fmt)
    w = _weights("softmax", shape[0], 3, seed=2, dtype=torch.float32, device=dev)
    y, dx, dw = run(x, dy, 4, w)
    assert y.dtype == torch.bfloat16 and dx.dtype == torch.bfloat16 and dw.dtype == torch.float32
    yf, dxf, dwf = run(x.float(), dy.float(), 4, w)
    assert torch.equal(y, yf.bfloat16()) and torch.equal(dx, dxf.bfloat16()) and torch.equal(dw, dwf)


@gpu
def test_channels_last_at_c_not_a_multiple_of_4_runs_as_nchw(dev):
    shape, gs = (8, 6, 14, 14), 2
    x, dy = images(shape, dev, gs, seed=6), grad(shape, dev)
    w = _weights("softmax", shape[0], 3, seed=2, dtype=torch.float32, device=dev)
    a = run(x, dy, gs, w)
    b = run(_cl(x), _cl(dy), gs, w)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


@gpu
def test_reruns_are_bit_identical(dev):
    for shape, gs, d, cl in (((192, 256, 56, 56), 4, 8, False), ((192, 64, 112, 112), 4, 3, True),
                             ((16, 16, 5, 5), 2, 3, False)):
        x, dy = images(shape, dev, gs, seed=7), grad(shape, dev)
        if cl:
            x, dy = _cl(x), _cl(dy)
        w = _weights("softmax", shape[0], d, seed=3, dtype=torch.float32, device=dev)
        ra, rb = fresh_running(x, gs, w), fresh_running(x, gs, w)
        a, b = run(x, dy, gs, w, running=ra), run(x, dy, gs, w, running=rb)
        for u, v in zip(a + ra, b + rb):
            assert torch.equal(u, v)


@gpu
@pytest.mark.parametrize("cl", [False, True])
def test_cuda_graph_capture_and_replay(dev, cl):
    import dwt_b200
    shape, gs = (16, 64, 28, 28), 4
    m = dwt_b200.LatentDomainWTransform2d(64, gs, 3).to(dev)
    x, dy = images(shape, dev, gs, seed=8), grad(shape, dev)
    if cl:
        x, dy = _cl(x), _cl(dy)
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


@gpu
def test_labels_without_grad_pass_no_dweights(dev):
    shape, gs = (48, 64, 28, 28), 4
    x, dy = images(shape, dev, gs, seed=19), grad(shape, dev)
    lab = torch.randint(0, 3, (shape[0],), generator=torch.Generator().manual_seed(1)).to(dev)
    w = torch.nn.functional.one_hot(lab, 3).float()
    ra, rb = fresh_running(x, gs, w), fresh_running(x, gs, w)
    y, dx, dw = run(x, dy, gs, w, "train", ra)
    yl, dxl, dwl = run(x, dy, gs, w, "train", rb, wgrad=False)
    assert dw is not None and dwl is None
    assert torch.equal(y, yl) and torch.equal(dx, dxl)
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1])


# =========================================================================== GPU: the header's edge rules
@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_zero_mass_domain_is_absent(dev, mode):
    """A zero-mass domain: no status, its buffers untouched, its dweights column 0, and y, dx and the other domains'
    buffers and dweights bit for bit those of the call without it."""
    from dwt_b200 import _native as nv
    shape, gs = (24, 64, 28, 28), 4
    x, dy = images(shape, dev, gs, seed=18), grad(shape, dev)
    w3 = _weights("softmax", shape[0], 3, seed=7, dtype=torch.float32, device=dev)
    w4 = torch.cat([w3[:, :1], torch.zeros(shape[0], 1, device=dev), w3[:, 1:]], 1)
    r3 = fresh_running(x, gs, w3)
    r4 = (torch.cat([r3[0][:1], torch.randn(1, 64, device=dev), r3[0][1:]]),
          torch.cat([r3[1][:1], torch.eye(gs, device=dev).expand(1, 16, gs, gs) * 2, r3[1][1:]]))
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
def test_nan_weight_sets_status_and_stays_in_its_domain(dev):
    from dwt_b200 import _native as nv
    shape, gs = (12, 64, 32, 32), 4
    x, dy = images(shape, dev, gs, seed=10), grad(shape, dev)
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


@gpu
def test_negative_mass_domain_sets_status_and_skips_its_ema(dev):
    from dwt_b200 import _native as nv
    shape, gs = (12, 64, 32, 32), 4
    x, dy = images(shape, dev, gs, seed=20), grad(shape, dev)
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
    assert not torch.equal(running[1][:2], before[1][:2]) and torch.isfinite(running[0]).all()


@gpu
@pytest.mark.parametrize("case", ["zero_row_train", "zero_row_eval", "negative_weight_eval"])
def test_image_without_a_positive_mix_sets_status_and_stays_local(dev, case):
    from dwt_b200 import _native as nv
    shape, gs = (12, 64, 32, 32), 4
    x, dy = images(shape, dev, gs, seed=21), grad(shape, dev)
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
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_indefinite_group_sets_status_and_stays_local(dev, mode):
    """eps < 0 and channels 16..31 (groups 4..7) constant over every image of domain 1: S_1 = eps I is indefinite there,
    W_1 is NaN in those groups, and only domain 1's images read NaN, only there."""
    from dwt_b200 import _native as nv
    shape, gs, eps = (12, 64, 32, 32), 4, -1e-3
    x, dy = images(shape, dev, gs, seed=11), grad(shape, dev)
    lab = torch.arange(12, device=dev) % 3
    w = torch.nn.functional.one_hot(lab, 3).float()
    x[lab == 1, 16:32] = 0.25
    running = fresh_running(images(shape, dev, gs, seed=11), gs, w)
    if mode == "eval":
        running[1][1, 4:8] = 0.0                      # domain 1, groups 4..7: zero covariance
    nv.clear_status(dev)
    y, dx, _ = run(x, dy, gs, w, "notrack" if mode == "train" else "eval", running, eps=eps)
    assert nv.status(dev) & nv.STATUS_NOT_PD
    nv.clear_status(dev)
    keep = torch.ones(shape[:2], dtype=torch.bool, device=dev)
    keep[lab == 1, 16:32] = False
    assert torch.isnan(y[lab == 1][:, 16:32]).all() and not torch.isnan(y[keep]).any()
    assert torch.isnan(dx[lab == 1][:, 16:32]).all() and not torch.isnan(dx[keep]).any()
