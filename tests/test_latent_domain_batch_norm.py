"""Latent-domain batch norm (LatentDomainBatchNorm1d / 2d, functional.latent_domain_batch_norm, dwt_bn_latent_*).

CPU: the float64 closed-form backward (tests/support/ldbn_reference.py) -- dx, dweights, dgamma, dbeta -- against autograd
and central finite differences, in train and eval, for 1, 3 and 8 domains under softmax, one-hot and zero-mass weights and
at M = 1; one-hot weights against F.batch_norm on every subset; the module surface; the refusals of the C ABI (argument
checks run before any device call, so fake pointers do), and that the other entry points keep theirs.

GPU: the kernels against the float64 reference at the ResNet-50 site shapes, a long-row shape and [N, C], in both layouts
and all three modes, with the bounds below; per-image mean offsets of ~100; the package's BatchNorm2d on one-hot subsets;
bit-for-bit checks (bf16 against fp32, reruns, graph replay, a zero-mass domain, weights without a gradient); every edge
rule; and a training step through a softmax domain branch.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import ldbn_reference as R  # noqa: E402

# norm-wise relative error against float64: y, dx, dbeta and the running buffers (measured on an H100: at most 1e-7);
# dgamma and dweights, sums over N*HW and over C of terms that largely cancel (measured: at most 1e-5)
BOUND, DW_BOUND = 1e-6, 1e-4
gpu = pytest.mark.gpu


def _weights(kind, n, d, seed=0, dtype=torch.float64, device="cpu"):
    """softmax: random soft assignments; onehot: image i in domain i % d; zero: onehot with the last domain's column 0."""
    g = torch.Generator(device=device).manual_seed(seed)
    if kind == "softmax":
        return torch.softmax(2.0 * torch.randn(n, d, generator=g, dtype=dtype, device=device), 1)
    w = torch.zeros(n, d, dtype=dtype, device=device)
    lab = torch.arange(n, device=device) % d
    if kind == "zero" and d > 1:
        lab[lab == d - 1] = 0
    w[torch.arange(n, device=device), lab] = 1.0
    return w


def _cpu_case(seed, n=7, c=5, hw=(3, 4)):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, c, *hw, generator=g, dtype=torch.float64) * 1.5 + torch.randn(n, c, *([1] * len(hw)), generator=g,
                                                                                       dtype=torch.float64)
    dout = torch.randn(x.shape, generator=g, dtype=torch.float64) + 0.3
    gamma = 1.0 + 0.3 * torch.randn(c, generator=g, dtype=torch.float64)
    beta = 0.2 * torch.randn(c, generator=g, dtype=torch.float64)
    return x, dout, gamma, beta


def _running(d, c, seed, dtype=torch.float64, device="cpu"):
    g = torch.Generator(device=device).manual_seed(seed)
    return (0.3 * torch.randn(d, c, generator=g, dtype=dtype, device=device),
            0.5 + torch.rand(d, c, generator=g, dtype=dtype, device=device))


# =========================================================================== CPU: the float64 reference
@pytest.mark.parametrize("hw", [(3, 4), ()], ids=["M12", "M1"])
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("kind", ["softmax", "onehot", "zero"])
@pytest.mark.parametrize("d", [1, 3, 8])
def test_closed_form_backward_matches_autograd(d, kind, train, hw):
    n = 17
    x, dout, gamma, beta = _cpu_case(d, n=n, hw=hw)
    w = _weights(kind, n, d, seed=d)
    running = None if train else _running(d, 5, 1)
    leaves = [t.clone().requires_grad_(True) for t in (x, w, gamma, beta)]
    y = R.ldbn_torch(leaves[0], leaves[1], leaves[2], leaves[3], running=running)["y"]
    want = torch.autograd.grad(y, leaves, dout)
    got = R.closed_form_backward(x, dout, w, gamma, running=running)
    for name, a, b in zip(("dx", "dweights", "dgamma", "dbeta"), got, want):
        assert (a - b).abs().max() <= 1e-10 * b.abs().max().clamp_min(1e-12), (name, float((a - b).abs().max()))
    if kind == "zero" and d > 1:
        assert torch.equal(got[1][:, -1], torch.zeros(n, dtype=x.dtype))


@pytest.mark.parametrize("train", [True, False])
def test_closed_form_backward_matches_finite_differences(train):
    d = 3
    x, dout, gamma, beta = _cpu_case(5, n=6)
    w = _weights("softmax", 6, d, seed=5)
    running = None if train else _running(d, 5, 2)
    dx, dw, dg, db = R.closed_form_backward(x, dout, w, gamma, running=running)
    loss = lambda t, ww, gg: float((dout * R.ldbn_torch(t, ww, gg, beta, running=running)["y"]).sum())
    h = 1e-6
    rng = np.random.default_rng(0)
    for _ in range(4):
        v = torch.tensor(rng.standard_normal(tuple(x.shape)))
        fd = (loss(x + h * v, w, gamma) - loss(x - h * v, w, gamma)) / (2 * h)
        assert abs(fd - float((dx * v).sum())) <= 1e-6 * max(abs(fd), 1.0)
        u = torch.tensor(rng.standard_normal(5))
        fd = (loss(x, w, gamma + h * u) - loss(x, w, gamma - h * u)) / (2 * h)
        assert abs(fd - float((dg * u).sum())) <= 1e-6 * max(abs(fd), 1.0)
    for n in range(6):
        for k in range(d):
            e = torch.zeros_like(w)
            e[n, k] = h
            fd = (loss(x, w + e, gamma) - loss(x, w - e, gamma)) / (2 * h)
            assert abs(fd - float(dw[n, k])) <= 1e-6 * max(abs(fd), 1.0), (n, k, fd, float(dw[n, k]))


def test_one_hot_weights_are_batch_norm_on_each_subset():
    x, _, gamma, beta = _cpu_case(4, n=9)
    lab = torch.tensor([2, 0, 0, 1, 2, 0, 1, 1, 0])
    w = torch.nn.functional.one_hot(lab, 3).double()
    run = _running(3, 5, 3)
    f = R.ldbn_torch(x, w, gamma, beta)
    rm, rv = R.running_update(f, run, 0.1, 12)
    for d in range(3):
        sub = x[lab == d]
        m_d, v_d = run[0][d].clone(), run[1][d].clone()
        want = torch.nn.functional.batch_norm(sub, m_d, v_d, gamma, beta, training=True, momentum=0.1, eps=1e-5)
        assert torch.allclose(f["y"][lab == d], want, atol=1e-12)
        assert torch.allclose(rm[d], m_d, atol=1e-12) and torch.allclose(rv[d], v_d, atol=1e-12)


# =========================================================================== CPU: module surface
def test_module_surface():
    import inspect
    import dwt_b200
    for cls in (dwt_b200.LatentDomainBatchNorm1d, dwt_b200.LatentDomainBatchNorm2d):
        assert cls.__name__ in dwt_b200.__all__
        assert list(inspect.signature(cls.__init__).parameters) == [
            "self", "num_features", "num_domains", "eps", "momentum", "affine", "track_running_stats"]
    m = dwt_b200.LatentDomainBatchNorm2d(64, 3)
    assert (m.num_features, m.num_domains, m.eps, m.momentum, m.affine, m.track_running_stats) == (64, 3, 1e-5, 0.1, True, True)
    assert torch.equal(m.weight, torch.ones(64)) and torch.equal(m.bias, torch.zeros(64))
    assert sorted(m.state_dict()) == ["bias", "num_batches_tracked", "running_mean", "running_var", "weight"]
    assert torch.equal(m.running_mean, torch.zeros(3, 64)) and torch.equal(m.running_var, torch.ones(3, 64))
    assert "num_domains=3" in repr(m)
    dwt_b200.LatentDomainBatchNorm2d(64, 3).load_state_dict(m.state_dict())
    u = dwt_b200.LatentDomainBatchNorm1d(10, 2, affine=False, track_running_stats=False)
    assert u.weight is None and u.bias is None and u.running_mean is None and sorted(u.state_dict()) == []


def test_bad_inputs_and_cpu_tensors_are_refused():
    import dwt_b200
    from dwt_b200 import functional as F
    m = dwt_b200.LatentDomainBatchNorm2d(8, 3)
    x = torch.zeros(4, 8, 5, 5)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(x, torch.full((4, 3), 1 / 3))
    with pytest.raises(ValueError, match=r"expected weights of shape \[4, 3\] \(got \[4, 2\]\)"):
        m(x, torch.ones(4, 2))
    with pytest.raises(ValueError, match=r"expected weights of shape \[4, 3\] \(got \[12\]\)"):
        m(x, torch.ones(12))
    with pytest.raises(TypeError, match="floating-point weights"):
        m(x, torch.ones(4, 3, dtype=torch.int64))
    with pytest.raises(ValueError, match="weights on x's device"):
        m(x, torch.ones(4, 3, device="meta"))
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(4, 8, 5), torch.ones(4, 3))
    with pytest.raises(ValueError, match=r"expected 2D or 3D input \(got 4D input\)"):
        dwt_b200.LatentDomainBatchNorm1d(8, 3)(x, torch.ones(4, 3))
    with pytest.raises(ValueError, match="expected 8 channels"):
        m(torch.zeros(4, 6, 5, 5), torch.ones(4, 3))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        dwt_b200.LatentDomainBatchNorm1d(8, 1)(torch.zeros(1, 8), torch.ones(1, 1))
    run = (m.running_mean, m.running_var)
    with pytest.raises(ValueError, match=r"weights of shape \[N, n_domains\] with N = 4"):
        F.latent_domain_batch_norm(x, torch.ones(5, 3), None, None, training_stats=True, eps=1e-5, momentum=0.1,
                                   update_running=False, running=run)
    with pytest.raises(ValueError, match="weight and bias together"):
        F.latent_domain_batch_norm(x, torch.ones(4, 3), m.weight, None, training_stats=True, eps=1e-5, momentum=0.1,
                                   update_running=False, running=run)


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _fp(v):
    return None if v is None else ctypes.c_void_p(v)


def _fwd(lib, N=8, C=64, HW=49, D=3, mode=0, x=_FAKE, y=_FAKE, w=_FAKE, save=_FAKE, running=_FAKE, update=1,
         gamma=_FAKE, beta=_FAKE, ws_bytes=1 << 40, **_):
    return lib.dwt_bn_latent_fwd(_fp(x), _fp(y), N, C, HW, D, mode, 1e-5, 0.1, update, _fp(running), _fp(running), _fp(w),
                                 _fp(gamma), _fp(beta), _fp(save), ctypes.c_void_p(_FAKE), ws_bytes, None)


def _bwd(lib, N=8, C=64, HW=49, D=3, mode=0, x=_FAKE, y=_FAKE, w=_FAKE, save=_FAKE, gamma=_FAKE, beta=_FAKE,
         ws_bytes=1 << 40, **_):
    return lib.dwt_bn_latent_bwd(_fp(x), ctypes.c_void_p(_FAKE), _fp(y), N, C, HW, D, mode, 1e-5, _fp(w), _fp(_FAKE),
                                 _fp(save), None, _fp(gamma), _fp(beta), ctypes.c_void_p(_FAKE), ws_bytes, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


@pytest.mark.parametrize("call", [_fwd, _bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(D=0), -1, b"n_domains 0 outside [1,8] (latent-domain batch norm)"),
    (dict(D=9), -1, b"n_domains 9 outside [1,8] (latent-domain batch norm)"),
    (dict(mode=0x2), -1, b"bad mode"), (dict(mode=0x400), -1, b"bad mode"), (dict(mode=0x3), -1, b"bad mode"),
    (dict(N=0), -1, b"empty tensor"), (dict(C=0), -1, b"empty tensor"), (dict(HW=0), -1, b"empty tensor"),
    (dict(N=1024, C=2048, HW=1024), -4, b"latent-domain batch norm needs N*C*HW < 2^31"),
    (dict(C=66, mode=0x100), -4, b"latent-domain batch norm runs channels-last at C % 4 == 0 only"),
    (dict(HW=49, mode=0x200), -4, b"latent-domain batch norm runs NCHW bf16 at HW % 4 == 0 only"),
    (dict(x=None), -1, b"null pointer argument"), (dict(y=None), -1, b"null pointer argument"),
    (dict(w=None), -1, b"null pointer argument"), (dict(save=None), -1, b"null pointer argument"),
    (dict(gamma=None), -1, b"must be both given or both NULL"), (dict(beta=None), -1, b"must be both given or both NULL"),
    (dict(x=_FAKE + 4), -1, b"activation tensors must be 16-byte aligned (latent-domain batch norm)"),
    (dict(y=_FAKE + 8), -1, b"activation tensors must be 16-byte aligned"),
    (dict(HW=196, mode=0x200, x=_FAKE + 4), -1, b"activation tensors must be 8-byte aligned"),
    (dict(w=_FAKE + 2), -1, b"must be 4-byte"), (dict(save=_FAKE + 4), -1, b"save_stats 16-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


@pytest.mark.parametrize("kw", [dict(mode=1), dict(mode=0, update=1)])
def test_missing_running_buffers_are_refused(lib, kw):
    assert _fwd(lib, running=None, **kw) == -1
    assert b"running buffer is null" in lib.dwt_last_error()


@pytest.mark.parametrize("call", [_fwd, _bwd])
@pytest.mark.parametrize("kw", [dict(N=192, C=2048, HW=49, D=8), dict(N=8, C=64, HW=12544, D=3, mode=0x301),
                                dict(N=64, C=100, HW=1, D=1), dict(N=3, C=5, HW=7, D=2, running=None, update=0),
                                dict(N=192, C=256, HW=3136, D=3, mode=0x200)])
def test_small_workspace_is_refused(lib, call, kw):
    assert lib.dwt_bn_latent_workspace_bytes(kw["N"], kw["C"], kw["HW"], kw["D"]) > 1 << 20
    assert call(lib, ws_bytes=1 << 20, **kw) == -2      # below the scratch of any call: no launch is ever reached
    assert b"workspace too small" in lib.dwt_last_error()


def test_workspace_query(lib):
    assert lib.dwt_bn_latent_workspace_bytes(8, 128, 3136, 8) > lib.dwt_bn_latent_workspace_bytes(8, 128, 3136, 1) > 0
    for args in ((0, 128, 49, 3), (8, 0, 49, 3), (8, 128, 0, 3), (8, 128, 49, 0), (8, 128, 49, 9), (1024, 2048, 1024, 3)):
        assert lib.dwt_bn_latent_workspace_bytes(*args) == 0
    _fwd(lib, x=None)
    err = lib.dwt_last_error()
    lib.dwt_bn_latent_workspace_bytes(8, 128, 49, 9)
    assert lib.dwt_last_error() == err                                           # a size query leaves the text alone


def test_other_entry_points_keep_their_refusals(lib):
    p = ctypes.c_void_p(_FAKE)
    assert lib.dwt_whiten_latent_fwd(p, p, 8, 128, 3136, 1, 3, 0, 1e-3, 0.1, 1, p, p, p, p, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_last_error().startswith(b"latent-domain whitening is built for the tensor-core kernels only")
    assert lib.dwt_whiten_latent_fwd(p, p, 8, 128, 196, 64, 3, 0, 1e-3, 0.1, 1, p, p, p, p, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_whiten_fwd(p, p, 8, 128, 3136, 64, 5, 0, 1e-3, 0.1, 0, None, None, None, None, None, None, 0, p, p, p,
                              1 << 40, None) == -1
    assert lib.dwt_last_error() == b"n_domains 5 outside [1,4]"
    assert lib.dwt_whiten_instance_fwd(p, p, 8, 128, 3136, 4, 0, 1e-3, p, p, p, 1 << 40, None) == -4
    assert lib.dwt_last_error().startswith(b"instance whitening is built for the tensor-core kernels only")
    assert lib.dwt_latent_workspace_bytes(8, 128, 3136, 4, 3) == 0


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nlatent-domain batch norm, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-60s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b, bound):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= bound, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def images(shape, dev, seed=0, offset=2.0):
    """float32 activations of `shape`: unit noise plus a per-image, per-channel mean of spread `offset`."""
    g = torch.Generator(device=dev).manual_seed(seed)
    n, c = shape[:2]
    x = 1.3 * torch.randn(shape, device=dev, generator=g) + 0.5
    return x + offset * torch.randn(n, c, *([1] * (len(shape) - 2)), device=dev, generator=g)


def grad(shape, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, device=dev, generator=g) + 0.5


def affine(c, dev, seed=2):
    g = torch.Generator(device=dev).manual_seed(seed)
    return 1.0 + 0.2 * torch.randn(c, device=dev, generator=g), 0.1 * torch.randn(c, device=dev, generator=g)


def run_layer(x, w, gamma, beta, mode, running, layout, eps=1e-5, momentum=0.1, dout=None):
    """One forward + backward through functional.latent_domain_batch_norm -> (y, dx, dweights, dgamma, dbeta, running)."""
    from dwt_b200 import functional as F
    rm, rv = (running[0].clone(), running[1].clone()) if running is not None else (None, None)
    xt = x.contiguous(memory_format=torch.channels_last if layout == "nhwc" else torch.contiguous_format)
    xt = xt.detach().requires_grad_(True)
    wt = w.detach().clone().requires_grad_(True)
    gt = None if gamma is None else gamma.detach().clone().requires_grad_(True)
    bt = None if beta is None else beta.detach().clone().requires_grad_(True)
    train = mode != "eval"
    y = F.latent_domain_batch_norm(xt, wt, gt, bt, training_stats=train, eps=eps, momentum=momentum,
                                   update_running=mode == "train", running=(rm, rv))
    leaves = [xt, wt] + ([gt, bt] if gt is not None else [])
    grads = torch.autograd.grad(y, leaves, dout if dout is not None else torch.ones_like(y))
    dg, db = (grads[2], grads[3]) if gt is not None else (None, None)
    return y, grads[0], grads[1], dg, db, (rm, rv)


def compare(worst, label, x, w, gamma, beta, mode, layout, dout, running):
    y, dx, dw, dg, db, (rm, rv) = run_layer(x, w, gamma, beta, mode, running, layout, dout=dout)
    xd, wd, dd = x.double(), w.double(), dout.double()
    gd, bd = gamma.double(), beta.double()
    run64 = None if mode != "eval" else (running[0].double(), running[1].double())
    f = R.ldbn_torch(xd, wd, gd, bd, running=run64)
    rx, rw, rg, rb = R.closed_form_backward(xd, dd, wd, gd, running=run64)
    check(worst, label, "y", y, f["y"], BOUND)
    check(worst, label, "dx", dx, rx, BOUND)
    check(worst, label, "dbeta", db, rb, BOUND)
    check(worst, label, "dgamma", dg, rg, DW_BOUND)
    check(worst, label, "dweights", dw, rw, DW_BOUND)
    if mode == "train":
        em, ev = R.running_update(f, (running[0].double(), running[1].double()), 0.1, x[0, 0].numel())
        check(worst, label, "running_mean", rm, em, BOUND)
        check(worst, label, "running_var", rv, ev, BOUND)


SHAPES = [((192, 256, 56, 56), 3), ((192, 256, 56, 56), 8), ((192, 512, 28, 28), 3), ((192, 512, 28, 28), 8),
          ((192, 1024, 14, 14), 3), ((192, 1024, 14, 14), 8), ((192, 2048, 7, 7), 3), ((192, 2048, 7, 7), 8),
          ((8, 64, 112, 112), 3), ((64, 100), 3)]


@gpu
@pytest.mark.parametrize("shape, d", SHAPES, ids=[f"{'x'.join(map(str, s))}-D{d}" for s, d in SHAPES])
def test_against_float64(dev, worst, shape, d):
    x = images(shape, dev)
    w = _weights("softmax", shape[0], d, seed=d, dtype=torch.float32, device=dev)
    gamma, beta = affine(shape[1], dev)
    dout = grad(shape, dev)
    running = tuple(t.float() for t in _running(d, shape[1], 4, device=dev))
    for layout in (["nchw", "nhwc"] if len(shape) == 4 else ["nchw"]):
        for mode in ("train", "eval", "untracked"):
            compare(worst, f"{shape} D={d} {layout} {mode}", x, w, gamma, beta, mode, layout, dout, running)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_large_mean_offsets_against_float64(dev, worst, layout):
    shape, d = (64, 128, 14, 14), 3
    x = images(shape, dev, seed=5, offset=100.0)
    w = _weights("softmax", 64, d, seed=6, dtype=torch.float32, device=dev)
    gamma, beta = affine(128, dev)
    running = tuple(t.float() for t in _running(d, 128, 4, device=dev))
    for mode in ("train", "untracked"):
        compare(worst, f"offset 100 {shape} {layout} {mode}", x, w, gamma, beta, mode, layout, grad(shape, dev), running)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_one_hot_subsets_match_batch_norm(dev, layout):
    import dwt_b200
    n, c = 192, 64
    shape = (n, c, 14, 14)
    g = torch.Generator().manual_seed(7)
    lab = torch.cat([torch.full((100,), 0), torch.full((60,), 1), torch.full((32,), 2)])[torch.randperm(n, generator=g)]
    w = torch.nn.functional.one_hot(lab, 3).float().to(dev)
    x, dout = images(shape, dev, seed=8), grad(shape, dev, seed=9)
    gamma, beta = affine(c, dev)
    running = (torch.zeros(3, c, device=dev), torch.ones(3, c, device=dev))
    y, dx, _, _, _, (rm, rv) = run_layer(x, w, gamma, beta, "train", running, layout, dout=dout)
    for d in range(3):
        sel = (lab == d).nonzero().flatten().to(dev)
        bm, bv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        bn = dwt_b200.BatchNorm2d(c, bm, bv).to(dev).train()
        with torch.no_grad():
            bn.weight.copy_(gamma)
            bn.bias.copy_(beta)
        xs = x[sel].clone().requires_grad_(True)
        ys = bn(xs)
        (dxs,) = torch.autograd.grad(ys, xs, dout[sel])
        assert rel(y[sel], ys)[0] < 1e-5 and rel(dx[sel], dxs)[0] < 1e-4
        assert rel(rm[d], bm)[0] < 1e-5 and rel(rv[d], bv)[0] < 1e-5
    # one domain of all-ones weights is BatchNorm2d on the whole batch
    y1, dx1, _, _, _, (rm1, rv1) = run_layer(x, torch.ones(n, 1, device=dev), gamma, beta, "train",
                                             (torch.zeros(1, c, device=dev), torch.ones(1, c, device=dev)), layout,
                                             dout=dout)
    bm, bv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    bn = dwt_b200.BatchNorm2d(c, bm, bv).to(dev).train()
    with torch.no_grad():
        bn.weight.copy_(gamma)
        bn.bias.copy_(beta)
    xs = x.clone().requires_grad_(True)
    ys = bn(xs)
    (dxs,) = torch.autograd.grad(ys, xs, dout)
    assert rel(y1, ys)[0] < 1e-5 and rel(dx1, dxs)[0] < 1e-4
    assert rel(rm1[0], bm)[0] < 1e-5 and rel(rv1[0], bv)[0] < 1e-5


@gpu
@pytest.mark.parametrize("layout, shape", [("nchw", (32, 64, 14, 14)), ("nhwc", (32, 64, 7, 7)),
                                           ("nhwc", (16, 64, 56, 56)), ("nchw", (16, 32, 56, 56))])
def test_bf16_is_fp32_rounded(dev, layout, shape):
    x = images(shape, dev, seed=11).bfloat16()
    dout = grad(shape, dev, seed=12).bfloat16()
    w = _weights("softmax", shape[0], 3, seed=3, dtype=torch.float32, device=dev)
    gamma, beta = affine(shape[1], dev)
    running = (torch.zeros(3, shape[1], device=dev), torch.ones(3, shape[1], device=dev))
    for mode in ("train", "eval"):
        b = run_layer(x, w, gamma, beta, mode, running, layout, dout=dout)
        f = run_layer(x.float(), w, gamma, beta, mode, running, layout, dout=dout.float())
        assert b[0].dtype == torch.bfloat16 and b[1].dtype == torch.bfloat16
        assert torch.equal(b[0], f[0].bfloat16()) and torch.equal(b[1], f[1].bfloat16())
        for k in (2, 3, 4):
            assert torch.equal(b[k], f[k])
        assert torch.equal(b[5][0], f[5][0]) and torch.equal(b[5][1], f[5][1])
        if layout == "nhwc":
            assert b[0].is_contiguous(memory_format=torch.channels_last)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_reruns_are_bit_identical(dev, layout):
    shape = (96, 128, 28, 28)
    x, dout = images(shape, dev, seed=13), grad(shape, dev, seed=14)
    w = _weights("softmax", 96, 8, seed=1, dtype=torch.float32, device=dev)
    gamma, beta = affine(128, dev)
    running = (torch.zeros(8, 128, device=dev), torch.ones(8, 128, device=dev))
    a = run_layer(x, w, gamma, beta, "train", running, layout, dout=dout)
    b = run_layer(x, w, gamma, beta, "train", running, layout, dout=dout)
    for u, v in zip(a[:5], b[:5]):
        assert torch.equal(u, v)
    assert torch.equal(a[5][0], b[5][0]) and torch.equal(a[5][1], b[5][1])


@gpu
def test_graph_replay_matches_eager(dev):
    import dwt_b200
    shape = (32, 64, 14, 14)
    m = dwt_b200.LatentDomainBatchNorm2d(64, 3).to(dev).train()
    x = images(shape, dev, seed=15).requires_grad_(True)
    w = _weights("softmax", 32, 3, seed=2, dtype=torch.float32, device=dev).requires_grad_(True)
    dout = grad(shape, dev)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for _ in range(2):                                                        # warm-up on the capture stream
            y = m(x, w)
            torch.autograd.grad(y, (x, w, m.weight, m.bias), dout)
    torch.cuda.current_stream(dev).wait_stream(s)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = m(x, w)
        gg = torch.autograd.grad(yg, (x, w, m.weight, m.bias), dout)
    m.load_state_dict(state)
    graph.replay()
    torch.cuda.synchronize(dev)
    after_graph = {k: v.clone() for k, v in m.state_dict().items()}
    m.load_state_dict(state)
    ye = m(x, w)
    ge = torch.autograd.grad(ye, (x, w, m.weight, m.bias), dout)
    assert torch.equal(yg, ye)
    for a, b in zip(gg, ge):
        assert torch.equal(a, b)
    for k in ("running_mean", "running_var"):
        assert torch.equal(after_graph[k], m.state_dict()[k])


@gpu
def test_zero_mass_domain_and_weights_without_gradient(dev):
    from dwt_b200 import _native as nv
    shape = (48, 64, 14, 14)
    x, dout = images(shape, dev, seed=16), grad(shape, dev, seed=17)
    w = _weights("zero", 48, 3, dtype=torch.float32, device=dev)
    gamma, beta = affine(64, dev)
    running = (torch.zeros(3, 64, device=dev), torch.ones(3, 64, device=dev))
    torch.cuda.synchronize(dev)
    nv.status_all(dev)
    for buf in nv._workspaces.values():
        buf[:4].zero_()
    y, dx, dw, _, _, (rm, rv) = run_layer(x, w, gamma, beta, "train", running, "nchw", dout=dout)
    assert nv.status_all(dev) == 0
    assert torch.equal(dw[:, 2], torch.zeros(48, device=dev))
    assert torch.equal(rm[2], running[0][2]) and torch.equal(rv[2], running[1][2])
    two = run_layer(x, w[:, :2].contiguous(), gamma, beta, "train", (running[0][:2], running[1][:2]), "nchw", dout=dout)
    assert torch.equal(y, two[0]) and torch.equal(dx, two[1])
    # weights without a gradient: no dweights buffer, the same dx
    from dwt_b200 import functional as F
    xt = x.clone().requires_grad_(True)
    yt = F.latent_domain_batch_norm(xt, w, gamma, beta, training_stats=True, eps=1e-5, momentum=0.1,
                                    update_running=False, running=(None, None))
    (dxt,) = torch.autograd.grad(yt, xt, dout)
    assert torch.equal(yt, y) and torch.equal(dxt, dx)


def _status_run(dev, x, w, running, mode="train", eps=1e-5):
    from dwt_b200 import _native as nv
    torch.cuda.synchronize(dev)
    for buf in nv._workspaces.values():
        buf[:4].zero_()
    out = run_layer(x, w, None, None, mode, running, "nchw", eps=eps, dout=grad(x.shape, dev))
    return out, nv.status_all(dev)


@gpu
def test_nan_weight(dev):
    x = images((16, 8, 7, 7), dev)
    w = _weights("softmax", 16, 3, dtype=torch.float32, device=dev)
    w[5, 1] = float("nan")
    running = (torch.zeros(3, 8, device=dev), torch.ones(3, 8, device=dev))
    (y, dx, *_, (rm, rv)), st = _status_run(dev, x, w, running)
    assert st & 1
    assert torch.equal(rm[1], running[0][1]) and torch.equal(rv[1], running[1][1])     # that domain's EMA skipped
    assert not torch.equal(rm[0], running[0][0])


@gpu
def test_negative_mass_domain(dev):
    x = images((16, 8, 7, 7), dev)
    w = _weights("onehot", 16, 3, dtype=torch.float32, device=dev)
    w[:, 2] = -w[:, 2]
    running = (torch.zeros(3, 8, device=dev), torch.ones(3, 8, device=dev))
    (y, dx, *_, (rm, rv)), st = _status_run(dev, x, w, running)
    assert st & 1
    assert torch.equal(rm[2], running[0][2]) and torch.equal(rv[2], running[1][2])
    on2 = w[:, 2] != 0
    assert torch.isnan(y[on2]).all() and torch.isfinite(y[~on2]).all() and torch.isfinite(dx[~on2]).all()


@gpu
@pytest.mark.parametrize("row", ["zero", "negative"])
def test_image_without_positive_mix(dev, row):
    x = images((16, 8, 7, 7), dev)
    w = _weights("softmax", 16, 3, dtype=torch.float32, device=dev)
    w[3] = 0.0 if row == "zero" else torch.tensor([-1.0, 0.0, 0.0], device=dev)
    running = (torch.zeros(3, 8, device=dev), torch.ones(3, 8, device=dev))
    (y, dx, *_), st = _status_run(dev, x, w, running, mode="untracked")
    assert st & 1
    assert torch.isnan(y[3]).all() and torch.isnan(dx[3]).all()
    if row == "zero":                                      # an image without weight leaves the others untouched
        others = torch.arange(16, device=dev) != 3
        assert torch.isfinite(y[others]).all() and torch.isfinite(dx[others]).all()


@gpu
def test_variance_plus_eps_not_positive(dev):
    x = images((16, 8, 7, 7), dev)
    x[:, 4] = 3.0                                          # a constant channel: sigma2 = 0, eps < 0
    w = _weights("softmax", 16, 2, dtype=torch.float32, device=dev)
    running = (torch.zeros(2, 8, device=dev), torch.ones(2, 8, device=dev))
    (y, dx, *_, (rm, rv)), st = _status_run(dev, x, w, running, eps=-1e-3)
    assert st & 1
    assert torch.isnan(y[:, 4]).all() and torch.isfinite(y[:, :4]).all()
    assert torch.equal(rm[:, 4], running[0][:, 4]) and torch.equal(rv[:, 4], running[1][:, 4])
    assert not torch.equal(rm[:, 3], running[0][:, 3])


@gpu
def test_small_mass_leaves_buffers_untouched(dev):
    x = images((12, 8), dev)                               # M = 1: domain 2 holds one image, M s_2 = 1
    w = torch.zeros(12, 3, device=dev)
    w[:6, 0] = 1.0
    w[6:11, 1] = 1.0
    w[11, 2] = 1.0
    running = (torch.zeros(3, 8, device=dev), torch.ones(3, 8, device=dev))
    (y, *_, (rm, rv)), st = _status_run(dev, x, w, running)
    assert st == 0
    assert torch.equal(rm[2], running[0][2]) and torch.equal(rv[2], running[1][2])
    assert not torch.equal(rm[1], running[0][1])
    f = R.ldbn_torch(x.double(), w.double())
    assert rel(y, f["y"])[0] < 1e-5                        # the biased (zero) variance still normalises


@gpu
def test_training_step_lowers_the_loss(dev):
    import dwt_b200
    torch.manual_seed(0)
    n, c = 64, 16
    x = images((n, c, 8, 8), dev, seed=21)
    target = torch.randn(n, c, 8, 8, device=dev)
    branch = torch.nn.Linear(c, 3).to(dev)
    norm = dwt_b200.LatentDomainBatchNorm2d(c, 3).to(dev).train()
    params = list(branch.parameters()) + list(norm.parameters())
    opt = torch.optim.SGD(params, lr=0.1)

    def loss_fn():
        w = torch.softmax(branch(x.mean((2, 3))), 1)
        return ((norm(x, w) - target) ** 2).mean()

    before = loss_fn()
    opt.zero_grad()
    before.backward()
    assert branch.weight.grad.abs().sum() > 0
    opt.step()
    assert loss_fn().item() < before.item()
