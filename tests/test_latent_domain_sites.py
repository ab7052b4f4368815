"""Latent-domain sites: latent-domain batch norm and small-group latent-domain whitening with the ResNet-50-DWT norm site
relu(gamma * zhat + beta [+ residual]) fused into their kernels (dwt_latent_site_*, functional.latent_domain_batch_norm /
latent_domain_whiten's relu / residual / weight / bias arguments, the modules' forward keywords).

CPU: the whitening site's closed-form dgamma (stated in dwt_b200.h) against float64 autograd; the refusals of the C ABI
pair (argument checks run before any device call, so fake pointers do); the module and functional argument errors.

GPU: every epilogue combination against the float64 composition at the model's site shapes and the launch edges, in both
layouts, in train, eval and untracked modes, for 3 and 8 domains; batch-norm sites bit for bit against the ATen
composition; bf16 bit for bit against the fp32 call on the widened inputs; reruns and graph replay; the edge rules
(zero-mass domain, NaN weight, image with no positive mix) under an epilogue; the tensor-core group sizes' tensor-op site.
"""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import ld_reference as LR  # noqa: E402
import ldbn_reference as LB  # noqa: E402

BOUND, DW_BOUND = 1e-4, 1e-3
EPIS = ["none", "affine", "relu", "residual"]
gpu = pytest.mark.gpu


def _ref_site(kind, x, w, gs, gamma, beta, relu, res, running, eps):
    """The float64 composition: the layer, then gamma / beta, the residual and the ReLU as tensor ops."""
    z = LB.ldbn_torch(x, w, eps=eps, running=running)["y"] if kind == "bn" else LR.ld_torch(x, gs, w, eps=eps,
                                                                                              running=running)["y"]
    if gamma is None:
        return z
    shape = (1, -1) + (1,) * (x.dim() - 2)
    y = z * gamma.view(shape) + beta.view(shape)
    if res is not None:
        y = y + res
    return torch.relu(y) if relu else y


# =========================================================================== CPU: the whitening site's dgamma
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("gs", [1, 2, 4])
def test_whitening_site_dgamma_closed_form(gs, train):
    n, c, d = 9, 2 * gs, 3
    g = torch.Generator().manual_seed(gs)
    x = torch.randn(n, c, 5, 5, generator=g, dtype=torch.float64) + torch.randn(n, c, 1, 1, generator=g, dtype=torch.float64)
    w = torch.softmax(torch.randn(n, d, generator=g, dtype=torch.float64), 1)
    running = None
    if not train:
        running = (0.1 * torch.randn(d, c, generator=g, dtype=torch.float64),
                   torch.eye(gs, dtype=torch.float64).expand(d, c // gs, gs, gs) * 1.3)
    f = LR.ld_torch(x, gs, w, running=running)
    dz = torch.randn(x.shape, generator=g, dtype=torch.float64)
    want = (dz * f["y"]).sum((0, 2, 3))
    # A_n = sum_d w_nd W_d, b_n = sum_d w_nd W_d mu_d; A_n (m_n - m~_n) = A_n m_n - b_n
    A = sum(w[:, k].view(n, 1, 1, 1) * f["w_mat"][k] for k in f["live"])
    b = sum(w[:, k].view(n, 1, 1) * (f["w_mat"][k] @ f["mu"][k].unsqueeze(-1)).squeeze(-1) for k in f["live"])
    xg, dzg = x.reshape(n, c // gs, gs, -1), dz.reshape(n, c // gs, gs, -1)
    gz = dzg.sum(-1)
    rz = dzg @ (xg - f["m"].unsqueeze(-1)).transpose(-1, -2)
    off = (A @ f["m"].unsqueeze(-1)).squeeze(-1) - b
    got = ((torch.tril(A) * rz).sum(-1) + off * gz).sum(0).reshape(c)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-10), (got, want)


# =========================================================================== CPU: C ABI refusals, no device call
_FAKE = 1 << 20


def _fp(v):
    return None if v is None else ctypes.c_void_p(v)


def _site_fwd(lib, kind=1, N=8, C=64, HW=784, gs=1, D=3, mode=0, epi=3, gamma=_FAKE, beta=_FAKE, res=None, mask=None,
              x=_FAKE):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_latent_site_fwd(kind, _fp(x), p, N, C, HW, gs, D, mode, 1e-5, 0.1, 1, p, p, p, _fp(gamma), _fp(beta),
                                   _fp(res), _fp(mask), epi, p, p, p, p, 1 << 40, None)


def _site_bwd(lib, kind=1, N=8, C=64, HW=784, gs=1, D=3, mode=0, epi=3, gamma=_FAKE, beta=_FAKE, res=None, mask=None,
              x=_FAKE, dgamma=None):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_latent_site_bwd(kind, _fp(x), p, p, N, C, HW, gs, D, mode, 1e-5, p, _fp(gamma), _fp(beta), _fp(mask),
                                   _fp(res), epi, p, p, p, None, _fp(dgamma), _fp(dgamma), p, 1 << 40, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


@pytest.mark.parametrize("call", [_site_fwd, _site_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(kind=2), -1, b"neither DWT_KIND_BN nor DWT_KIND_WHITEN (latent-domain site)"),
    (dict(kind=1, gs=4), -1, b"a batch-norm latent-domain site takes group_size 1"),
    (dict(kind=0, gs=8), -4, b"a whitening latent-domain site runs at group sizes 1, 2, 4 only"),
    (dict(kind=0, gs=64), -4, b"latent-domain site"),
    (dict(epi=8), -1, b"bad epilogue"), (dict(epi=2), -1, b"RELU epilogue needs AFFINE"),
    (dict(epi=5), -1, b"RESIDUAL epilogue needs AFFINE|RELU"),
    (dict(epi=0), -1, b"gamma and beta exactly with the AFFINE epilogue"),
    (dict(gamma=None, beta=None), -1, b"gamma and beta exactly with the AFFINE epilogue"),
    (dict(beta=None), -1, b"gamma and beta exactly"),
    (dict(gamma=_FAKE + 2), -1, b"gamma and beta must be 4-byte aligned (latent-domain site)"),
    (dict(mask=_FAKE), -1, b"ReLU byte map exactly with the channels-last RESIDUAL epilogue"),
    (dict(epi=7, res=_FAKE, mask=_FAKE), -1, b"ReLU byte map exactly"),         # NCHW residual: no byte map
    (dict(epi=7, res=_FAKE, mode=0x100), -1, b"ReLU byte map exactly"),          # channels-last residual needs one
    (dict(epi=7, res=_FAKE + 4, mask=_FAKE, mode=0x100), -1, b"must be 16-byte aligned (latent-domain site)"),
    (dict(epi=7, res=_FAKE + 4, mask=_FAKE, mode=0x300), -1, b"must be 8-byte aligned (latent-domain site)"),
    (dict(epi=7, res=None, mask=_FAKE, mode=0x100), -1, b"exactly with the RESIDUAL epilogue"),
    (dict(epi=3, res=_FAKE), -1, b"exactly with the RESIDUAL epilogue"),
    # the layers' own refusals follow
    (dict(kind=1, D=9), -1, b"n_domains 9 outside [1,8] (latent-domain batch norm)"),
    (dict(kind=0, gs=4, D=0), -1, b"(latent-domain whitening)"),
    (dict(kind=1, C=6, mode=0x100), -4, b"latent-domain batch norm runs channels-last at C % 4 == 0 only"),
    (dict(kind=0, gs=2, C=6, mode=0x100), -4, b"latent-domain whitening at group sizes 1, 2, 4 runs channels-last"),
    (dict(kind=0, gs=4, C=6), -4, b"needs group_size 1, 2 or 4 dividing C"),
    (dict(kind=1, x=_FAKE + 4), -1, b"activation tensors must be 16-byte aligned (latent-domain batch norm)"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    if call is _site_bwd and kw.get("epi") == 7 and "res" in kw and kw.get("mode", 0) & 0x100 == 0 and kw.get("mask"):
        text = b"NCHW latent-domain site's residual backward"                 # checked first in the backward
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


@pytest.mark.parametrize("call", [_site_fwd, _site_bwd])
@pytest.mark.parametrize("kw", [dict(kind=1, D=9), dict(kind=0, gs=4, C=6), dict(kind=1, x=_FAKE + 4)])
def test_layer_refusals_name_the_site(lib, call, kw):
    assert call(lib, **kw) != 0
    assert lib.dwt_last_error().endswith(b" [latent-domain site]"), lib.dwt_last_error()


def test_nchw_residual_backward_is_refused(lib):
    assert _site_bwd(lib, epi=7, res=_FAKE) == -1
    assert b"NCHW latent-domain site's residual backward is the AFFINE one" in lib.dwt_last_error()


def test_backward_affine_gradients_need_affine(lib):
    assert _site_bwd(lib, epi=0, gamma=None, beta=None, dgamma=_FAKE) == -1
    assert b"dgamma and dbeta go together and need the AFFINE epilogue" in lib.dwt_last_error()


@pytest.mark.parametrize("kind, gs", [(1, 1), (0, 1), (0, 2), (0, 4)])
@pytest.mark.parametrize("epi, mode, res, mask", [(3, 0, None, None), (7, 0x100, _FAKE, _FAKE), (7, 0, _FAKE, None)])
def test_valid_site_calls_pass_every_check_up_to_the_workspace(lib, kind, gs, epi, mode, res, mask):
    p = ctypes.c_void_p(_FAKE)
    rc = lib.dwt_latent_site_fwd(kind, p, p, 8, 64, 784, gs, 3, mode, 1e-5, 0.1, 1, p, p, p, p, p, _fp(res), _fp(mask),
                                 epi, p, p, p, p, 256, None)
    assert rc == -2 and b"workspace too small" in lib.dwt_last_error()


# =========================================================================== CPU: module and functional errors
def test_module_and_functional_argument_errors():
    import dwt_b200
    from dwt_b200 import functional as F
    x, w = torch.zeros(4, 8, 5, 5), torch.full((4, 3), 1 / 3)
    bn = dwt_b200.LatentDomainBatchNorm2d(8, 3, affine=False)
    with pytest.raises(ValueError, match="needs the layer's affine parameters"):
        bn(x, w, relu=True)
    with pytest.raises(ValueError, match="needs the layer's affine parameters"):
        bn(x, w, residual=x)
    m = dwt_b200.LatentDomainWTransform2d(8, 4, 3)
    g, b = torch.ones(8), torch.zeros(8)
    with pytest.raises(ValueError, match="weight and bias together"):
        m(x, w, gamma=g)
    with pytest.raises(ValueError, match="needs weight and bias"):
        m(x, w, relu=True)
    with pytest.raises(ValueError, match="needs relu=True"):
        m(x, w, gamma=g, beta=b, residual=x)
    with pytest.raises(ValueError, match="shaped like x"):
        m(x, w, gamma=g, beta=b, relu=True, residual=x[:2])
    kw = dict(training_stats=True, eps=1e-5, momentum=0.1, update_running=False, running=(None, None))
    with pytest.raises(ValueError, match="needs relu=True"):
        F.latent_domain_batch_norm(x, w, g, b, residual=x, **kw)
    with pytest.raises(ValueError, match="needs weight and bias"):
        F.latent_domain_batch_norm(x, w, None, None, relu=True, **kw)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        F.latent_domain_batch_norm(x, w, g, b, relu=True, **kw)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(x, w, gamma=g, beta=b, relu=True)


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nlatent-domain sites, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-60s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b, bound=BOUND):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= bound, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


class Case:
    """Inputs of one site call: x, dout, weights, gamma, beta, residual, running buffers (float32, on dev)."""

    def __init__(self, kind, shape, gs, d, dev, seed=0, wkind="softmax"):
        g = torch.Generator(device=dev).manual_seed(seed)
        n, c = shape[:2]
        self.kind, self.gs, self.d = kind, (1 if kind == "bn" else gs), d
        self.eps = 1e-5 if kind == "bn" else 1e-3
        bshape = (n, c) + (1,) * (len(shape) - 2)
        self.x = torch.randn(shape, device=dev, generator=g) + 1.5 * torch.randn(bshape, device=dev, generator=g) + 0.5
        self.dout = torch.randn(shape, device=dev, generator=g) + 0.2
        self.res = torch.randn(shape, device=dev, generator=g)
        self.gamma = 1.0 + 0.3 * torch.randn(c, device=dev, generator=g)
        self.beta = 0.2 * torch.randn(c, device=dev, generator=g)
        if wkind == "softmax":
            self.w = torch.softmax(2.0 * torch.randn(n, d, device=dev, generator=g), 1)
        else:
            self.w = torch.zeros(n, d, device=dev)
            self.w[torch.arange(n, device=dev), torch.arange(n, device=dev) % d] = 1.0
        gs = self.gs
        self.rm = 0.1 * torch.randn(d, c, device=dev, generator=g)
        if kind == "bn":
            self.rv = 1.0 + 0.2 * torch.rand(d, c, device=dev, generator=g)
        else:
            self.rv = (1.2 * torch.eye(gs, device=dev)).expand(d, c // gs, gs, gs).contiguous()

    def running(self):
        return self.rm.clone(), self.rv.clone()


def site_call(cs, epi, layout="nchw", mode="train", dtype=torch.float32, running=None, x=None, dout=None, w=None,
              res=None):
    """One forward + backward of the site under epilogue epi -> dict of y, dx, dw, dgamma, dbeta, dres and the running
    buffers (updated in place in train mode)."""
    from dwt_b200 import functional as F
    x = cs.x if x is None else x
    w = cs.w if w is None else w
    dout = cs.dout if dout is None else dout
    res = cs.res if res is None else res
    fmt = torch.channels_last if layout == "cl" else torch.contiguous_format
    xg = x.to(dtype).contiguous(memory_format=fmt).detach().requires_grad_(True)
    wg = w.detach().clone().requires_grad_(True)
    affine = epi != "none"
    gg = cs.gamma.detach().clone().requires_grad_(True) if affine else None
    bg = cs.beta.detach().clone().requires_grad_(True) if affine else None
    rg = res.to(dtype).contiguous(memory_format=fmt).detach().requires_grad_(True) if epi == "residual" else None
    relu = epi in ("relu", "residual")
    running = cs.running() if running is None else running
    kw = dict(training_stats=mode != "eval", eps=cs.eps, momentum=0.1, update_running=mode == "train", running=running)
    if cs.kind == "bn":
        y = F.latent_domain_batch_norm(xg, wg, gg, bg, relu=relu, residual=rg, **kw)
    else:
        y = F.latent_domain_whiten(xg, wg, group_size=cs.gs, weight=gg, bias=bg, relu=relu, residual=rg, **kw)
    y.backward(dout.to(dtype).contiguous(memory_format=fmt))
    return dict(y=y.detach(), dx=xg.grad, dw=wg.grad, dgamma=None if gg is None else gg.grad,
                dbeta=None if bg is None else bg.grad, dres=None if rg is None else rg.grad, running=running)


def ref_call(cs, epi, mode="train", mask=None):
    """The float64 composition's outputs and gradients.  mask: the fp32 call's ReLU pass map (out != 0), so that a
    pre-activation within rounding of 0 takes the kernels' side of the ReLU instead of counting as a gradient error.
    The forward's ReLU decision is therefore checked separately: compare() bounds the number of elements where that
    map and the float64 pre-activation's sign disagree (returned as "pre")."""
    x = cs.x.double().requires_grad_(True)
    w = cs.w.double().requires_grad_(True)
    affine = epi != "none"
    g = cs.gamma.double().requires_grad_(True) if affine else None
    b = cs.beta.double().requires_grad_(True) if affine else None
    r = cs.res.double().requires_grad_(True) if epi == "residual" else None
    running = None if mode != "eval" else (cs.rm.double(), cs.rv.double())
    relu = epi in ("relu", "residual")
    pre = _ref_site(cs.kind, x, w, cs.gs, g, b, False, r, running, cs.eps)
    y = torch.relu(pre) if relu else pre
    pre.backward(cs.dout.double() * mask if relu else cs.dout.double())
    return dict(y=y.detach(), dx=x.grad, dw=w.grad, dgamma=None if g is None else g.grad,
                dbeta=None if b is None else b.grad, dres=None if r is None else r.grad,
                pre=pre.detach() if relu else None)


def compare(worst, label, got, want):
    if want.get("pre") is not None:      # the ReLU decisions: fp32 out != 0 against float64 pre > 0
        flips = int(((got["y"] != 0) != (want["pre"] > 0)).sum())
        worst.setdefault(label, {})["relu flips"] = (float(flips), flips / want["pre"].numel())
        assert flips <= max(16, 1e-5 * want["pre"].numel()), f"{label}: {flips} ReLU decisions differ"
    for k in ("y", "dx", "dgamma", "dbeta", "dres"):
        if want[k] is not None:
            check(worst, label, k, got[k], want[k])
    check(worst, label, "dw", got["dw"], want["dw"], DW_BOUND)


def plain_running(cs, mode, layout):
    """The running buffers after the layer without an epilogue: the site changes nothing of the statistics."""
    return site_call(cs, "none", layout, mode)["running"]


MODEL_SITES = [("whiten", (192, 64, 112, 112), 4), ("whiten", (192, 256, 56, 56), 4), ("bn", (192, 512, 28, 28), 1),
               ("bn", (192, 1024, 14, 14), 1), ("bn", (192, 2048, 7, 7), 1)]


@gpu
@pytest.mark.parametrize("layout", ["nchw", "cl"])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("kind, shape, gs", MODEL_SITES)
def test_model_sites_against_float64(dev, worst, kind, shape, gs, epi, layout):
    cs = Case(kind, shape, gs, 3, dev)
    got = site_call(cs, epi, layout)
    compare(worst, f"{kind} {list(shape)} {layout} {epi}", got, ref_call(cs, epi, mask=(got["y"] != 0).double()))
    for a, b in zip(got["running"], plain_running(cs, "train", layout)):
        assert torch.equal(a, b)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval", "notrack"])
@pytest.mark.parametrize("d", [3, 8])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("kind, shape, gs, layout", [
    ("bn", (16, 64, 28, 28), 1, "nchw"), ("bn", (16, 64, 28, 28), 1, "cl"), ("bn", (13, 6, 5, 5), 1, "nchw"),
    ("bn", (64, 100), 1, "nchw"), ("whiten", (16, 64, 28, 28), 1, "cl"), ("whiten", (16, 64, 28, 28), 2, "nchw"),
    ("whiten", (16, 64, 28, 28), 4, "cl"), ("whiten", (13, 8, 5, 5), 4, "nchw"), ("whiten", (13, 6, 5, 5), 2, "nchw"),
    # channels-last widths off the power-of-two slabs: C/4 = 3 and 25 (qc does not divide 256), 65 (a 1-column last slab)
    ("bn", (8, 12, 14, 14), 1, "cl"), ("bn", (8, 100, 7, 7), 1, "cl"), ("bn", (4, 260, 7, 7), 1, "cl"),
    ("whiten", (8, 12, 14, 14), 1, "cl"), ("whiten", (8, 100, 7, 7), 2, "cl"), ("whiten", (4, 260, 7, 7), 1, "cl")])
def test_modes_and_edges_against_float64(dev, worst, kind, shape, gs, layout, epi, d, mode):
    if len(shape) == 2 and epi not in ("none", "relu"):
        pytest.skip("[N, C]: batch norm with ReLU")
    cs = Case(kind, shape, gs, d, dev, seed=d)
    got = site_call(cs, epi, layout, mode)
    compare(worst, f"{kind} gs{gs} {list(shape)} {layout} D{d} {mode} {epi}", got,
            ref_call(cs, epi, mode, mask=(got["y"] != 0).double()))
    for a, b in zip(got["running"], plain_running(cs, mode, layout)):
        assert torch.equal(a, b)


def _composition(cs, epi, layout, x=None, w=None):
    """The layer without an epilogue, then gamma / beta, the residual and the ReLU as ATen ops (fp32)."""
    from dwt_b200 import functional as F
    fmt = torch.channels_last if layout == "cl" else torch.contiguous_format
    xg = (cs.x if x is None else x).contiguous(memory_format=fmt).detach().requires_grad_(True)
    wg = (cs.w if w is None else w).detach().clone().requires_grad_(True)
    gg, bg = cs.gamma.detach().clone().requires_grad_(True), cs.beta.detach().clone().requires_grad_(True)
    rg = cs.res.contiguous(memory_format=fmt).detach().requires_grad_(True)
    kw = dict(training_stats=True, eps=cs.eps, momentum=0.1, update_running=True, running=cs.running())
    if cs.kind == "bn":
        y = F.latent_domain_batch_norm(xg, wg, gg, bg, **kw)
    else:
        shape = (1, -1, 1, 1)
        y = F.latent_domain_whiten(xg, wg, group_size=cs.gs, **kw) * gg.view(shape) + bg.view(shape)
    if epi == "residual":
        y = y + rg
    if epi in ("relu", "residual"):
        y = torch.relu(y)
    y.backward(cs.dout.contiguous(memory_format=fmt))
    return dict(y=y.detach(), dx=xg.grad, dw=wg.grad, dgamma=gg.grad, dbeta=bg.grad, dres=rg.grad if epi == "residual" else None)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "cl"])
@pytest.mark.parametrize("epi", ["affine", "relu", "residual"])
@pytest.mark.parametrize("shape", [(64, 256, 28, 28), (32, 64, 7, 7), (13, 8, 5, 5)])
def test_batch_norm_sites_equal_the_aten_composition_bit_for_bit(dev, shape, epi, layout):
    cs = Case("bn", shape, 1, 3, dev)
    got, want = site_call(cs, epi, layout), _composition(cs, epi, layout)
    for k in ("y", "dx", "dw", "dgamma", "dbeta", "dres"):
        if want[k] is not None:
            assert torch.equal(got[k], want[k]), (k, float((got[k] - want[k]).abs().max()))


@gpu
@pytest.mark.parametrize("layout", ["nchw", "cl"])
@pytest.mark.parametrize("epi", ["affine", "relu", "residual"])
@pytest.mark.parametrize("kind, gs", [("whiten", 1), ("whiten", 2), ("whiten", 4)])
def test_whitening_sites_agree_with_the_aten_composition(dev, worst, kind, gs, epi, layout):
    cs = Case(kind, (32, 64, 28, 28), gs, 3, dev)
    got, want = site_call(cs, epi, layout), _composition(cs, epi, layout)
    for k in ("y", "dx", "dgamma", "dbeta", "dres"):
        if want[k] is not None:
            check(worst, f"whiten gs{gs} vs ATen {layout} {epi}", k, got[k], want[k], 2e-6)
    check(worst, f"whiten gs{gs} vs ATen {layout} {epi}", "dw", got["dw"], want["dw"], 1e-5)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "cl"])
@pytest.mark.parametrize("epi", ["affine", "relu", "residual"])
@pytest.mark.parametrize("kind, gs", [("bn", 1), ("whiten", 1), ("whiten", 2), ("whiten", 4)])
def test_bf16_is_the_fp32_call_on_widened_inputs_rounded(dev, kind, gs, epi, layout):
    cs = Case(kind, (16, 64, 28, 28), gs, 3, dev)
    xb, rb, db = cs.x.bfloat16(), cs.res.bfloat16(), cs.dout.bfloat16()
    got = site_call(cs, epi, layout, dtype=torch.bfloat16, x=xb, dout=db, res=rb)
    want = site_call(cs, epi, layout, x=xb.float(), dout=db.float(), res=rb.float())
    for k in ("y", "dx", "dres"):
        if want[k] is not None:
            assert got[k].dtype == torch.bfloat16 and torch.equal(got[k], want[k].bfloat16()), k
    for k in ("dw", "dgamma", "dbeta"):
        assert torch.equal(got[k], want[k]), k
    for a, b in zip(got["running"], want["running"]):
        assert torch.equal(a, b)


@gpu
@pytest.mark.parametrize("layout", ["nchw", "cl"])
@pytest.mark.parametrize("kind, gs", [("bn", 1), ("whiten", 4)])
def test_reruns_and_graph_replay_are_bit_identical(dev, kind, gs, layout):
    from dwt_b200 import functional as F
    cs = Case(kind, (16, 64, 28, 28), gs, 3, dev)
    outs = [site_call(cs, epi, layout) for epi in ("relu", "residual") for _ in range(2)]
    for a, b in ((outs[0], outs[1]), (outs[2], outs[3])):
        for k in ("y", "dx", "dw", "dgamma", "dbeta"):
            assert torch.equal(a[k], b[k]), k
    fmt = torch.channels_last if layout == "cl" else torch.contiguous_format
    x = cs.x.contiguous(memory_format=fmt).detach().requires_grad_(True)
    r = cs.res.contiguous(memory_format=fmt).detach().requires_grad_(True)
    w = cs.w.clone().requires_grad_(True)
    g, b = cs.gamma.clone().requires_grad_(True), cs.beta.clone().requires_grad_(True)
    dout = cs.dout.contiguous(memory_format=fmt)
    rm, rv = cs.running()

    def step():
        kw = dict(training_stats=True, eps=cs.eps, momentum=0.1, update_running=False, running=(rm, rv))
        if kind == "bn":
            y = F.latent_domain_batch_norm(x, w, g, b, relu=True, residual=r, **kw)
        else:
            y = F.latent_domain_whiten(x, w, group_size=gs, weight=g, bias=b, relu=True, residual=r, **kw)
        return (y,) + torch.autograd.grad(y, (x, w, g, b, r), dout)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):                                 # warm-up on the side stream
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    for a, c in zip(eager, static):
        assert torch.equal(a, c)


def _edge_weights(cs, rule):
    w = cs.w.clone()
    if rule == "zero_mass":
        w[:, -1] = 0.0
    elif rule == "nan_weight":
        w[3, 1] = float("nan")
    else:                                                  # an image with no positive mix
        w[5] = 0.0
    return w


@gpu
@pytest.mark.parametrize("layout", ["nchw", "cl"])
@pytest.mark.parametrize("epi", ["relu", "residual"])
@pytest.mark.parametrize("rule", ["zero_mass", "nan_weight", "no_mix"])
@pytest.mark.parametrize("kind, gs", [("bn", 1), ("whiten", 2)])
def test_edge_rules_hold_under_an_epilogue(dev, kind, gs, rule, epi, layout):
    cs = Case(kind, (12, 16, 14, 14), gs, 3, dev)
    w = _edge_weights(cs, rule)
    got, want = site_call(cs, epi, layout, w=w), _composition(cs, epi, layout, w=w)
    for k in ("y", "dx", "dgamma", "dbeta", "dres"):
        if want[k] is None:
            continue
        a, b = got[k], want[k]
        assert torch.equal(torch.isnan(a), torch.isnan(b)), k
        if kind == "bn":
            assert torch.equal(a, b) or torch.equal(torch.nan_to_num(a), torch.nan_to_num(b)), k
        else:
            assert torch.allclose(torch.nan_to_num(a), torch.nan_to_num(b), rtol=1e-4, atol=1e-5), k
    if rule == "zero_mass":
        assert torch.equal(got["dw"][:, -1], torch.zeros_like(got["dw"][:, -1]))


@gpu
def test_tensor_core_group_sizes_run_the_site_as_tensor_ops(dev):
    from dwt_b200 import functional as F
    cs = Case("whiten", (16, 64, 16, 16), 16, 3, dev)
    kw = dict(group_size=16, training_stats=True, eps=1e-3, momentum=0.1, update_running=False, running=cs.running())
    y = F.latent_domain_whiten(cs.x, cs.w, weight=cs.gamma, bias=cs.beta, relu=True, residual=cs.res, **kw)
    z = F.latent_domain_whiten(cs.x, cs.w, **kw)
    assert torch.equal(y, torch.relu(z * cs.gamma.view(1, -1, 1, 1) + cs.beta.view(1, -1, 1, 1) + cs.res))


@gpu
def test_modules_run_the_site(dev):
    import dwt_b200
    cs = Case("bn", (8, 32, 7, 7), 1, 3, dev)
    bn = dwt_b200.LatentDomainBatchNorm2d(32, 3).to(dev)
    y = bn(cs.x, cs.w, relu=True, residual=cs.res)
    bn2 = dwt_b200.LatentDomainBatchNorm2d(32, 3).to(dev)
    assert torch.equal(y, torch.relu(bn2(cs.x, cs.w) + cs.res))
    wt = dwt_b200.LatentDomainWTransform2d(32, 4, 3).to(dev)
    y = wt(cs.x, cs.w, gamma=cs.gamma, beta=cs.beta, relu=True)
    assert torch.isfinite(y).all() and (y >= 0).all()


# =========================================================================== the latent ResNet-50-DWT (harness)
def _latent_model(sd, site_mode="modules", channels_last=False, num_domains=3):
    import dwt_b200
    from harness.resnet50_dwt import build_resnet50_dwt
    return build_resnet50_dwt(sd, dwt_b200, site_mode=site_mode, domains="latent", num_domains=num_domains,
                              channels_last=channels_last)


def test_latent_harness_builds_from_the_checkpoint():
    from harness.synth import synth_state_dict
    sd = synth_state_dict(seed=1)
    m = _latent_model(sd)
    params = dict(m.named_parameters())
    bufs = dict(m.named_buffers())
    # convolution and fc weights under the DWT model's names, loaded from the checkpoint
    for k in ("conv1.weight", "layer1.0.conv1.weight", "layer2.0.downsample.0.weight", "fc_out.weight", "fc_out.bias"):
        assert torch.equal(params[k].detach(), sd[k]), k
    # whitening sites (stem, layer1): the latent layer's K buffer pairs and the site's gamma / beta
    assert params["bn1.gamma"].shape == (64,) and torch.equal(params["bn1.gamma"].detach(), sd["bn1.gamma"].reshape(64))
    assert torch.equal(params["layer1.0.downsample_bn.beta"].detach(), sd["layer1.0.downsample_bn.beta"].reshape(256))
    for d in range(3):
        assert torch.equal(bufs["bn1.norm.running_mean"][d], sd["bn1.wh.running_mean"].reshape(64))
        assert torch.equal(bufs["layer1.2.bn3.norm.running_variance"][d], sd["layer1.2.bn3.wh.running_variance"])
        # batch-norm sites (layers 2-4): the layer's own weight / bias are the site's gamma / beta
        assert torch.equal(bufs["layer3.4.bn2.norm.running_var"][d], sd["layer3.4.bn2.running_var"])
        assert torch.equal(bufs["layer4.0.downsample_bn.norm.running_mean"][d], sd["layer4.0.downsample_bn.running_mean"])
    assert torch.equal(params["layer2.0.bn1.norm.weight"].detach(), sd["layer2.0.bn1.weight"])
    assert bufs["layer1.0.bn1.norm.running_mean"].shape == (3, 64)
    assert bufs["layer1.0.bn1.norm.running_variance"].shape == (3, 16, 4, 4)
    assert "bn1.norm.weight" not in params and "layer2.0.bn1.gamma" not in params
    # every site of ResNet50DWT has one LatentSite: the stem + 16 blocks x 3 + 4 downsample sites
    from harness.resnet50_dwt import LatentSite
    assert sum(isinstance(x, LatentSite) for x in m.modules()) == 53
    with pytest.raises(ValueError, match="domains must be"):
        from harness.resnet50_dwt import build_resnet50_dwt
        import dwt_b200
        build_resnet50_dwt(sd, dwt_b200, domains="soft")


def _dwt_site_params(model):
    """{latent parameter name: the DWT model's gamma / beta parameter} for every site."""
    out = {}
    for owner_name, owner in model.named_modules():
        for tag, (_, gname, bname, whiten) in getattr(owner, "_sites", {}).items():
            pre = owner_name + "." if owner_name else ""
            site = pre + ("downsample_bn" if tag == "downsample" else f"bn{tag}")
            g, b = ("gamma", "beta") if whiten else ("norm.weight", "norm.bias")
            out[f"{site}.{g}"] = getattr(owner, gname)
            out[f"{site}.{b}"] = getattr(owner, bname)
    return out


def _step(model, x, labels, weights=None):
    model.zero_grad(set_to_none=True)
    logits = model(x) if weights is None else model(x, weights)
    n = labels.shape[0]
    loss = torch.nn.functional.cross_entropy(logits[:n].float(), labels) + 0.1 * logits.float().square().mean()
    loss.backward()
    return logits.detach().float(), loss.detach()


@pytest.fixture
def no_tf32():
    """Model comparisons: cuDNN's default TF32 convolutions would differ by ~1e-3 per layer between two runs of the same
    network and swamp the sites' differences; full fp32 convolutions, deterministic algorithms."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic = old


# logits and loss (norm-wise); each parameter's gradient (norm-wise).  The gradients are the looser bound: the synthetic
# checkpoint's 53-site backward at 4 images per domain amplifies last-bit differences of the forward (logits agree to
# ~2e-5) to ~2e-2 in every stage, between two runs that differ only in the whitening sites' rounding.
MODEL_BOUND = (1e-4, 5e-2)


def _stem(name):
    return name.startswith(("conv1.", "bn1.", "layer1."))


def _check_grads(worst, label, pairs):
    """pairs: (name, grad, reference grad); every parameter within MODEL_BOUND[1]; the worst of the whitening stages
    (stem, layer1) and of the rest recorded."""
    worst_stem = worst_rest = 0.0
    bad = []
    for name, a, b in pairs:
        r, _ = rel(a.reshape(-1), b.reshape(-1))
        if _stem(name):
            worst_stem = max(worst_stem, r)
        else:
            worst_rest = max(worst_rest, r)
        if r > MODEL_BOUND[1]:
            bad.append((name, r))
    worst.setdefault(label, {})["grads stem + layer1 (worst)"] = (worst_stem, worst_stem)
    worst.setdefault(label, {})["grads layers 2-4, fc (worst)"] = (worst_rest, worst_rest)
    assert not bad, bad


def _thirds(n, dev):
    w = torch.zeros(3 * n, 3, device=dev)
    w[torch.arange(3 * n, device=dev), torch.arange(3 * n, device=dev) // n] = 1.0
    return w


@gpu
def test_one_hot_thirds_reproduce_the_dwt_model(dev, worst, no_tf32):
    import dwt_b200
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
    x, y = synth_batch(seed=2, per_domain=4, size=128)
    x, y = x.to(dev), y.to(dev)
    dwt = build_resnet50_dwt(sd, dwt_b200, site_mode="modules").to(dev).train()
    lat = _latent_model(sd, "modules").to(dev).train()
    la, ls = _step(dwt, x, y)
    lb, lt = _step(lat, x, y, _thirds(4, dev))
    label = "latent model one-hot thirds vs DWT modules"
    check(worst, label, "logits", lb, la, MODEL_BOUND[0])
    check(worst, label, "loss", lt, ls, MODEL_BOUND[0])
    dwt_p, site_p = dict(dwt.named_parameters()), _dwt_site_params(dwt)
    _check_grads(worst, label, [(name, p.grad, (site_p[name] if name in site_p else dwt_p[name]).grad)
                                for name, p in lat.named_parameters()])


@gpu
@pytest.mark.parametrize("channels_last", [False, True])
def test_fused_and_modules_latent_models_agree(dev, worst, channels_last, no_tf32):
    from harness.synth import synth_batch, synth_state_dict
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=3).items()}
    x, y = synth_batch(seed=4, per_domain=4, size=128)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    x, y = x.to(dev).contiguous(memory_format=fmt), y.to(dev)
    w = torch.softmax(torch.randn(12, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(5)), 1)
    mods = _latent_model(sd, "modules", channels_last).to(dev).train()
    fused = _latent_model(sd, "fused", channels_last).to(dev).train()
    la, ls = _step(mods, x, y, w)
    lb, lt = _step(fused, x, y, w)
    label = f"latent model fused vs modules {'cl' if channels_last else 'nchw'}"
    check(worst, label, "logits", lb, la, MODEL_BOUND[0])
    check(worst, label, "loss", lt, ls, MODEL_BOUND[0])
    pa = dict(mods.named_parameters())
    _check_grads(worst, label, [(name, p.grad, pa[name].grad) for name, p in fused.named_parameters()])
    bm, bf = dict(mods.named_buffers()), dict(fused.named_buffers())
    for k in bm:
        if bm[k].is_floating_point():
            assert rel(bf[k], bm[k])[0] <= 1e-4, k


@gpu
@pytest.mark.parametrize("autocast", [False, True])
def test_channels_last_step_runs_in_fp32_and_under_bf16_autocast(dev, autocast):
    from harness.synth import synth_batch, synth_state_dict
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=5).items()}
    x, y = synth_batch(seed=6, per_domain=4, size=128)
    x, y = x.to(dev).contiguous(memory_format=torch.channels_last), y.to(dev)
    model = _latent_model(sd, "fused", channels_last=True).to(dev).train()
    w = torch.softmax(torch.randn(12, 3, device=dev), 1)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        logits, loss = _step(model, x, y, w)
    assert torch.isfinite(loss) and torch.isfinite(logits).all()
    for name, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name


@gpu
def test_sgd_with_a_softmax_domain_branch_lowers_the_loss(dev):
    from harness.synth import synth_batch, synth_state_dict
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=7).items()}
    x, y = synth_batch(seed=8, per_domain=4, size=128)
    x, y = x.to(dev).contiguous(memory_format=torch.channels_last), y.to(dev)
    model = _latent_model(sd, "fused", channels_last=True).to(dev).train()
    g = torch.Generator().manual_seed(9)
    branch = torch.nn.Linear(3 * 8 * 8, 3).to(dev)
    with torch.no_grad():
        branch.weight.copy_(0.05 * torch.randn(3, 192, generator=g))
    opt = torch.optim.SGD(list(model.parameters()) + list(branch.parameters()), lr=0.002)
    losses = []
    for it in range(4):
        opt.zero_grad(set_to_none=True)
        w = torch.softmax(branch(torch.nn.functional.adaptive_avg_pool2d(x, 8).flatten(1)), 1)
        logits = model(x, w)
        loss = torch.nn.functional.cross_entropy(logits[:4], y) + 0.1 * logits.square().mean()
        loss.backward()
        if it == 0:
            for p in branch.parameters():
                assert torch.isfinite(p.grad).all() and p.grad.abs().max() > 0
        opt.step()
        losses.append(float(loss))
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
