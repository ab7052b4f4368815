"""Channels-last whitening at group sizes 8..64 on the tensor-core kernels, against the NCHW tensor-core call, bit for bit.

A dense channels-last whitening call on a tensor-core geometry (group size 8, 16, 32, 64; HW >= 32 and a multiple of 4;
at least 4096 samples per domain; 16-byte-aligned tensors) runs tc_stats / tc_apply / tc_bwd_reduce / tc_bwd_apply on the
NHWC tensor itself (DWT_LAYOUT_NHWC): the NCHW schedule of its shape, tiles read through a channels-innermost tensor map
and transposed in shared memory (include/dwt_b200.h).  So every comparison here is torch.equal, with NaN equal to NaN,
against the NCHW call on x.contiguous(): y, dx, save_mean / save_w, every running buffer and the status word; y and dx
come back channels-last.

  * group sizes 8/16/32/64, C = 64, 96 (a partial super-block) and 256, HW = 32, 36 (a partial 32-pixel tile), 12544
    (the stem) and 3136, N * HW = 4096 exactly, 1 to 4 domains on shared / distinct / mixed running buffers;
  * train, no-grad train, eval forward + backward, default buffers, DomainTripleNorm at gs 8 and 64 (gamma / beta / ReLU,
    a residual, dgamma and dbeta);
  * BASELINE config 2 (N=256 C=256 56^2 gs 64), the two pilot-shift inputs at that size, a NaN input, no copy of x;
  * bf16: the NHWC bf16 call is the NHWC fp32 call on x.float(), rounded, and (HW % 8 == 0) the NCHW bf16 call;
  * routing edges that keep the NCHW copy (a misaligned view, HW % 4 != 0, N * HW < 4096, gs 12) against the fp64
    oracle, and a forked gs-64 output;
  * C = 8, 16, 32: channel boxes wider than the tensor;
  * return codes of the C ABI; CUDA-graph capture and replay in fp32 and bf16;
  * the harness ResNet-50-DWT at group_size=64, channels-last, fused, against the NCHW port.
"""
import ctypes
import time

import pytest
import torch

from conftest import max_err, rel_err
from oracle import dwt_oracle as O

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
CL = torch.channels_last


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    d = torch.device("cuda", 0)
    t0 = time.perf_counter()
    yield d
    print(f"\ntest_channels_last_tensor_core: {time.perf_counter() - t0:.1f} s")


def _same(a, b):
    """torch.equal of the values (any memory format), with NaN equal to NaN."""
    if a is None or b is None:
        return a is None and b is None
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.isnan(), b.isnan()) and \
        torch.equal(a.nan_to_num(0.0), b.nan_to_num(0.0))


def _is_cl(t):
    return t.is_contiguous(memory_format=CL) and not t.is_contiguous()


def _activation(gen, shape, d, dev):
    """float32 activations: correlated neighbouring channels, per-channel scales, a mean per domain."""
    z = torch.randn(shape, device=dev, generator=gen)
    z.add_(z.roll(1, 1), alpha=0.6)
    z.mul_(0.5 + torch.rand(shape[1], 1, 1, device=dev, generator=gen))
    n = shape[0] // d
    for k in range(d):
        z[k * n:(k + 1) * n].add_(0.6 * k - 0.5)
    return z


def _microbench(gen, shape, d, dev):
    """bench.py's microbench input: x = mix . randn + 2.0 (BASELINE.json configs[1])."""
    n, c, h, w = shape
    mix = torch.randn(c, c, device=dev, generator=gen) / c ** 0.5 + torch.eye(c, device=dev)
    return (torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, h, w, device=dev, generator=gen)) + 2.0).contiguous()


def _pilot_30sigma(gen, shape, d, dev):
    """Image 0 of every domain 30 sigma off in the pilot window (the <= 32 mid-image pixels K is estimated from)."""
    x = _microbench(gen, shape, d, dev)
    n, hw = shape[0] // d, shape[2] * shape[3]
    npx = min(hw, 32)
    p0 = ((hw - npx) // 2) & ~3
    flat = x.view(shape[0], shape[1], hw)
    for k in range(d):
        sigma = x[k * n:(k + 1) * n].std(dim=(0, 2, 3))
        flat[k * n, :, p0:p0 + npx] += 30.0 * sigma.view(-1, 1)
    return x


def _mean_50sigma(gen, shape, d, dev):
    """|mean| >= 50 sigma in every channel."""
    x = _microbench(gen, shape, d, dev).mul_(0.1).add_(10.0)
    return x.add_(torch.linspace(0.0, 40.0, shape[1], device=dev).view(1, -1, 1, 1))


class _Site:
    """D domains of one whitening site on running buffers aliased 'shared', 'distinct' or 'mixed'; one copy per arm."""

    def __init__(self, c, gs, d, layout, gen, dev):
        self.c, self.gs, self.d = c, gs, d
        self.owner = {"shared": [0] * d, "distinct": list(range(d)), "mixed": [0] + [1] * (d - 1)}[layout]
        self.init = {}
        for o in sorted(set(self.owner)):
            a = torch.randn(c // gs, gs, gs, device=dev, generator=gen)
            self.init[o] = (0.1 * torch.randn(1, c, 1, 1, device=dev, generator=gen),
                            a @ a.transpose(1, 2) / gs + 0.5 * torch.eye(gs, device=dev))

    def buffers(self):
        return {o: (rm.clone(), rv.clone()) for o, (rm, rv) in self.init.items()}


def _norm_node(y):
    """The _NormFunction node behind y (the upcast path puts a dtype cast in front of it)."""
    node = y.grad_fn
    while not type(node).__name__.startswith("_NormFunction"):
        node = node.next_functions[0][0]
    return node


def _run_arm(x, site, mode, g1, g2=None, measure=False):
    """One arm: the site on x as given (layout, dtype, view).  Returns everything to compare."""
    import dwt_b200
    from dwt_b200 import _native as nv, functional as F
    dev = x.device
    bufs = site.buffers()
    running = [bufs[o] for o in site.owner]
    grad = mode in ("train", "eval")
    x = x.detach().requires_grad_(grad)
    nv.clear_status(dev)
    if measure:
        torch.cuda.synchronize(dev)
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
    nv.profile_begin()
    with torch.set_grad_enabled(grad):
        y = F.norm(x, None, None, kind="whiten", group_size=site.gs, n_domains=site.d, training_stats=mode != "eval",
                   eps=1e-3, momentum=0.1, update_running=mode != "eval", running=running)
    out = {"y": y.detach(), "status": nv.status(dev), "stats": None, "dx": None}
    if grad:
        node = _norm_node(y)
        out["stats"] = list(node.saved_tensors[1:3])
        out["route"] = node.cfg[3]
        del node
        if g2 is not None:
            u, v = dwt_b200.fork_for_sum(y)
            torch.autograd.backward([u, v], [g1.to(y.dtype), g2.to(y.dtype)])
        else:
            y.backward(g1.to(y.dtype))
        out["dx"] = x.grad
    out["families"] = set(nv.by_family(nv.profile_end()))
    if measure:
        torch.cuda.synchronize(dev)
        out["peak"] = torch.cuda.max_memory_allocated(dev) - base
    out["running"] = [t for o in sorted(bufs) for t in bufs[o]]
    return out


def _compare(a, ref, cast=None):
    """a against ref (ref's y / dx rounded to `cast` first, if given)."""
    rnd = (lambda t: t.to(cast)) if cast is not None else (lambda t: t)
    assert _same(a["y"], rnd(ref["y"])), "y"
    assert a["status"] == ref["status"], (a["status"], ref["status"])
    for k, (p, q) in enumerate(zip(a["running"], ref["running"])):
        assert _same(p, q), f"running buffer {k}"
    if ref["stats"] is not None:
        for k, (p, q) in enumerate(zip(a["stats"], ref["stats"])):
            assert _same(p, q), f"save_mean / save_w {k}"
        assert _same(a["dx"], rnd(ref["dx"])), "dx"


def _nhwc_families(fams):
    return {f for f in fams if "_nhwc" in f}


def _case(dev, *, c, gs, d, n, hw, mode="train", layout="shared", seed=0, make_x=_activation, nan=False, fork=False,
          measure=False, dtype=torch.float32):
    """The site on channels-last x and on x.contiguous(); asserts every comparison and which kernels ran."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    h, w = hw
    shape = (d * n, c, h, w)
    x = make_x(gen, shape, d, dev).to(dtype)
    if nan:
        x[0, 1, 0, 0] = float("nan")
    site = _Site(c, gs, d, layout, gen, dev)
    g1 = torch.randn(shape, device=dev, generator=gen).to(dtype).contiguous(memory_format=CL)
    g2 = torch.randn(shape, device=dev, generator=gen).to(dtype).contiguous(memory_format=CL) if fork else None
    xcl = x.contiguous(memory_format=CL)
    cl = _run_arm(xcl, site, mode, g1, g2, measure=measure)
    ref = _run_arm(x, site, mode, g1.contiguous(), None if g2 is None else g2.contiguous())
    _compare(cl, ref)
    assert _is_cl(cl["y"]), "y is not channels-last"
    if cl["dx"] is not None:
        assert _is_cl(cl["dx"]), "dx is not channels-last"
    suffix = "_nhwc_bf16" if dtype == BF else "_nhwc"
    tc = {f for f in cl["families"] if f.startswith("tc_")}
    assert tc and all(f.endswith(suffix) for f in tc), sorted(cl["families"])
    assert not _nhwc_families(ref["families"]), sorted(ref["families"])
    return cl, ref


# --------------------------------------------------------------------------- group sizes, shapes, domains, buffers
CASES = [   # gs, C, domains, N per domain, (H, W), running buffers
    (8, 64, 1, 128, (4, 8), "shared"),        # HW = 32: one tile per image; N * HW = 4096 exactly
    (16, 96, 2, 4, (32, 32), "distinct"),     # C = 96: a partial super-block; N * HW = 4096
    (32, 96, 3, 120, (6, 6), "mixed"),        # HW = 36: a partial 32-pixel tile
    (64, 64, 4, 2, (112, 112), "mixed"),      # HW = 12544: the stem site
    (64, 256, 3, 2, (56, 56), "distinct"),    # HW = 3136
    (8, 256, 2, 2, (56, 56), "shared"),
    (16, 64, 1, 114, (6, 6), "shared"),       # HW = 36, N * HW = 4104
    (32, 32, 2, 64, (8, 8), "distinct"),      # C = 32 < 64: the fp32 second channel box lies wholly past C
    (8, 8, 1, 128, (6, 6), "shared"),         # C = 8: one group; HW = 36
]


@pytest.mark.parametrize("gs,c,d,n,hw,layout", CASES,
                         ids=[f"gs{k[0]}-c{k[1]}-d{k[2]}-n{k[3]}-{k[4][0]}x{k[4][1]}-{k[5]}" for k in CASES])
def test_geometries(gs, c, d, n, hw, layout, dev):
    _case(dev, c=c, gs=gs, d=d, n=n, hw=hw, layout=layout, seed=gs + c + d)


MODES = [   # gs, C, domains, N, (H, W), mode, buffers
    (16, 64, 3, 8, (24, 24), "nograd", "mixed"),
    (32, 64, 2, 8, (32, 32), "eval", "distinct"),
    (64, 128, 1, 4, (32, 40), "eval", "shared"),
    (8, 96, 3, 120, (6, 6), "nograd", "distinct"),
    (64, 128, 2, 120, (6, 6), "eval", "mixed"),
]


@pytest.mark.parametrize("gs,c,d,n,hw,mode,layout", MODES,
                         ids=[f"gs{k[0]}-c{k[1]}-d{k[2]}-{k[4][0]}x{k[4][1]}-{k[5]}-{k[6]}" for k in MODES])
def test_modes(gs, c, d, n, hw, mode, layout, dev):
    _case(dev, c=c, gs=gs, d=d, n=n, hw=hw, mode=mode, layout=layout, seed=3 * gs + d)


def test_default_buffers(dev):
    """WTransform2d with its own default buffers (zero mean, all-ones second moment), training, forward + backward."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(21)
    x = torch.randn(4, 64, 32, 32, device=dev, generator=gen) * 2 + 1
    g = torch.randn(x.shape, device=dev, generator=gen)
    ma, mb = dwt_b200.WTransform2d(64, 8).to(dev).train(), dwt_b200.WTransform2d(64, 8).to(dev).train()
    xa, xb = x.contiguous(memory_format=CL).requires_grad_(True), x.clone().requires_grad_(True)
    ya, yb = ma(xa), mb(xb)
    assert ya.grad_fn.cfg[3] & dwt_b200._native.LAYOUT_NHWC, "the channels-last kernels did not run"
    assert _is_cl(ya) and _same(ya, yb)
    ya.backward(g.contiguous(memory_format=CL))
    yb.backward(g)
    assert _is_cl(xa.grad) and _same(xa.grad, xb.grad)
    assert _same(ma.running_mean, mb.running_mean) and _same(ma.running_variance, mb.running_variance)


@pytest.mark.parametrize("gs,residual", [(8, False), (64, True)], ids=["gs8-affine-relu", "gs64-residual"])
def test_domain_triple_norm(gs, residual, dev):
    """A DomainTripleNorm site at gs >= 8 (the kernels, then gamma / beta / ReLU / residual as tensor ops), channels-last
    against NCHW.  y, dx and d(residual) are bit for bit; dgamma and dbeta are ATen reductions over the spatial and batch
    axes, whose summation order follows the memory format, so they agree to fp32 rounding."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(gs)
    c, nper, h = 64, 2, 48                           # N * HW = 4608 per domain
    x = _activation(gen, (3 * nper, c, h, h), 3, dev)
    g = torch.randn(x.shape, device=dev, generator=gen)
    res = torch.randn(x.shape, device=dev, generator=gen) if residual else None
    gamma0 = 0.5 + torch.rand(c, 1, 1, device=dev, generator=gen)
    beta0 = 0.1 * torch.randn(c, 1, 1, device=dev, generator=gen)

    def arm(fmt):
        mods = [dwt_b200.WTransform2d(c, gs).to(dev).train() for _ in range(3)]
        site = dwt_b200.DomainTripleNorm("whiten", c, group_size=gs)
        gamma, beta = gamma0.clone().requires_grad_(True), beta0.clone().requires_grad_(True)
        xi = x.contiguous(memory_format=fmt).requires_grad_(True)
        ri = None if res is None else res.contiguous(memory_format=fmt).requires_grad_(True)
        y = site(xi, mods, gamma, beta, relu=True, residual=ri)
        y.backward(g.contiguous(memory_format=fmt))
        bufs = [t for m in mods for t in (m.running_mean, m.running_variance)]
        return y.detach(), xi.grad, None if ri is None else ri.grad, gamma.grad, beta.grad, bufs
    a, b = arm(CL), arm(torch.contiguous_format)
    assert _is_cl(a[0]) and _is_cl(a[1])
    assert _same(a[0], b[0]) and _same(a[1], b[1]) and _same(a[2], b[2])
    for p, q in zip(a[3:5], b[3:5]):
        torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-4)
    assert all(_same(p, q) for p, q in zip(a[5], b[5]))


# --------------------------------------------------------------------------- the microbench size, pilot inputs, NaN
def test_config2_no_copy_of_x(dev):
    """BASELINE config 2 (N=256 C=256 56^2 gs 64), forward + backward.  The device memory the channels-last call adds
    stays under y + dx + 5 %: no copy of x (NCHW or otherwise) is made."""
    cl, _ = _case(dev, c=256, gs=64, d=1, n=256, hw=(56, 56), make_x=_microbench, seed=0, measure=True)
    xbytes = 256 * 256 * 56 * 56 * 4
    assert cl["peak"] < 2.1 * xbytes, (cl["peak"], xbytes)


@pytest.mark.parametrize("make_x", [_pilot_30sigma, _mean_50sigma], ids=["pilot_30sigma", "mean_50sigma"])
def test_pilot_shift_inputs(make_x, dev):
    _case(dev, c=256, gs=64, d=1, n=256, hw=(56, 56), make_x=make_x, seed=1)


def test_nan_input_sets_the_same_status(dev):
    from dwt_b200 import _native
    cl, _ = _case(dev, c=256, gs=64, d=1, n=256, hw=(56, 56), make_x=_microbench, seed=5, nan=True)
    assert cl["status"] & _native.STATUS_NOT_PD
    _native.clear_status(dev)


# --------------------------------------------------------------------------- bf16
BF_CASES = [   # gs, C, domains, N, (H, W), mode
    (64, 64, 1, 4, (32, 32), "train"),
    (32, 96, 3, 120, (6, 6), "train"),        # HW = 36: accepted channels-last (HW % 4), refused NCHW (HW % 8)
    (16, 256, 2, 2, (56, 56), "eval"),
    (8, 64, 2, 128, (4, 8), "nograd"),
    (16, 16, 1, 120, (6, 6), "train"),        # C = 16: the 64-channel box is four times wider than the tensor
    (32, 32, 2, 64, (8, 8), "train"),
]


@pytest.mark.parametrize("gs,c,d,n,hw,mode", BF_CASES, ids=[f"gs{k[0]}-c{k[1]}-{k[4][0]}x{k[4][1]}-{k[5]}" for k in BF_CASES])
def test_bf16(gs, c, d, n, hw, mode, dev):
    """bf16 channels-last == fp32 channels-last on x.float(), rounded; == bf16 NCHW where HW % 8 == 0.  Only the
    *_nhwc_bf16 tensor-core families run."""
    gen = torch.Generator(device=dev).manual_seed(gs + n)
    shape = (d * n, c) + hw
    x = _activation(gen, shape, d, dev).to(BF).contiguous(memory_format=CL)
    site = _Site(c, gs, d, "mixed", gen, dev)
    g = torch.randn(shape, device=dev, generator=gen).to(BF).contiguous(memory_format=CL)
    a = _run_arm(x, site, mode, g)
    f32 = _run_arm(x.float(), site, mode, g.float())
    assert a["y"].dtype == BF and _is_cl(a["y"])
    _compare(a, f32, cast=BF)
    tc = {f for f in a["families"] if f.startswith("tc_")}
    assert tc and all(f.endswith("_nhwc_bf16") for f in tc), sorted(a["families"])
    assert not any(f.endswith("_bf16") for f in f32["families"])
    if (hw[0] * hw[1]) % 8 == 0:
        _compare(a, _run_arm(x.contiguous(), site, mode, g.contiguous()))


# --------------------------------------------------------------------------- routing edges: the NCHW copy
def _misaligned_cl(x):
    """x's values in a dense channels-last view whose data_ptr() is 4 bytes past a 16-byte boundary."""
    n, c, h, w = x.shape
    buf = torch.empty(x.numel() + 4, dtype=x.dtype, device=x.device)
    v = buf[1:1 + x.numel()].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(x)
    assert _is_cl(v) and v.data_ptr() % 16 == 4
    return v


EDGES = [   # gs, C, N, (H, W), view, what
    (64, 64, 4, (32, 32), _misaligned_cl, "misaligned"),
    (16, 64, 84, (7, 7), None, "hw49"),       # HW % 4 != 0
    (16, 64, 63, (8, 8), None, "nhw4032"),    # N * HW = 4032 < 4096
    (12, 48, 8, (32, 32), None, "gs12"),      # 64 % 12 != 0: the tiled kernels
]


@pytest.mark.parametrize("gs,c,n,hw,view,what", EDGES, ids=[k[5] for k in EDGES])
def test_routing_edges_keep_the_nchw_copy(gs, c, n, hw, view, what, dev):
    """Channels-last calls the NHWC tensor-core kernels do not take are copied to NCHW, as before, and still match the
    fp64 oracle; no *_nhwc family runs."""
    gen = torch.Generator(device=dev).manual_seed(gs + n)
    shape = (n, c) + hw
    x = _activation(gen, shape, 1, dev)
    xcl = view(x) if view is not None else x.contiguous(memory_format=CL)
    g = torch.randn(shape, device=dev, generator=gen)
    site = _Site(c, gs, 1, "shared", gen, dev)
    out = _run_arm(xcl, site, "train", g)
    assert not _nhwc_families(out["families"]), sorted(out["families"])
    assert not out["route"] & 0x100
    xd, gd = x.double().cpu().numpy(), g.double().cpu().numpy()
    y_o, mean_o, w_o, *_ = O.whiten_forward(xd, gs)
    dx_o = O.whiten_backward(xd, gd, mean_o, w_o)
    y, dx = out["y"].double().cpu().numpy(), out["dx"].double().cpu().numpy()
    assert rel_err(y, y_o) < 1e-3 and max_err(y, y_o) < 5e-3, (rel_err(y, y_o), max_err(y, y_o))
    assert rel_err(dx, dx_o) < 1e-3 and max_err(dx, dx_o) < 5e-3, (rel_err(dx, dx_o), max_err(dx, dx_o))


def test_fork_for_sum(dev):
    """Both gradients of a forked gs-64 channels-last output: added in Python (dout2 is a channels-last gs 1/2/4
    feature), then the NHWC kernels; same as the NCHW call."""
    _case(dev, c=128, gs=64, d=3, n=4, hw=(32, 32), layout="mixed", fork=True, seed=8)


def test_misaligned_gradient(dev):
    """An incoming gradient that is a misaligned channels-last view is copied, not refused."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(13)
    x = _activation(gen, (6, 64, 32, 32), 3, dev)
    g = torch.randn(x.shape, device=dev, generator=gen)
    ma, mb = dwt_b200.WTransform2d(64, 32).to(dev).train(), dwt_b200.WTransform2d(64, 32).to(dev).train()
    xa, xb = x.contiguous(memory_format=CL).requires_grad_(True), x.clone().requires_grad_(True)
    ya, yb = ma(xa), mb(xb)
    assert ya.grad_fn.cfg[3] & dwt_b200._native.LAYOUT_NHWC
    ya.backward(_misaligned_cl(g))
    yb.backward(g)
    assert _same(ya, yb) and _same(xa.grad, xb.grad) and _is_cl(xa.grad)


# --------------------------------------------------------------------------- the C ABI
def test_c_abi_return_codes(dev):
    """Accepted calls run on random inputs with their own output, statistics and gradient buffers (no status bit set);
    refused ones return before anything is launched."""
    from dwt_b200 import _native
    lib = _native.lib()
    c, gs, d = 64, 64, 1
    gen = torch.Generator(device=dev).manual_seed(31)
    numel = 128 * 36 * c                                     # the larger of the two geometries below (4 x 1024 x c)
    xs = {False: torch.randn(numel + 64, device=dev, generator=gen), True: torch.randn(numel + 64, device=dev, generator=gen).to(BF)}
    douts = {k: torch.randn_like(v) for k, v in xs.items()}    # dout
    ys = {k: torch.empty_like(v) for k, v in xs.items()}     # y
    dxs = {k: torch.empty_like(v) for k, v in xs.items()}    # dx
    save_mean, save_w = torch.empty(d, c, device=dev), torch.empty(d, c // gs, gs, gs, device=dev)
    gamma = torch.ones(c, device=dev)
    nhwc, bf = _native.LAYOUT_NHWC, _native.DTYPE_BF16
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)          # noqa: E731

    def fwd(n, hw, layout=nhwc, x_off=0, y_off=0, epi=0):
        b = bool(layout & bf)
        ws = _native.workspace(dev, n, c, hw, gs, d)
        g = _native.ptr(gamma) if epi else None
        return lib.dwt_whiten_fwd(p(xs[b], x_off), p(ys[b], y_off), n, c, hw, gs, d, layout, 1e-3, 0.1, 0, None, None, g, g,
                                  None, None, epi, _native.ptr(save_mean), _native.ptr(save_w), _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr(dev))

    def bwd(n, hw, layout=nhwc, dout_off=0, dout2=False, epi=0):
        b = bool(layout & bf)
        ws = _native.workspace(dev, n, c, hw, gs, d)
        g = _native.ptr(gamma) if epi else None
        return lib.dwt_whiten_bwd(p(xs[b]), p(douts[b], dout_off), p(douts[b]) if dout2 else None, p(dxs[b]), n, c, hw, gs, d,
                                  layout, 1e-3, _native.ptr(save_mean), _native.ptr(save_w), g, g, None, None, epi, None, None,
                                  _native.ptr(ws), ws.numel(), _native.stream_ptr(dev))
    _native.clear_status(dev)
    _native.profile_begin()
    assert fwd(4, 1024) == 0                                 # accepted: 4 x 32^2, gs 64
    assert bwd(4, 1024) == 0
    assert fwd(128, 36, layout=nhwc | bf) == 0               # HW = 36 in bf16: the channels-last rule is HW % 4
    assert bwd(128, 36, layout=nhwc | bf) == 0
    assert {f for f in _native.by_family(_native.profile_end()) if f.startswith("tc_")} == {
        "tc_stats_nhwc", "tc_apply_nhwc", "tc_bwd_reduce_nhwc", "tc_bwd_apply_nhwc",
        "tc_stats_nhwc_bf16", "tc_apply_nhwc_bf16", "tc_bwd_reduce_nhwc_bf16", "tc_bwd_apply_nhwc_bf16"}
    assert _native.status(dev) == 0
    assert torch.isfinite(dxs[True][:numel].float()).all() and torch.isfinite(save_w).all()
    assert fwd(4, 1024, x_off=4) == -1                       # misaligned x
    assert b"16-byte" in lib.dwt_last_error()
    assert fwd(4, 1024, y_off=4) == -1                       # misaligned y
    assert bwd(4, 1024, dout_off=4) == -1                    # misaligned dout
    assert bwd(4, 1024, dout2=True) == -4                    # a second gradient addend
    assert fwd(4, 1024, epi=_native.EPI_AFFINE) == -4        # an epilogue
    assert bwd(4, 1024, epi=_native.EPI_AFFINE) == -4
    assert fwd(84, 49) == -4                                 # HW % 4 != 0: the caller copies to NCHW
    assert fwd(63, 64) == -4                                 # N * HW < 4096
    torch.cuda.synchronize(dev)


# --------------------------------------------------------------------------- CUDA-graph capture
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_graph_capture(dtype, dev):
    """A channels-last gs-64 WTransform2d forward + backward captures into a CUDA graph (nothing on the path syncs,
    allocates through the driver or touches the context), and two replays reproduce the eager result bit for bit."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(3)
    shape = (8, 128, 24, 24)                                 # N * HW = 4608 >= 4096
    x = (torch.randn(shape, device=dev, generator=gen) + 2.0).to(dtype).contiguous(memory_format=CL)
    dy = torch.randn(shape, device=dev, generator=gen).to(dtype).contiguous(memory_format=CL)
    m = dwt_b200.WTransform2d(128, 64).to(dev).train()
    rm0, rv0 = m.running_mean.clone(), m.running_variance.clone()

    def step():
        # a fresh leaf per step: a gradient accumulator kept from an eager step is tied to the default stream, and
        # autograd's end-of-backward sync with that stream is illegal inside a capture (a PyTorch rule)
        xi = x.detach().requires_grad_(True)
        y = m(xi)
        assert y.grad_fn.cfg[3] & dwt_b200._native.LAYOUT_NHWC, "the channels-last kernels did not run"
        return y, torch.autograd.grad(y, xi, dy)[0]
    y_e, dx_e = (t.detach().clone() for t in step())         # eager, default stream: one EMA step from the initial buffers
    rm1, rv1 = m.running_mean.clone(), m.running_variance.clone()
    side = torch.cuda.Stream(dev)                            # the usual pre-capture warm-up on a side stream
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y_g, dx_g = step()
    for _ in range(2):
        m.running_mean.copy_(rm0)
        m.running_variance.copy_(rv0)
        g.replay()
        torch.cuda.synchronize(dev)
        assert _is_cl(y_g) and _is_cl(dx_g)
        assert _same(y_g, y_e) and _same(dx_g, dx_e)
        assert _same(m.running_mean, rm1) and _same(m.running_variance, rv1)


# --------------------------------------------------------------------------- the model at group_size=64
def _model_run(dev, layers, site_mode, cl, images, labels, sd):
    import torch.nn.functional as Fn
    import dwt_b200
    from harness.resnet50_dwt import build_resnet50_dwt
    model = build_resnet50_dwt({k: v.clone() for k, v in sd.items()}, layers, site_mode=site_mode, channels_last=cl,
                               group_size=64).to(dev).train()
    x = images.contiguous(memory_format=CL) if cl else images.contiguous()
    stem = {}                                        # the stem site's output: the max-pool's input
    model.maxpool.register_forward_hook(lambda m, i, o: stem.setdefault("out", i[0]))
    logits = model(x)
    s, t, a = torch.split(logits, logits.shape[0] // 3, dim=0)
    loss = Fn.nll_loss(Fn.log_softmax(s, dim=1), labels) + 0.1 * dwt_b200.MinEntropyConsensusLoss(65, dev)(t, a)
    loss.backward()
    grads = {k: p.grad.detach().double().cpu().numpy() for k, p in model.named_parameters() if p.grad is not None}
    bufs = {k: v.detach().double().cpu().numpy() for k, v in model.state_dict().items() if "running" in k}
    model.eval()
    with torch.no_grad():
        eval_logits = model(x)
    return logits.detach().double().cpu().numpy(), grads, bufs, eval_logits.double().cpu().numpy(), stem.get("out")


def test_resnet50_group_size_64_channels_last(dev):
    """The harness ResNet-50-DWT at group_size=64 (the stem site at gs 64, resnet50_dwt_mec_officehome.py:266),
    channels-last, fused sites, 3 x 2 images of 224^2: the train step runs end to end, the stem site's output is
    channels-last (the library max-pool takes it), eval runs; logits, gradients and buffers against the same topology on
    the NCHW port.  Gradient bound: max(1e-2, 1.5 x yardstick), the yardstick being the port channels-last against the
    port NCHW (cuDNN's own layout noise)."""
    import oracle.torch_port as port
    import dwt_b200
    from harness.synth import synth_batch, synth_state_dict
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        sd["bn1.wh.running_variance"] = synth_state_dict(seed=1, group_size=64, with_convs=False)["bn1.wh.running_variance"].to(dev)
        images, labels = synth_batch(seed=2, per_domain=2, size=224)
        images, labels = images.to(dev), labels.to(dev)
        lg, gr, bf, ev, stem = _model_run(dev, dwt_b200, "fused", True, images, labels, sd)
        assert stem is not None and _is_cl(stem), "the stem site's output is not channels-last"
        rl, rg, rb, rev, _ = _model_run(dev, port, "modules", False, images, labels, sd)
        _, yg, _, _, _ = _model_run(dev, port, "modules", True, images, labels, sd)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    assert rel_err(lg, rl) < 2e-4 and max_err(lg, rl) < 5e-4, (rel_err(lg, rl), max_err(lg, rl))
    assert rel_err(ev, rev) < 5e-4, rel_err(ev, rev)
    for k in rg:
        yard = rel_err(yg[k], rg[k])
        assert rel_err(gr[k], rg[k]) < max(1e-2, 1.5 * yard), (k, rel_err(gr[k], rg[k]), yard)
    for k in rb:
        assert rel_err(bf[k], rb[k]) < 1e-3, (k, rel_err(bf[k], rb[k]))
