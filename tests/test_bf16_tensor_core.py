"""bfloat16 activations on the NCHW tensor-core whitening kernels (group sizes 8..64), against the float32 kernels, bit for
bit.

A bf16 NCHW whitening call on a tensor-core geometry (group size 8, 16, 32, 64; HW >= 32 and a multiple of 8; at least
4096 samples per domain; 16-byte-aligned tensors) runs tc_stats / tc_apply / tc_bwd_reduce / tc_bwd_apply in bf16: the
float32 schedule of its shape with loads widened and stores rounded to nearest-even (include/dwt_b200.h, DWT_DTYPE_BF16).
So every comparison here is torch.equal, with NaN equal to NaN, against the float32 kernels on x.float():
y == y32.to(bf16), dx == dx32.to(bf16), save_mean / save_w, every running buffer and the status word.

  * group sizes 8/16/32/64, C = 96 (a partial super-block), HW = 32, 40 (a partial 32-pixel box) and 3136,
    N * HW = 4096 exactly, 1 to 4 domains on shared / distinct / mixed running buffers;
  * train, no-grad train, eval forward + backward, default buffers;
  * BASELINE config 2 (N=256 C=256 56^2 gs 64), the two pilot-shift inputs at that size, a NaN input;
  * routing: only the *_bf16 tensor-core families run, no float32 copy of x is made; the geometries and alignments the
    bf16 kernels lack run the float32 kernels on upcast copies (and still match);
  * fork_for_sum, a misaligned bf16 gradient, a conv -> WTransform2d(gs 64) -> conv model under autocast;
  * return codes of the C ABI.
"""
import ctypes
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
GIB = 1 << 30
BF16_TC_FAMILIES = {"tc_stats_bf16", "dense_fwd_finalize_bf16", "tc_apply_bf16", "eval_prep_bf16", "tc_bwd_reduce_bf16",
                    "dense_bwd_finalize_bf16", "tc_bwd_apply_bf16", "bwd_prep_bf16"}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    d = torch.device("cuda", 0)
    torch.cuda.reset_peak_memory_stats(d)
    t0 = time.perf_counter()
    yield d
    print(f"\ntest_bf16_tensor_core: {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated(d) / GIB:.2f} GiB")


def _same(a, b):
    """torch.equal, with NaN equal to NaN (bf16 NaN payloads are not compared)."""
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.isnan(), b.isnan()) and \
        torch.equal(a.nan_to_num(0.0), b.nan_to_num(0.0))


def _activation(gen, shape, d, dev):
    """NCHW float32 activations: correlated neighbouring channels, per-channel scales, a mean per domain."""
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


def _run_arm(dt, x0, site, mode, g1, g2=None, measure=False):
    """One arm: the site on x0 (bf16: as given, views included; float32: x0.float()).  Returns everything to compare."""
    import dwt_b200
    from dwt_b200 import _native as nv, functional as F
    dev = x0.device
    bufs = site.buffers()
    running = [bufs[o] for o in site.owner]
    grad = mode in ("train", "eval")
    x = (x0.detach() if dt == BF else x0.float()).requires_grad_(grad)
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
            torch.autograd.backward([u, v], [g1, g2])
        else:
            y.backward(g1 if dt == BF else g1.float())
        out["dx"] = x.grad
    out["families"] = set(nv.by_family(nv.profile_end()))
    if measure:
        torch.cuda.synchronize(dev)
        out["peak"] = torch.cuda.max_memory_allocated(dev) - base
    out["running"] = [t for o in sorted(bufs) for t in bufs[o]]
    return out


def _compare(bf, ref):
    assert bf["y"].dtype == BF and bf["y"].is_contiguous()
    assert _same(bf["y"], ref["y"].to(BF)), "y"
    assert bf["status"] == ref["status"], (bf["status"], ref["status"])
    for k, (p, q) in enumerate(zip(bf["running"], ref["running"])):
        assert _same(p, q), f"running buffer {k}"
    if ref["stats"] is not None:
        for k, (p, q) in enumerate(zip(bf["stats"], ref["stats"])):
            assert _same(p, q), f"save_mean / save_w {k}"
        assert bf["dx"].dtype == BF and _same(bf["dx"], ref["dx"].to(BF)), "dx"


def _case(dev, *, c, gs, d, n, hw, mode="train", layout="shared", seed=0, make_x=_activation, nan=False, bf16_route=True,
          x_view=None, fork=False, measure=False):
    """The site in bf16 and in float32 on the upcast input; asserts every comparison and which kernels ran."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    h, w = hw
    shape = (d * n, c, h, w)
    x = make_x(gen, shape, d, dev).to(BF)
    if nan:
        x[0, 1, 0, 0] = float("nan")
    if x_view is not None:
        x = x_view(x)
    site = _Site(c, gs, d, layout, gen, dev)
    g1 = torch.randn(shape, device=dev, generator=gen).to(BF)
    g2 = torch.randn(shape, device=dev, generator=gen).to(BF) if fork else None
    bf = _run_arm(BF, x, site, mode, g1, g2, measure=measure)
    # the float32 reference takes RN_bf16(g1 + g2) -- autograd's own bf16 sum -- as its one gradient
    ref = _run_arm(torch.float32, x, site, mode, (g1 + g2) if fork else g1)
    _compare(bf, ref)
    assert not any(f.endswith("_bf16") for f in ref["families"]), ref["families"]
    if bf16_route:
        assert bf["families"] <= BF16_TC_FAMILIES and "tc_apply_bf16" in bf["families"], sorted(bf["families"])
    else:
        assert bf["families"] == ref["families"], (sorted(bf["families"]), sorted(ref["families"]))
    return bf, ref


# --------------------------------------------------------------------------- group sizes, shapes, domains, buffers
CASES = [   # gs, C, domains, N per domain, (H, W), running buffers
    (8, 64, 1, 4, (32, 32), "shared"),        # N * HW = 4096 exactly
    (16, 128, 2, 2, (48, 48), "distinct"),
    (32, 96, 3, 104, (5, 8), "mixed"),        # C = 96: a partial super-block; HW = 40: a partial 32-pixel box
    (64, 64, 4, 128, (1, 32), "mixed"),       # HW = 32: one box per row; N * HW = 4096
    (64, 256, 3, 2, (56, 56), "distinct"),    # HW = 3136
    (32, 128, 4, 3, (56, 56), "shared"),
]


@pytest.mark.parametrize("gs,c,d,n,hw,layout", CASES,
                         ids=[f"gs{k[0]}-c{k[1]}-d{k[2]}-n{k[3]}-{k[4][0]}x{k[4][1]}-{k[5]}" for k in CASES])
def test_geometries(gs, c, d, n, hw, layout, dev):
    _case(dev, c=c, gs=gs, d=d, n=n, hw=hw, layout=layout, seed=gs + c + d)


MODES = [   # gs, C, domains, N, (H, W), mode, buffers
    (16, 64, 3, 8, (24, 24), "nograd", "mixed"),
    (32, 64, 2, 8, (32, 32), "eval", "distinct"),
    (64, 128, 1, 4, (32, 40), "eval", "shared"),
    (8, 96, 3, 8, (32, 24), "nograd", "distinct"),
]


@pytest.mark.parametrize("gs,c,d,n,hw,mode,layout", MODES,
                         ids=[f"gs{k[0]}-c{k[1]}-d{k[2]}-{k[5]}-{k[6]}" for k in MODES])
def test_modes(gs, c, d, n, hw, mode, layout, dev):
    _case(dev, c=c, gs=gs, d=d, n=n, hw=hw, mode=mode, layout=layout, seed=3 * gs + d)


def test_default_buffers(dev):
    """WTransform2d with its own default buffers (zero mean, all-ones second moment), training, forward + backward."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(21)
    x = (torch.randn(4, 64, 32, 32, device=dev, generator=gen) * 2 + 1).to(BF)
    g = torch.randn(x.shape, device=dev, generator=gen).to(BF)
    ma, mb = dwt_b200.WTransform2d(64, 8).to(dev).train(), dwt_b200.WTransform2d(64, 8).to(dev).train()
    xa, xb = x.clone().requires_grad_(True), x.float().requires_grad_(True)
    ya, yb = ma(xa), mb(xb)
    assert ya.grad_fn.cfg[3] & dwt_b200._native.DTYPE_BF16, "the bf16 kernels did not run"
    assert _same(ya, yb.to(BF))
    ya.backward(g)
    yb.backward(g.float())
    assert _same(xa.grad, xb.grad.to(BF))
    assert _same(ma.running_mean, mb.running_mean) and _same(ma.running_variance, mb.running_variance)


# --------------------------------------------------------------------------- the microbench size, pilot inputs, NaN
def test_config2_bf16_kernels_without_a_float32_copy(dev):
    """BASELINE config 2 (N=256 C=256 56^2 gs 64), forward + backward.  The device memory the bf16 call adds stays under
    three bf16 copies of x: y and dx are two; a float32 copy of x alone would be two more (the upcast path makes five)."""
    bf, _ = _case(dev, c=256, gs=64, d=1, n=256, hw=(56, 56), make_x=_microbench, seed=0, measure=True)
    xbytes = 256 * 256 * 56 * 56 * 2
    assert bf["peak"] < 3 * xbytes, (bf["peak"], xbytes)


@pytest.mark.parametrize("make_x", [_pilot_30sigma, _mean_50sigma], ids=["pilot_30sigma", "mean_50sigma"])
def test_pilot_shift_inputs(make_x, dev):
    _case(dev, c=256, gs=64, d=1, n=256, hw=(56, 56), make_x=make_x, seed=1)


def test_nan_input_sets_the_same_status(dev):
    from dwt_b200 import _native
    bf, _ = _case(dev, c=64, gs=16, d=3, n=8, hw=(32, 32), layout="distinct", seed=5, nan=True)
    assert bf["status"] & _native.STATUS_NOT_PD
    _native.clear_status(dev)


# --------------------------------------------------------------------------- routing edges: the float32 kernels
def _off_by_2_bytes(x):
    """x's values in a contiguous bf16 view whose data_ptr() is 2 bytes past a 16-byte boundary."""
    buf = torch.empty(x.numel() + 8, dtype=BF, device=x.device)
    v = buf[1:1 + x.numel()].view(x.shape)
    v.copy_(x)
    assert v.is_contiguous() and v.data_ptr() % 16 == 2
    return v


FALLBACKS = [   # gs, C, domains, N, (H, W), view, what
    (64, 64, 1, 128, (6, 6), None, "hw36"),          # HW % 4 == 0 but HW % 8 != 0
    (16, 64, 1, 63, (8, 8), None, "nhw4032"),        # N * HW = 4032 < 4096
    (12, 48, 2, 8, (32, 32), None, "gs12"),          # 64 % 12 != 0: the tiled kernels
    (64, 64, 1, 4, (32, 32), _off_by_2_bytes, "misaligned"),
]


@pytest.mark.parametrize("gs,c,d,n,hw,view,what", FALLBACKS, ids=[k[6] for k in FALLBACKS])
def test_fallback_geometries(gs, c, d, n, hw, view, what, dev):
    """Calls the bf16 tensor-core kernels do not take run the float32 kernels on an upcast copy, and match."""
    bf, _ = _case(dev, c=c, gs=gs, d=d, n=n, hw=hw, x_view=view, bf16_route=False, seed=gs + n)
    assert not bf["route"] & 0x200


# --------------------------------------------------------------------------- other paths
def test_fork_for_sum(dev):
    """Both gradients of a forked NCHW bf16 site: summed once by autograd's bf16 add, then the bf16 kernels."""
    _case(dev, c=128, gs=32, d=3, n=4, hw=(32, 32), layout="mixed", fork=True, seed=8)


def test_misaligned_gradient(dev):
    """An incoming bf16 gradient that is a misaligned view is copied, not refused: the forward ran the bf16 kernels."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(13)
    x = _activation(gen, (6, 64, 32, 32), 3, dev).to(BF)
    g = _off_by_2_bytes(torch.randn(x.shape, device=dev, generator=gen).to(BF))
    ma, mb = dwt_b200.WTransform2d(64, 32).to(dev).train(), dwt_b200.WTransform2d(64, 32).to(dev).train()
    xa, xb = x.clone().requires_grad_(True), x.float().requires_grad_(True)
    ya, yb = ma(xa), mb(xb)
    assert ya.grad_fn.cfg[3] & dwt_b200._native.DTYPE_BF16
    ya.backward(g)
    yb.backward(g.float())
    assert _same(ya, yb.to(BF)) and _same(xa.grad, xb.grad.to(BF))


def test_conv_whitening_conv_model_under_autocast(dev, monkeypatch):
    """conv -> WTransform2d(64, 64) -> ReLU -> conv under autocast: the bf16 kernels give the very step of the upcast path
    (x.float() -> float32 kernels -> bf16) -- outputs, loss, every gradient and running buffer."""
    import dwt_b200
    from dwt_b200 import _native, functional as F
    gen = torch.Generator(device=dev).manual_seed(17)
    images = torch.randn(4, 3, 32, 32, device=dev, generator=gen)
    torch.manual_seed(17)
    proto = torch.nn.Sequential(torch.nn.Conv2d(3, 64, 3, padding=1), dwt_b200.WTransform2d(64, 64), torch.nn.ReLU(),
                                torch.nn.Conv2d(64, 8, 3, padding=1)).to(dev)
    cudnn = torch.backends.cudnn
    monkeypatch.setattr(cudnn, "deterministic", True)
    monkeypatch.setattr(cudnn, "benchmark", False)

    def step(upcast):
        model = __import__("copy").deepcopy(proto).train()
        with monkeypatch.context() as mp:
            if upcast:
                mp.setattr(F, "_bf16_tensor_core", lambda *a, **k: False)
            _native.profile_begin()
            with torch.autocast("cuda", dtype=BF):
                out = model(images)
                loss = out.float().square().mean()
            loss.backward()
            fams = set(_native.by_family(_native.profile_end()))
        return out.detach(), loss.detach(), [p.grad for p in model.parameters()], list(model.buffers()), fams
    a, b = step(False), step(True)
    assert a[0].dtype == BF and _same(a[0], b[0]) and _same(a[1], b[1])
    assert all(_same(p, q) for p, q in zip(a[2], b[2])), "gradients"
    assert all(_same(p, q) for p, q in zip(a[3], b[3])), "running buffers"
    assert a[4] <= BF16_TC_FAMILIES and "tc_bwd_apply_bf16" in a[4], sorted(a[4])
    assert not any(f.endswith("_bf16") for f in b[4]), sorted(b[4])


# --------------------------------------------------------------------------- the C ABI
def test_c_abi_return_codes(dev):
    from dwt_b200 import _native
    lib = _native.lib()
    c, gs, d = 64, 64, 1
    buf = torch.zeros(2 * 128 * c * 1024 + 64, dtype=BF, device=dev)
    ok, off = buf.data_ptr(), buf.data_ptr() + 2            # 256-byte aligned / 2 bytes off
    out = torch.zeros_like(buf)
    st = torch.zeros(d * c * gs, device=dev)
    rm = _native.ptr_array([st] * d)
    bf = _native.DTYPE_BF16

    def fwd(x, n, hw):
        ws = _native.workspace(dev, n, c, hw, gs, d)
        return lib.dwt_whiten_fwd(ctypes.c_void_p(x), _native.ptr(out), n, c, hw, gs, d, bf, 1e-3, 0.1, 0, rm, rm, None,
                                  None, None, None, 0, _native.ptr(st), _native.ptr(st), _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr(dev))

    def bwd(x, dout, n, hw):
        ws = _native.workspace(dev, n, c, hw, gs, d)
        return lib.dwt_whiten_bwd(ctypes.c_void_p(x), ctypes.c_void_p(dout), None, _native.ptr(out), n, c, hw, gs, d, bf, 1e-3,
                                  _native.ptr(st), _native.ptr(st), None, None, None, None, 0, None, None, _native.ptr(ws),
                                  ws.numel(), _native.stream_ptr(dev))
    assert fwd(ok, 4, 1024) == 0                            # accepted: 4 x 32^2, gs 64
    assert bwd(ok, ok, 4, 1024) == 0
    assert fwd(ok, 128, 36) == -4                           # HW = 36: HW % 8 != 0
    assert b"multiple of 8" in lib.dwt_last_error()
    assert bwd(ok, ok, 128, 36) == -4
    assert fwd(off, 4, 1024) == -1                          # misaligned base
    assert b"16-byte" in lib.dwt_last_error()
    assert bwd(ok, off, 4, 1024) == -1
    torch.cuda.synchronize(dev)
    _native.clear_status(dev)
