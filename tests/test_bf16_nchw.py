"""bfloat16 activations on the NCHW register-resident kernels (whitening at group sizes 1, 2, 4 and domain batch norm),
against the float32 kernels, bit for bit.

A bf16 NCHW call with HW % 4 == 0 and 8-byte-aligned tensors runs small_stats / small_apply / small_bwd_reduce /
small_bwd_apply in bf16: the float32 plan of its shape (vec = 4) with loads widened and stores rounded to nearest-even
(include/dwt_b200.h, DWT_DTYPE_BF16).  So every comparison here is torch.equal, with NaN equal to NaN, against the float32
kernels on the upcast inputs (where the output is forked, RN_bf16(dout + dout2).float() as the single gradient):
y == y32.to(bf16), dx == dx32.to(bf16), the residual's gradient, dgamma / dbeta, save_mean / save_w, every running buffer,
num_batches_tracked and the status word.

  * every NCHW site geometry of the harness ResNet-50-DWT at 224^2 with HW % 4 == 0 (2 images per domain), the LeNet
    sites, the stem at the benchmark's 3 x 64 images;
  * epilogues none / AFFINE / AFFINE|RELU / RESIDUAL; 1 to 4 domains on shared / distinct / mixed buffers; train,
    no-grad train, eval and replicated; fork_for_sum against autograd's bf16 add;
  * launch edges of norm_small.cu: 2, 4 and 8 problems per CTA, nchunks 1 and 2, the chunk cap, fewer items than a team
    has threads, HW = 4;
  * the pilot-shift inputs, a NaN input and a non-positive-definite running covariance;
  * routing (only small_*_bf16 families, no float32 copy of x) and the upcast fallbacks; the C ABI; CUDA-graph replay;
  * whole models under autocast against the same step with the new routing patched off.
"""
import copy
import ctypes
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
GIB = 1 << 30
SMALL_BF16 = {"small_stats_bf16", "small_apply_bf16", "small_bwd_reduce_bf16", "small_bwd_apply_bf16", "eval_prep_bf16",
              "bwd_prep_bf16"}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    d = torch.device("cuda", 0)
    torch.cuda.reset_peak_memory_stats(d)
    t0 = time.perf_counter()
    yield d
    print(f"\ntest_bf16_nchw: {time.perf_counter() - t0:.1f} s, peak device memory "
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


def _pilot_30sigma(gen, shape, d, dev):
    """Image 0 of every domain 30 sigma off in the pilot window (the <= 32 mid-image pixels K is estimated from)."""
    x = _activation(gen, shape, d, dev)
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
    x = _activation(gen, shape, d, dev).mul_(0.1).add_(10.0)
    return x.add_(torch.linspace(0.0, 40.0, shape[1], device=dev).view(1, -1, 1, 1))


def _off_by_2_bytes(x):
    """x's values in a contiguous bf16 view whose data_ptr() is 2 bytes past a 16-byte boundary."""
    buf = torch.empty(x.numel() + 8, dtype=BF, device=x.device)
    v = buf[1:1 + x.numel()].view(x.shape)
    v.copy_(x)
    assert v.is_contiguous() and v.data_ptr() % 16 == 2
    return v


class _Site:
    """A norm site's state -- the D domain modules on running buffers aliased 'shared', 'distinct' or 'mixed', gamma,
    beta -- built again from the same values for every arm."""

    def __init__(self, kind, c, gs, d, layout, gen, dev):
        self.kind, self.c, self.gs, self.d = kind, c, gs, d
        self.owner = {"shared": [0] * d, "distinct": list(range(d)), "mixed": [0] + [1] * (d - 1)}[layout]
        self.init = {}
        for o in sorted(set(self.owner)):
            rm = 0.1 * torch.randn(c, device=dev, generator=gen)
            if kind == "whiten":
                a = torch.randn(c // gs, gs, gs, device=dev, generator=gen)
                self.init[o] = (rm.view(1, c, 1, 1), a @ a.transpose(1, 2) / gs + 0.5 * torch.eye(gs, device=dev))
            else:
                self.init[o] = (rm, 0.5 + torch.rand(c, device=dev, generator=gen))
        self.g0 = 0.5 + torch.rand(c, 1, 1, device=dev, generator=gen)
        self.b0 = 0.3 * torch.randn(c, 1, 1, device=dev, generator=gen)

    def arm(self):
        import dwt_b200
        bufs = {o: (rm.clone(), rv.clone()) for o, (rm, rv) in self.init.items()}
        if self.kind == "whiten":
            mods = [dwt_b200.WTransform2d(self.c, self.gs, running_m=bufs[o][0], running_var=bufs[o][1]).train()
                    for o in self.owner]
        else:
            mods = [dwt_b200.BatchNorm2d(self.c, *bufs[o], affine=False, momentum=None).train() for o in self.owner]
            for m in mods:
                m.num_batches_tracked.fill_(2)
        a = type("Arm", (), {})()
        a.bufs, a.mods = bufs, mods
        a.gamma, a.beta = self.g0.clone().requires_grad_(True), self.b0.clone().requires_grad_(True)
        a.norm = dwt_b200.DomainTripleNorm(self.kind, self.c, self.gs, n_domains=self.d)
        return a

    @staticmethod
    def running(a):
        out = [t for o in sorted(a.bufs) for t in a.bufs[o]]
        return out + [m.num_batches_tracked for m in a.mods if hasattr(m, "num_batches_tracked")]


def _norm_node(y):
    """The _NormFunction node behind y (the upcast path puts a dtype cast in front of it)."""
    node = y.grad_fn
    while not type(node).__name__.startswith("_NormFunction"):
        node = node.next_functions[0][0]
    return node


def _run_arm(site, x, r, g1, g2, *, epi, mode, fork, measure=False):
    """One arm: the site on x (and r) as given.  g1 (and g2, forked) in x's dtype.  Returns everything to compare."""
    import dwt_b200
    from dwt_b200 import _native as nv, functional as F
    dev = x.device
    a = site.arm()
    grad = mode in ("train", "eval")
    x = x.detach().requires_grad_(grad)
    r = r.detach().requires_grad_(grad) if r is not None else None
    gamma, beta = (None, None) if epi == "none" else (a.gamma, a.beta)
    relu = epi in ("relu", "residual")
    nv.clear_status(dev)
    if measure:
        torch.cuda.synchronize(dev)
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
    nv.profile_begin()
    with torch.set_grad_enabled(grad):
        if mode == "eval":
            second = "running_variance" if site.kind == "whiten" else "running_var"
            y = F.norm(x, gamma, beta, kind=site.kind, group_size=site.gs, n_domains=site.d, training_stats=False,
                       eps=1e-5, momentum=0.1, update_running=False,
                       running=[(m.running_mean, getattr(m, second)) for m in a.mods], relu=relu, residual=r)
        else:
            y = a.norm(x, a.mods, gamma, beta, relu, residual=r, replicated=mode == "replicated")
    out = {"y": y.detach(), "status": nv.status(dev), "dx": None}
    if grad:
        node = _norm_node(y)
        out["stats"], out["route"] = list(node.saved_tensors[1:3]), node.cfg[3]
        del node
        if fork == "kernels":                        # the two gradients reach the kernels apart
            u, v = dwt_b200.fork_for_sum(y)
            torch.autograd.backward([u, v], [g1, g2])
        elif fork == "autograd":                     # y used twice: autograd adds the two gradients (in bf16)
            ((y * g1).sum() + (y * g2).sum()).backward()
        else:
            y.backward(g1)
        out["dx"] = x.grad
        out["d_res"] = r.grad if r is not None else None
        out["dgb"] = [t.grad for t in (gamma, beta) if t is not None]
    prof = nv.by_family(nv.profile_end())
    out["families"] = set(prof)
    out["launches"] = {k: v["launches"] for k, v in prof.items()}
    if measure:
        torch.cuda.synchronize(dev)
        out["peak"] = torch.cuda.max_memory_allocated(dev) - base
    out["running"] = _Site.running(a)
    return out


def _compare(bf, ref):
    assert bf["y"].dtype == BF and bf["y"].is_contiguous()
    assert _same(bf["y"], ref["y"].to(BF)), "y"
    assert bf["status"] == ref["status"], (bf["status"], ref["status"])
    for k, (p, q) in enumerate(zip(bf["running"], ref["running"])):
        assert _same(p, q), f"running buffer {k}"
    if ref["dx"] is None:
        return
    for k, (p, q) in enumerate(zip(bf["stats"], ref["stats"])):
        assert _same(p, q), f"save_mean / save_w {k}"
    assert bf["dx"].dtype == BF and _same(bf["dx"], ref["dx"].to(BF)), "dx"
    # the residual's gradient comes back in the residual's dtype (float32 for a mixed-dtype call)
    assert _same(bf["d_res"], None if ref["d_res"] is None else ref["d_res"].to(bf["d_res"].dtype)), "residual gradient"
    assert len(bf["dgb"]) == len(ref["dgb"])
    for k, (p, q) in enumerate(zip(bf["dgb"], ref["dgb"])):
        assert _same(p, q), f"dgamma / dbeta {k}"


def _case(dev, *, kind, c, gs, d, n, h, w, epi="relu", mode="train", fork=False, layout="shared", seed=0,
          make_x=_activation, nan=False, x_view=None, r_float=False, bf16_route=True, measure=False):
    """One site in bf16 and in float32 on the upcast inputs; asserts every comparison and which kernels ran."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    shape = (d * n, c, h, w)
    x = make_x(gen, shape, d, dev).to(BF)
    if nan:
        x[0, 1, 0, 0] = float("nan")
    r = _activation(gen, shape, d, dev).to(BF) if epi == "residual" else None
    g1 = torch.randn(shape, device=dev, generator=gen).to(BF)
    g2 = torch.randn(shape, device=dev, generator=gen).to(BF) if fork else None
    site = _Site(kind, c, gs, d, layout, gen, dev)
    xb = x_view(x) if x_view is not None else x
    rb = None if r is None else (r.float() if r_float else r)
    bf = _run_arm(site, xb, rb, g1, g2, epi=epi, mode=mode, fork="kernels" if fork else None, measure=measure)
    ref = _run_arm(site, x.float(), None if r is None else r.float(), ((g1 + g2) if fork else g1).float(), None, epi=epi,
                   mode=mode, fork=None)
    _compare(bf, ref)
    assert not any(f.endswith("_bf16") for f in ref["families"]), sorted(ref["families"])
    if bf16_route:
        assert bf["families"] <= SMALL_BF16 and "small_apply_bf16" in bf["families"], sorted(bf["families"])
    else:
        assert bf["families"] == ref["families"], (sorted(bf["families"]), sorted(ref["families"]))
    return bf, ref


# --------------------------------------------------------------------------- every NCHW site of the models
@pytest.fixture(scope="module")
def model_sites(dev):
    """(kind, C, H, W, gs, epilogue, forked) of every DomainTripleNorm call of an NCHW fused training forward of the
    harness ResNet-50-DWT at 224^2 (2 images per domain), recorded at functional.norm, duplicates removed."""
    import dwt_b200
    from dwt_b200 import functional as F
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    calls, forked = [], []
    norm, fork = F.norm, dwt_b200.fork_for_sum

    def rec_norm(x, gamma, beta, **kw):
        y = norm(x, gamma, beta, **kw)
        epi = "none" if gamma is None else ("residual" if kw.get("residual") is not None else
                                             ("relu" if kw.get("relu") else "affine"))
        calls.append(((kw["kind"], x.shape[1], x.shape[2], x.shape[3], kw["group_size"], epi), y))
        return y

    def rec_fork(y):
        forked.append(y)
        return fork(y)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(F, "norm", rec_norm)
        mp.setattr(dwt_b200, "fork_for_sum", rec_fork)
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        model = build_resnet50_dwt(sd, dwt_b200, site_mode="fused").to(dev).train()
        images, _ = synth_batch(seed=2, per_domain=2, size=224)
        model(images.to(dev))
    sites = []
    for key, y in calls:
        entry = key + (any(f is y for f in forked),)
        if entry not in sites:
            sites.append(entry)
    del model, calls, forked
    return sites


def test_every_model_site_geometry(model_sites, dev):
    """Each distinct NCHW site of the training step with HW % 4 == 0, at 2 images per domain, as the model runs it."""
    todo = [s for s in model_sites if (s[2] * s[3]) % 4 == 0]
    assert ("whiten", 64, 112, 112, 4, "relu", False) in todo, model_sites
    assert {s[5] for s in todo} == {"affine", "relu", "residual"}, todo
    assert len(todo) >= 12 and len(model_sites) - len(todo) >= 3, model_sites      # layer4's 7x7 sites stay upcast
    failures = []
    for i, (kind, c, h, w, gs, epi, fork) in enumerate(todo):
        try:
            _case(dev, kind=kind, c=c, gs=gs, d=3, n=2, h=h, w=w, epi=epi, fork=fork, seed=200 + i)
        except AssertionError as e:
            failures.append(f"{kind} {c}@{h}x{w} gs{gs} {epi}{' forked' if fork else ''}: {e}")
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("c,h", [(32, 28), (48, 14)], ids=["conv1-32x28", "conv2-48x14"])
def test_lenet_sites(c, h, dev):
    """The LeNet's two whitening sites (usps_mnist.py --group_size 4), one WTransform2d per domain as the LeNet calls them."""
    _case(dev, kind="whiten", c=c, gs=4, d=1, n=64, h=h, w=h, epi="none", seed=c)


def test_stem_at_bench_size_without_a_float32_copy(dev):
    """The stem site at the benchmark's 3 x 64 images (problems split over CTAs, the arrival counter runs).  The device
    memory the bf16 call adds stays under three bf16 copies of x: y and dx are two; a float32 copy of x alone would be
    two more."""
    bf, _ = _case(dev, kind="whiten", c=64, gs=4, d=3, n=64, h=112, w=112, seed=7, measure=True)
    xbytes = 3 * 64 * 64 * 112 * 112 * 2
    assert bf["peak"] < 3 * xbytes, (bf["peak"], xbytes)


# --------------------------------------------------------------------------- epilogues, modes, domains, buffers
MODES = [   # kind, C, gs, domains, epilogue, mode, forked, running buffers
    ("whiten", 64, 4, 3, "relu", "nograd", False, "shared"),
    ("whiten", 64, 2, 3, "residual", "eval", False, "distinct"),
    ("bn", 256, 1, 3, "relu", "eval", False, "mixed"),
    ("whiten", 64, 2, 2, "none", "eval", False, "shared"),        # no reduction in backward: bwd_prep
    ("whiten", 64, 4, 3, "relu", "replicated", False, "shared"),
    ("bn", 256, 1, 3, "residual", "replicated", False, "distinct"),
    ("whiten", 128, 1, 4, "affine", "train", False, "mixed"),
    ("whiten", 128, 2, 3, "residual", "train", True, "distinct"),
    ("bn", 512, 1, 1, "none", "train", True, "shared"),
    ("whiten", 64, 4, 4, "relu", "train", False, "mixed"),
    ("bn", 128, 1, 2, "affine", "train", False, "distinct"),
]


@pytest.mark.parametrize("kind,c,gs,d,epi,mode,fork,layout", MODES,
                         ids=[f"{m[0]}-c{m[1]}-gs{m[2]}-d{m[3]}-{m[4]}-{m[5]}{'-forked' if m[6] else ''}-{m[7]}" for m in MODES])
def test_modes_and_buffers(kind, c, gs, d, epi, mode, fork, layout, dev):
    _case(dev, kind=kind, c=c, gs=gs, d=d, n=2, h=8, w=8, epi=epi, mode=mode, fork=fork, layout=layout, seed=c + gs + d)


# --------------------------------------------------------------------------- launch edges of norm_small.cu
EDGES = [   # kind, C, gs, domains, (N, H, W) per domain, what
    ("bn", 256, 1, 3, (2, 4, 4), "ppc2"),           # 768 problems over 528 stats CTAs: 2 problems per CTA
    ("bn", 512, 1, 3, (2, 4, 4), "ppc4"),
    ("bn", 1024, 1, 3, (2, 4, 4), "ppc8"),
    ("whiten", 2048, 4, 3, (1, 4, 4), "gs4-ppc4"),
    ("bn", 64, 1, 3, (4, 32, 32), "nchunks2"),       # 192 problems: each split over 2 CTAs
    ("whiten", 16, 4, 1, (64, 32, 32), "nchunks-many"),
    ("bn", 1, 1, 1, (4, 1040, 1040), "chunk-cap"),   # one problem: the apply kernel splits it over the chunk cap
    ("whiten", 8, 2, 2, (1, 4, 4), "few-items"),     # 4 items per problem, a team of 256 threads
    ("whiten", 16, 4, 3, (3, 2, 2), "hw4"),
]


@pytest.mark.parametrize("kind,c,gs,d,nhw,what", EDGES, ids=[e[5] for e in EDGES])
def test_launch_edges(kind, c, gs, d, nhw, what, dev):
    n, h, w = nhw
    _case(dev, kind=kind, c=c, gs=gs, d=d, n=n, h=h, w=w, epi="relu", fork=True, layout="mixed", seed=c + d)


# --------------------------------------------------------------------------- pilot shift, NaN, non-PD
@pytest.mark.parametrize("make_x", [_pilot_30sigma, _mean_50sigma], ids=["pilot_30sigma", "mean_50sigma"])
@pytest.mark.parametrize("kind,gs", [("whiten", 4), ("bn", 1)])
def test_pilot_shift_inputs(make_x, kind, gs, dev):
    _case(dev, kind=kind, c=64, gs=gs, d=1, n=64, h=28, w=28, make_x=make_x, seed=1)


def test_nan_input_sets_the_same_status_and_skips_the_same_ema(dev):
    from dwt_b200 import _native
    bf, _ = _case(dev, kind="whiten", c=64, gs=4, d=3, n=2, h=8, w=8, layout="distinct", seed=5, nan=True)
    assert bf["status"] & _native.STATUS_NOT_PD
    _native.clear_status(dev)


def test_non_positive_definite_running_covariance(dev):
    """Eval on a running covariance that is not positive definite in group 0: the same status bit and NaN pattern."""
    from dwt_b200 import _native
    gen = torch.Generator(device=dev).manual_seed(6)
    site = _Site("whiten", 32, 4, 2, "shared", gen, dev)
    site.init[0][1][0] = -torch.eye(4, device=dev)
    x = _activation(gen, (4, 32, 8, 8), 2, dev).to(BF)
    g = torch.randn(x.shape, device=dev, generator=gen).to(BF)
    bf = _run_arm(site, x, None, g, None, epi="affine", mode="eval", fork=None)
    ref = _run_arm(site, x.float(), None, g.float(), None, epi="affine", mode="eval", fork=None)
    _compare(bf, ref)
    assert bf["status"] & _native.STATUS_NOT_PD and bf["y"][:, :4].isnan().all()
    assert bf["families"] <= SMALL_BF16
    _native.clear_status(dev)


# --------------------------------------------------------------------------- fork_for_sum
@pytest.mark.parametrize("epi", ["relu", "residual"])
def test_fork_for_sum_equals_autograds_add(epi, dev):
    """The two gradients of a forked bf16 NCHW output, added by the backward before the call == autograd's bf16 add."""
    gen = torch.Generator(device=dev).manual_seed(3)
    shape = (6, 128, 14, 14)
    x = _activation(gen, shape, 3, dev).to(BF)
    r = _activation(gen, shape, 3, dev).to(BF) if epi == "residual" else None
    g1, g2 = (torch.randn(shape, device=dev, generator=gen).to(BF) for _ in range(2))
    site = _Site("bn", 128, 1, 3, "shared", gen, dev)
    a = _run_arm(site, x, r, g1, g2, epi=epi, mode="train", fork="kernels")
    b = _run_arm(site, x, r, g1, g2, epi=epi, mode="train", fork="autograd")
    assert a["route"] & 0x200 and a["families"] <= SMALL_BF16
    for key in ("dx", "d_res"):
        assert _same(a[key], b[key]), key
    for p, q in zip(a["dgb"] + a["running"], b["dgb"] + b["running"]):
        assert _same(p, q)


# --------------------------------------------------------------------------- routing edges: the float32 kernels
FALLBACKS = [   # kind, C, gs, (H, W), x view, float32 residual, what
    ("whiten", 64, 4, (7, 7), None, False, "hw49"),
    ("bn", 64, 1, (8, 8), _off_by_2_bytes, False, "misaligned"),
    ("whiten", 64, 2, (8, 8), None, True, "float32-residual"),
]


@pytest.mark.parametrize("kind,c,gs,hw,view,r_float,what", FALLBACKS, ids=[k[6] for k in FALLBACKS])
def test_fallbacks_upcast_and_match(kind, c, gs, hw, view, r_float, what, dev):
    """Calls the bf16 kernels do not take run the float32 kernels on upcast copies, and match."""
    bf, _ = _case(dev, kind=kind, c=c, gs=gs, d=3, n=2, h=hw[0], w=hw[1], epi="residual" if r_float else "relu",
                  x_view=view, r_float=r_float, bf16_route=False, seed=c + gs)
    assert not bf["route"] & 0x200


def test_misaligned_gradient_is_copied(dev):
    """An incoming bf16 gradient that is a 2-byte-offset view is copied in backward, not refused."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(13)
    x = _activation(gen, (6, 64, 8, 8), 3, dev).to(BF)
    g = _off_by_2_bytes(torch.randn(x.shape, device=dev, generator=gen).to(BF))
    ma, mb = dwt_b200.WTransform2d(64, 4).to(dev).train(), dwt_b200.WTransform2d(64, 4).to(dev).train()
    xa, xb = x.clone().requires_grad_(True), x.float().requires_grad_(True)
    ya, yb = ma(xa), mb(xb)
    assert ya.grad_fn.cfg[3] & dwt_b200._native.DTYPE_BF16
    ya.backward(g)
    yb.backward(g.float())
    assert _same(ya, yb.to(BF)) and _same(xa.grad, xb.grad.to(BF))


# --------------------------------------------------------------------------- the C ABI
def test_c_abi_return_codes(dev):
    from dwt_b200 import _native
    lib = _native.lib()
    assert lib.dwt_abi_version() == 10
    n, c, d = 2, 64, 1
    buf = torch.zeros(2 * n * c * 64 + 64, dtype=BF, device=dev)
    ok, off = buf.data_ptr(), buf.data_ptr() + 2            # 256-byte aligned / 2 bytes off
    out, res = torch.zeros_like(buf), torch.zeros_like(buf)
    st = torch.zeros(4 * c * 4, device=dev)
    gb = _native.ptr(st)
    rm = _native.ptr_array([st] * d)
    bf = _native.DTYPE_BF16
    V = ctypes.c_void_p

    def wfwd(x, hw, gs=4, residual=None, epi=0):
        ws = _native.workspace(dev, n, c, hw, gs, d)
        return lib.dwt_whiten_fwd(V(x), _native.ptr(out), n, c, hw, gs, d, bf, 1e-3, 0.1, 0, rm, rm, gb, gb,
                                  None if residual is None else V(residual), None, epi, gb, gb, _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr(dev))

    def wbwd(x, dout, hw, dout2=None):
        ws = _native.workspace(dev, n, c, hw, 4, d)
        return lib.dwt_whiten_bwd(V(x), V(dout), None if dout2 is None else V(dout2), _native.ptr(out), n, c, hw, 4, d, bf,
                                  1e-3, gb, gb, None, None, None, None, 0, None, None, _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr(dev))

    def bfwd(x, hw):
        ws = _native.workspace(dev, n, c, hw, 1, d)
        return lib.dwt_bn_fwd(V(x), _native.ptr(out), n, c, hw, d, bf, 1e-5, 0.1, 0, rm, rm, None, None, None, None, 0,
                              gb, gb, _native.ptr(ws), ws.numel(), _native.stream_ptr(dev))

    def bbwd(x, dout, hw):
        ws = _native.workspace(dev, n, c, hw, 1, d)
        return lib.dwt_bn_bwd(V(x), V(dout), None, _native.ptr(out), n, c, hw, d, bf, gb, gb, None, None, None, None, 0,
                              None, None, _native.ptr(ws), ws.numel(), _native.stream_ptr(dev))
    assert wfwd(ok, 16) == 0 and wbwd(ok, ok, 16) == 0      # 4 x 4, gs 4
    assert bfwd(ok, 16) == 0 and bbwd(ok, ok, 16) == 0
    assert wfwd(ok, 16, residual=res.data_ptr(), epi=7) == 0
    assert wfwd(ok, 9) == -4 and bfwd(ok, 9) == -4           # HW = 9: HW % 4 != 0
    assert b"multiple of 4" in lib.dwt_last_error()
    assert wbwd(ok, ok, 9) == -4
    for rc in (wfwd(off, 16), wbwd(ok, off, 16), wfwd(ok, 16, residual=res.data_ptr() + 2, epi=7), bfwd(off, 16),
               bbwd(ok, off, 16)):
        assert rc == -1
        assert b"8-byte" in lib.dwt_last_error()
    assert wbwd(ok, ok, 16, dout2=ok) == -4                  # NCHW dout2: added by the caller
    torch.cuda.synchronize(dev)
    _native.clear_status(dev)


# --------------------------------------------------------------------------- CUDA-graph capture
def test_graph_capture(dev):
    """A bf16 NCHW DomainTripleNorm site (gs 4, AFFINE|RELU) forward + backward captures into a CUDA graph, and two
    replays reproduce the eager result bit for bit."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(3)
    shape = (6, 64, 16, 16)
    x = _activation(gen, shape, 3, dev).to(BF)
    dy = torch.randn(shape, device=dev, generator=gen).to(BF)
    site = _Site("whiten", 64, 4, 3, "distinct", gen, dev)
    a = site.arm()
    r0 = [t.clone() for t in _Site.running(a)]

    def step():
        # a fresh leaf per step (see test_channels_last_tensor_core.test_graph_capture)
        xi = x.detach().requires_grad_(True)
        y = a.norm(xi, a.mods, a.gamma, a.beta, True)
        assert y.grad_fn.cfg[3] & dwt_b200._native.DTYPE_BF16, "the bf16 kernels did not run"
        return (y,) + torch.autograd.grad(y, (xi, a.gamma, a.beta), dy)
    eager = [t.detach().clone() for t in step()]
    r1 = [t.clone() for t in _Site.running(a)]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = step()
    for _ in range(2):
        for t, v in zip(_Site.running(a), r0):
            t.copy_(v)
        g.replay()
        torch.cuda.synchronize(dev)
        assert all(_same(p, q) for p, q in zip(got, eager))
        assert all(_same(p, q) for p, q in zip(_Site.running(a), r1))


# --------------------------------------------------------------------------- whole models under autocast
def _step(dev, build, images, patched, monkeypatch):
    """One training step under autocast; patched: the new routing off (the upcast path for every NCHW bf16 call)."""
    from dwt_b200 import _native, functional as F
    model = build()
    with monkeypatch.context() as mp:
        if patched:
            mp.setattr(F, "_bf16_small", lambda *a, **k: False)
        _native.profile_begin()
        with torch.autocast("cuda", dtype=BF):
            logits = model(images)
        loss = logits.float().logsumexp(1).mean()
        loss.backward()
        launches = {k: v["launches"] for k, v in _native.by_family(_native.profile_end()).items()}
    grads = [p.grad for p in model.parameters()]
    return logits.detach(), loss.detach(), grads, [b.clone() for b in model.buffers()], launches


@pytest.mark.parametrize("model_name", ["resnet-modules", "resnet-fused", "lenet"])
def test_model_step_equals_upcast_path(model_name, dev, monkeypatch):
    """A training step under torch.autocast: the bf16 kernels give the very step of the upcast path -- logits, loss,
    every parameter gradient and every buffer.  The only float32 small_stats launches left are layer4's 7x7 sites."""
    import dwt_b200
    from harness.lenet_dwt import LeNetDWT
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    if model_name == "lenet":
        torch.manual_seed(5)
        proto = LeNetDWT(dwt_b200).to(dev).train()
        images = torch.randn(2 * 64, 1, 28, 28, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
        build, fp32_stats = (lambda: copy.deepcopy(proto)), 0
    else:
        mode = model_name.split("-")[1]
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        images = synth_batch(seed=2, per_domain=2, size=224)[0].to(dev)
        build = lambda: build_resnet50_dwt({k: v.clone() for k, v in sd.items()}, dwt_b200, site_mode=mode).to(dev).train()  # noqa: E731
        fp32_stats = 27 if mode == "modules" else 9
    a = _step(dev, build, images, False, monkeypatch)
    b = _step(dev, build, images, True, monkeypatch)
    # (the LeNet's logits leave its last, stock BatchNorm1d site through a float32 affine: float32)
    assert a[0].dtype == (torch.float32 if model_name == "lenet" else BF)
    assert _same(a[0], b[0]) and _same(a[1], b[1]), "logits / loss"
    assert all(_same(p, q) for p, q in zip(a[2], b[2])), "gradients"
    assert all(_same(p, q) for p, q in zip(a[3], b[3])), "buffers"
    assert a[4].get("small_stats", 0) == fp32_stats, a[4]
    assert a[4].get("small_stats_bf16", 0) > 0 and "small_stats_bf16" not in b[4], (a[4], b[4])
