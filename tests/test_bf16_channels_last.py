"""bfloat16 activations (torch.autocast) on the channels-last kernels, against the float32 kernels, bit for bit.

A bf16 call runs the float32 schedule of its shape with loads widened and stores rounded to nearest-even
(include/dwt_b200.h, DWT_DTYPE_BF16).  So every comparison here is torch.equal (NaN-aware where NaN is the point):

  * each site in bf16 against the float32 kernels on x.float() (residual.float(); where the output is forked,
    RN_bf16(dout + dout2).float() as the single gradient): y == y32.to(bf16), the byte map, dx == dx32.to(bf16),
    d_identity == dz32.to(bf16), dgamma / dbeta, save_mean / save_w, every running buffer, num_batches_tracked and the
    status word -- at every site geometry of the harness ResNet-50-DWT (2 images per domain), at launch edges of
    norm_cl.cu, at the benchmark's 3 x 64 images, in train / no-grad / eval / replicated mode, and with a NaN input;
  * the two-site tail against its own bf16 two-call composition, fork_for_sum against autograd's bf16 add;
  * MaxPool2d against F.max_pool2d; the upcast fallbacks; the head losses; refusals;
  * the whole model under autocast: only bf16 kernel families run, and loss and logits stay near the float32 step.
"""
import ctypes
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
CL = torch.channels_last
GIB = 1 << 30


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    d = torch.device("cuda", 0)
    torch.cuda.reset_peak_memory_stats(d)
    t0 = time.perf_counter()
    yield d
    print(f"\ntest_bf16_channels_last: {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated(d) / GIB:.2f} GiB")


def _same(a, b):
    """torch.equal, with NaN equal to NaN (bf16 NaN payloads are not compared)."""
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.isnan(), b.isnan()) and \
        torch.equal(a.nan_to_num(0.0), b.nan_to_num(0.0))


def _activation(gen, shape, d, dev):
    """Channels-last float32 activations: correlated neighbouring channels, per-channel scales, a mean per domain."""
    n_all, c, h, w = shape
    z = torch.randn(n_all, h, w, c, device=dev, generator=gen).permute(0, 3, 1, 2)
    z.add_(z.roll(1, 1), alpha=0.6)
    z.mul_(0.5 + torch.rand(c, 1, 1, device=dev, generator=gen))
    n = n_all // d
    for k in range(d):
        z[k * n:(k + 1) * n].add_(0.6 * k - 0.5)
    return z


class _Site:
    """A norm site's state -- the D domain modules on running buffers aliased 'shared', 'distinct' or 'mixed', gamma,
    beta -- built twice from the same values: one copy per arm."""

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
        """Every running tensor of an arm, in a fixed order."""
        out = [t for o in sorted(a.bufs) for t in a.bufs[o]]
        return out + [m.num_batches_tracked for m in a.mods if hasattr(m, "num_batches_tracked")]


def _run_arm(dt, sites, x0, r0, xd0, g1, g2, *, path, mode, fork):
    """One arm: the site(s) on x0 (and r0 / xd0) cast to dt.  Returns a dict of everything to compare."""
    import dwt_b200
    from dwt_b200 import _native, functional as F
    dev = x0.device
    arms = [s.arm() for s in sites]
    a = arms[0]
    grad = mode == "train"
    x = x0.to(dt).detach().requires_grad_(grad)
    r = r0.to(dt).detach().requires_grad_(grad) if r0 is not None else None
    xd = xd0.to(dt).detach().requires_grad_(grad) if xd0 is not None else None
    _native.clear_status(dev)
    with torch.set_grad_enabled(grad):
        if mode == "eval":
            s = sites[0]
            second = "running_variance" if s.kind == "whiten" else "running_var"
            y = F.norm(x, a.gamma, a.beta, kind=s.kind, group_size=s.gs, n_domains=s.d, training_stats=False, eps=1e-5,
                       momentum=0.1, update_running=False, running=[(m.running_mean, getattr(m, second)) for m in a.mods],
                       relu=True, residual=r)
        elif mode == "replicated":
            y = a.norm(x, a.mods, a.gamma, a.beta, relu=True, residual=r, replicated=True)
        elif path == "tail2":
            b = arms[1]
            y = a.norm.forward_with_downsample(x, a.mods, a.gamma, a.beta, xd, b.norm, b.mods, b.gamma, b.beta)
        elif path in ("tail2_composed", "tail2_rounded"):
            b = arms[1]
            identity = b.norm(xd, b.mods, b.gamma, b.beta, relu=False)
            if path == "tail2_rounded":              # the identity as a bf16 caller stores it (its gradient is exact in bf16)
                identity = identity.to(BF).to(dt)
            y = a.norm(x, a.mods, a.gamma, a.beta, True, residual=identity)
        else:
            y = a.norm(x, a.mods, a.gamma, a.beta, relu=True, residual=r)
    out = {"y": y.detach(), "status": _native.status(dev)}
    if grad:
        saved = y.grad_fn.saved_tensors
        name = type(y.grad_fn).__name__
        if name.startswith("_TailPairFunction"):
            out["mask"], out["stats"] = saved[2], [saved[3], saved[4], saved[6], saved[7]]
        elif name.startswith("_NormFunction"):
            assert dt == torch.float32 or y.grad_fn.cfg[3] & _native.DTYPE_BF16, "the bf16 kernels did not run"
            out["mask"] = saved[5] if len(saved) > 5 else None
            out["stats"] = [saved[1], saved[2]]
        del saved
        if fork == "kernels":                        # the two gradients reach the kernels apart
            u, v = dwt_b200.fork_for_sum(y)
            torch.autograd.backward([u, v], [g1.to(dt), g2.to(dt)])
        elif fork == "autograd":                     # y used twice: autograd adds the two gradients (in dt)
            ((y * g1.to(dt)).sum() + (y * g2.to(dt)).sum()).backward()
        else:
            y.backward(g1.to(dt))
        out["dx"] = x.grad
        out["d_res"] = r.grad if r is not None else None
        out["dxd"] = xd.grad if xd is not None else None
        out["dgb"] = [t.grad for s in arms for t in (s.gamma, s.beta)]
    out["running"] = [t for s, arm in zip(sites, arms) for t in _Site.running(arm)]
    return out


def _compare_to_fp32(bf, ref, grad):
    """bf16 arm against the float32 arm on the upcast inputs."""
    assert bf["y"].dtype == BF and bf["y"].is_contiguous(memory_format=CL)
    assert _same(bf["y"], ref["y"].to(BF)), "y"
    assert bf["status"] == ref["status"], (bf["status"], ref["status"])
    for k, (p, q) in enumerate(zip(bf["running"], ref["running"])):
        assert _same(p, q), f"running buffer {k}"
    if not grad:
        return
    assert _same(bf.get("mask"), ref.get("mask")), "byte map"
    for k, (p, q) in enumerate(zip(bf["stats"], ref["stats"])):
        assert _same(p, q), f"save_mean / save_w {k}"
    assert _same(bf["dx"], ref["dx"].to(BF)), "dx"
    for key in ("d_res", "dxd"):
        assert _same(bf[key], None if ref[key] is None else ref[key].to(BF)), key
    for k, (p, q) in enumerate(zip(bf["dgb"], ref["dgb"])):
        assert _same(p, q), f"dgamma / dbeta {k}"


def _case(dev, *, kind, c, gs, d, n, h, w, path, fork=False, mode="train", layouts=("shared", "shared"), seed=0, nan=False):
    """One site in bf16 and in float32 on the upcast inputs; asserts every comparison."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    shape = (d * n, c, h, w)
    x = _activation(gen, shape, d, dev).to(BF)
    if nan:
        x[0, 1, 0, 0] = float("nan")
    r = _activation(gen, shape, d, dev).to(BF) if path == "residual" else None
    xd = _activation(gen, shape, d, dev).to(BF) if path == "tail2" else None
    g1 = torch.randn(shape, device=dev, generator=gen).to(BF).contiguous(memory_format=CL)
    g2 = torch.randn(shape, device=dev, generator=gen).to(BF).contiguous(memory_format=CL) if fork else None
    sites = [_Site(kind, c, gs, d, layouts[0], gen, dev)]
    if path == "tail2":
        sites.append(_Site(kind, c, gs, d, layouts[1], gen, dev))
    bf = _run_arm(BF, sites, x, r, xd, g1, g2, path=path, mode=mode, fork="kernels" if fork else None)
    # the float32 reference takes RN_bf16(dout + dout2) -- autograd's bf16 sum -- as its one gradient; for the two-site
    # tail it is the float32 two-call composition (bit for bit the float32 two-site kernels) with the identity rounded
    # to bf16, as the bf16 kernels round it before they add it
    ref = _run_arm(torch.float32, sites, x, r, xd, (g1 + g2) if fork else g1, None, path="tail2_rounded" if path == "tail2" else path,
                   mode=mode, fork=None)
    _compare_to_fp32(bf, ref, mode == "train")
    return bf, ref


# --------------------------------------------------------------------------- every site of the training step
@pytest.fixture(scope="module")
def model_sites(dev):
    """(kind, C, H, W, gs, path, forked) of every DomainTripleNorm call of a channels-last fused training forward of
    the harness ResNet-50-DWT at 224^2, recorded at the functional entry points, duplicates removed."""
    import dwt_b200
    from dwt_b200 import functional as F
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    calls, forked = [], []
    norm, tail_pair, fork = F.norm, F.tail_pair, dwt_b200.fork_for_sum

    def rec_norm(x, *args, **kw):
        y = norm(x, *args, **kw)
        calls.append(((kw["kind"], x.shape[1], x.shape[2], x.shape[3], kw["group_size"],
                       "plain" if kw.get("residual") is None else "residual"), y))
        return y

    def rec_tail_pair(x, xd, *args, **kw):
        y = tail_pair(x, xd, *args, **kw)
        calls.append(((kw["kind"], x.shape[1], x.shape[2], x.shape[3], kw["group_size"], "tail2"), y))
        return y

    def rec_fork(y):
        forked.append(y)
        return fork(y)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(F, "norm", rec_norm)
        mp.setattr(F, "tail_pair", rec_tail_pair)
        mp.setattr(dwt_b200, "fork_for_sum", rec_fork)
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        model = build_resnet50_dwt(sd, dwt_b200, site_mode="fused", channels_last=True).to(dev).train()
        images, _ = synth_batch(seed=2, per_domain=1, size=224)
        model(images.to(dev).contiguous(memory_format=CL))
    sites = []
    for key, y in calls:
        entry = key + (any(f is y for f in forked),)
        if entry not in sites:
            sites.append(entry)
    return sites


def test_every_model_site_geometry(model_sites, dev):
    """Each distinct site of the training step at 2 images per domain, as the model runs it (forked where it is)."""
    assert len(model_sites) == 17, model_sites
    failures = []
    for i, (kind, c, h, w, gs, path, fork) in enumerate(model_sites):
        try:
            _case(dev, kind=kind, c=c, gs=gs, d=3, n=2, h=h, w=w, path=path, fork=fork, seed=200 + i)
        except AssertionError as e:
            failures.append(f"{kind} {c}@{h}x{w} gs{gs} {path}{' forked' if fork else ''}: {e}")
    assert not failures, "\n".join(failures)


# --------------------------------------------------------------------------- modes, buffers, forks, edges
MODES = [   # kind, C, gs, path, mode, fork, running buffers (site, downsample site)
    ("whiten", 64, 4, "plain", "nograd", False, ("shared", None)),
    ("whiten", 64, 2, "residual", "eval", False, ("distinct", None)),
    ("bn", 256, 1, "plain", "eval", False, ("mixed", None)),
    ("whiten", 64, 4, "plain", "replicated", False, ("shared", None)),
    ("bn", 256, 1, "residual", "replicated", False, ("distinct", None)),
    ("whiten", 128, 1, "plain", "train", False, ("mixed", None)),
    ("whiten", 128, 2, "residual", "train", True, ("distinct", None)),
    ("bn", 512, 1, "tail2", "train", False, ("distinct", "mixed")),
    ("whiten", 256, 4, "tail2", "train", True, ("mixed", "shared")),
]


@pytest.mark.parametrize("kind,c,gs,path,mode,fork,layouts", MODES,
                         ids=[f"{m[0]}-c{m[1]}-gs{m[2]}-{m[3]}-{m[4]}{'-forked' if m[5] else ''}-{m[6][0]}" for m in MODES])
def test_modes_and_buffers(kind, c, gs, path, mode, fork, layouts, dev):
    _case(dev, kind=kind, c=c, gs=gs, d=3, n=2, h=9, w=9, path=path, fork=fork, mode=mode, layouts=layouts, seed=c + gs)


EDGES = [   # C, path, kind, gs, domains, (N, H, W) per domain, forked, layouts
    (4, "plain", "whiten", 4, 3, (1, 2, 2), False, ("shared", None)),        # < 8 rows
    (4, "tail2", "bn", 1, 4, (1, 1, 64 * 8), True, ("distinct", "shared")),  # one chunk (rpi 64 x unroll 8)
    (16, "residual", "whiten", 2, 2, (1, 1, 64 * 8 + 1), True, ("shared", None)),   # one chunk + 1 (rpi 16 -> 128 rows)
    (1024, "plain", "bn", 1, 3, (3, 57, 61), False, ("shared", None)),       # capped, ragged grid
    (4096, "residual", "whiten", 4, 1, (1, 3, 3), True, ("shared", None)),   # grid.y = 4
    (4096, "tail2", "whiten", 2, 3, (2, 5, 7), False, ("mixed", "distinct")),
]


@pytest.mark.parametrize("c,path,kind,gs,d,nhw,fork,layouts", EDGES,
                         ids=[f"c{e[0]}-{e[1]}-{e[2]}-gs{e[3]}-d{e[4]}-{'x'.join(map(str, e[5]))}" for e in EDGES])
def test_launch_edges(c, path, kind, gs, d, nhw, fork, layouts, dev):
    n, h, w = nhw
    _case(dev, kind=kind, c=c, gs=gs, d=d, n=n, h=h, w=w, path=path, fork=fork, layouts=layouts, seed=c + d)


def test_bench_size_site(dev):
    """layer1.0's two-site tail at the benchmark's 3 x 64 images per call (grid.x capped, hundreds of rows per thread)."""
    _case(dev, kind="whiten", c=256, gs=4, d=3, n=64, h=56, w=56, path="tail2", fork=True, seed=7)


@pytest.mark.parametrize("path", ["plain", "tail2"])
def test_nan_input_sets_the_same_status_and_skips_the_same_ema(path, dev):
    """A NaN in domain 0: its group's covariance is not positive definite -- the same status bit as float32, the same
    skipped running-statistic update, and NaN in the same places of every output and gradient."""
    from dwt_b200 import _native
    bf, _ = _case(dev, kind="whiten", c=64, gs=4, d=3, n=2, h=6, w=6, path=path, layouts=("distinct", "distinct"),
                  seed=5, nan=True)
    assert bf["status"] & _native.STATUS_NOT_PD
    _native.clear_status(dev)


# --------------------------------------------------------------------------- the two-site tail, fork_for_sum
@pytest.mark.parametrize("fork", [False, True], ids=["single", "forked"])
@pytest.mark.parametrize("kind,c,gs,h", [("whiten", 256, 4, 56), ("bn", 512, 1, 28)])
def test_tail_pair_equals_two_call_composition(kind, c, gs, h, fork, dev):
    """forward_with_downsample in bf16 == its bf16 two-call composition (identity stored in bf16, then added)."""
    gen = torch.Generator(device=dev).manual_seed(c + int(fork))
    shape = (6, c, h, h)
    x, xd = (_activation(gen, shape, 3, dev).to(BF) for _ in range(2))
    g1 = torch.randn(shape, device=dev, generator=gen).to(BF).contiguous(memory_format=CL)
    g2 = torch.randn(shape, device=dev, generator=gen).to(BF).contiguous(memory_format=CL)
    sites = [_Site(kind, c, gs, 3, "shared", gen, dev) for _ in range(2)]
    mode = "kernels" if fork else None
    a = _run_arm(BF, sites, x, None, xd, g1, g2, path="tail2", mode="train", fork=mode)
    b = _run_arm(BF, sites, x, None, xd, g1, g2, path="tail2_composed", mode="train", fork=mode)
    assert _same(a["y"], b["y"]) and _same(a["mask"], b["mask"])
    for key in ("dx", "dxd"):
        assert _same(a[key], b[key]), key
    for p, q in zip(a["dgb"] + a["running"], b["dgb"] + b["running"]):
        assert _same(p, q)


@pytest.mark.parametrize("path", ["plain", "residual", "tail2"])
def test_fork_for_sum_equals_autograds_add(path, dev):
    """The two gradients of a forked bf16 output summed in the kernels == autograd's own bf16 addition."""
    gen = torch.Generator(device=dev).manual_seed(3)
    shape = (6, 256, 14, 14)
    x = _activation(gen, shape, 3, dev).to(BF)
    r = _activation(gen, shape, 3, dev).to(BF) if path == "residual" else None
    xd = _activation(gen, shape, 3, dev).to(BF) if path == "tail2" else None
    g1, g2 = (torch.randn(shape, device=dev, generator=gen).to(BF).contiguous(memory_format=CL) for _ in range(2))
    sites = [_Site("bn", 256, 1, 3, "shared", gen, dev) for _ in range(2 if path == "tail2" else 1)]
    a = _run_arm(BF, sites, x, r, xd, g1, g2, path=path, mode="train", fork="kernels")
    b = _run_arm(BF, sites, x, r, xd, g1, g2, path=path, mode="train", fork="autograd")
    for key in ("dx", "d_res", "dxd"):
        assert _same(a[key], b[key]), key
    for p, q in zip(a["dgb"], b["dgb"]):
        assert _same(p, q)


# --------------------------------------------------------------------------- max-pool
@pytest.mark.parametrize("shape,k,s,p", [((6, 64, 112, 112), 3, 2, 1), ((3, 8, 9, 7), 3, 2, 1), ((2, 16, 8, 8), 2, 2, 0),
                                          ((2, 4, 5, 6), 3, 1, 1), ((1, 12, 7, 7), 5, 3, 2), ((2, 8, 10, 6), 3, 2, 1),
                                          ((3, 4, 2, 2), 3, 2, 1), ((2, 12, 8, 8), 3, 2, 1), ((1, 4, 4, 4), 3, 2, 1)])
def test_maxpool_bf16_matches_torch(shape, k, s, p, dev):
    """MaxPool2d on bf16 channels-last input == F.max_pool2d on it, forward and backward: ties (post-ReLU zeros and
    values rounded to bf16) and NaN."""
    import torch.nn.functional as Fn
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(sum(shape) + k)
    x = torch.relu(torch.randn(*shape, device=dev, generator=gen)).to(BF).contiguous(memory_format=CL)
    x[0, 0, 0, 0] = float("nan")
    oh, ow = (shape[2] + 2 * p - k) // s + 1, (shape[3] + 2 * p - k) // s + 1
    g = torch.randn(shape[0], shape[1], oh, ow, device=dev, generator=gen).to(BF)
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    ya = dwt_b200.MaxPool2d(k, s, p)(xa)
    yb = Fn.max_pool2d(xb, k, s, p)
    assert ya.dtype == BF and ya.is_contiguous(memory_format=CL)
    assert _same(ya, yb)
    ya.backward(g)
    yb.backward(g)
    assert xa.grad.dtype == BF and _same(xa.grad, xb.grad)


# --------------------------------------------------------------------------- fallbacks, losses, refusals
def test_upcast_fallbacks(dev):
    """bf16 calls without a bf16 kernel run the float32 kernels on upcast copies: == fp32(x.float()).to(bf16)."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(9)
    cases = [(dwt_b200.WTransform2d(64, 4), torch.randn(6, 64, 9, 9, device=dev, generator=gen)),              # NCHW gs 4
             (dwt_b200.WTransform2d(64, 64), torch.randn(4, 64, 32, 32, device=dev, generator=gen) * 2 + 1)]   # M = 4096: tensor cores
    for mod, x32 in cases:
        ma, mb = mod.to(dev).train(), type(mod)(64, mod.group_size).to(dev).train()
        x = x32.to(BF)
        xa, xb = x.clone().requires_grad_(True), x.float().requires_grad_(True)
        ya, yb = ma(xa), mb(xb)
        assert ya.dtype == BF and _same(ya, yb.to(BF))
        g = torch.randn(x.shape, device=dev, generator=gen).to(BF)
        ya.backward(g)
        yb.backward(g.float())
        assert xa.grad.dtype == BF and _same(xa.grad, xb.grad.to(BF))
        assert _same(ma.running_mean, mb.running_mean) and _same(ma.running_variance, mb.running_variance)
    # a fused site with gs 8 (tensor epilogue) returns x's dtype
    site = dwt_b200.DomainTripleNorm("whiten", 64, 8)
    mods = [dwt_b200.WTransform2d(64, 8).to(dev).train() for _ in range(3)]
    g, b = torch.ones(64, 1, 1, device=dev), torch.zeros(64, 1, 1, device=dev)
    y = site(torch.randn(6, 64, 5, 5, device=dev, generator=gen).to(BF).contiguous(memory_format=CL), mods, g, b, relu=True)
    assert y.dtype == BF


def test_head_losses_on_bf16_logits(dev):
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(4)
    logits = (3 * torch.randn(3 * 8, 65, device=dev, generator=gen)).to(BF)
    labels = torch.randint(0, 65, (8,), device=dev, generator=gen)
    la, lb = logits.clone().requires_grad_(True), logits.float().requires_grad_(True)
    head = dwt_b200.HeadLoss(65, 0.1)
    ta, tb = head(la, labels), head(lb, labels)
    assert ta.dtype == torch.float32 and torch.equal(ta, tb)
    ta.backward()
    tb.backward()
    assert la.grad.dtype == BF and torch.equal(la.grad, lb.grad.to(BF))
    mec = dwt_b200.MinEntropyConsensusLoss(65, dev)
    xa, ya_ = (t.clone().requires_grad_(True) for t in logits[:16].split(8))
    xb, yb_ = (t.float().requires_grad_(True) for t in logits[:16].split(8))
    ma, mb = mec(xa, ya_), mec(xb, yb_)
    assert torch.equal(ma, mb)
    ma.backward()
    mb.backward()
    assert torch.equal(xa.grad, xb.grad.to(BF)) and torch.equal(ya_.grad, yb_.grad.to(BF))


def test_refusals(dev):
    import dwt_b200
    from dwt_b200 import _native
    with pytest.raises(_native.NativeError, match="float32"):
        dwt_b200.WTransform2d(8, 4).to(dev)(torch.zeros(2, 8, 3, 3, device=dev, dtype=torch.float16))
    with pytest.raises(_native.NativeError, match="float32"):
        dwt_b200.MaxPool2d(3, 2, 1)(torch.zeros(2, 8, 4, 4, device=dev, dtype=torch.float16).contiguous(memory_format=CL))
    lib = _native.lib()
    n, c, hw, d = 2, 64, 9, 3
    ws = _native.workspace(dev, n, c, hw, 8, d)
    t = torch.zeros(2 * d * n * c * hw + 64, dtype=BF, device=dev)
    ok, off = t.data_ptr(), t.data_ptr() + 2               # 256-byte aligned / 2 bytes off
    st = torch.zeros(d * c * 8, device=dev)
    rm = _native.ptr_array([st] * d)

    def whiten(x, gs, mode):
        return lib.dwt_whiten_fwd(ctypes.c_void_p(x), ctypes.c_void_p(ok), n, c, hw, gs, d, mode, 1e-5, 0.1, 0, rm, rm, None,
                                  None, None, None, 0, _native.ptr(st), _native.ptr(st), _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr(dev))
    bf, nhwc = _native.DTYPE_BF16, _native.LAYOUT_NHWC
    assert whiten(ok, 4, bf) == -4                          # NCHW
    assert whiten(ok, 8, bf | nhwc) == -4                   # gs 8
    assert whiten(off, 4, bf | nhwc) == -1                  # misaligned
    assert b"8-byte" in lib.dwt_last_error()
    rc = lib.dwt_whiten_bwd(ctypes.c_void_p(ok), ctypes.c_void_p(ok), None, ctypes.c_void_p(ok), n, c, hw, 8, d, bf | nhwc, 1e-5,
                            _native.ptr(st), _native.ptr(st), None, None, None, None, 0, None, None, _native.ptr(ws), ws.numel(),
                            _native.stream_ptr(dev))
    assert rc == -4
    rc = lib.dwt_maxpool_fwd(ctypes.c_void_p(off), ctypes.c_void_p(ok), ctypes.c_void_p(ok), 1, 4, 4, 8, 3, 2, 1, bf,
                             _native.stream_ptr(dev))
    assert rc == -1
    torch.cuda.synchronize(dev)


# --------------------------------------------------------------------------- the whole model under autocast
# Accuracy of the bf16 step against the float32 step (3 x 2 images at 224^2, harness ResNet-50-DWT, fused sites,
# channels-last, s2d stem, synthetic weights), measured on an H100 80GB HBM3 over image seeds 0, 1, 2:
#   loss relative error      8.9e-3, 1.3e-3, 9.3e-3
#   logits norm-wise         8.3e-2, 8.5e-2, 9.2e-2
#   logits max-elementwise   1.14e-1, 1.14e-1, 1.15e-1   (relative to max |logit|)
# The bounds are twice the worst of the three.
MODEL_BOUNDS = (1.86e-2, 1.84e-1, 2.31e-1)


def _model_step(dev, seed, autocast):
    import dwt_b200
    from dwt_b200 import _native
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
    model = build_resnet50_dwt(sd, dwt_b200, site_mode="fused", channels_last=True, stem_s2d=True).to(dev).train()
    images, labels = synth_batch(seed=seed, per_domain=2, size=224)
    images, labels = images.to(dev).contiguous(memory_format=CL), labels.to(dev)
    head = dwt_b200.HeadLoss(65, 0.1)
    _native.profile_begin()
    with torch.autocast("cuda", dtype=BF, enabled=autocast):
        logits = model(images)
        loss = head(logits, labels)
    loss.backward()
    fams = _native.by_family(_native.profile_end())
    return float(loss.detach()), logits.detach().float(), fams


def test_model_step_under_autocast(dev):
    """The harness model's training step under autocast: no float32 norm or max-pool kernel runs, and loss and logits
    stay within MODEL_BOUNDS of the float32 step."""
    errs = []
    for seed in range(3):
        l32, z32, _ = _model_step(dev, seed, False)
        l16, z16, fams = _model_step(dev, seed, True)
        lib_fams = [f for f in fams if f.startswith(("cl_", "maxpool", "small_", "tiled_", "tc_", "dense_", "eval_prep",
                                                     "bwd_prep"))]
        assert lib_fams and all(f.endswith("_bf16") for f in lib_fams), sorted(fams)
        assert any(f.startswith("maxpool_fwd") for f in lib_fams) and any(f.startswith("cl_tail2") for f in lib_fams)
        errs.append((abs(l16 - l32) / abs(l32), ((z16 - z32).norm() / z32.norm()).item(),
                     ((z16 - z32).abs().max() / z32.abs().max()).item()))
    print("bf16 vs fp32 step (loss rel, logits norm-wise, logits max-elementwise):", errs)
    for e in errs:
        assert all(v <= b for v, b in zip(e, MODEL_BOUNDS)), (e, MODEL_BOUNDS)
