"""The channels-last (NHWC) norm sites -- plain, residual tail, two-site tail -- against an fp64 reference on the GPU.

Reference: oracle/torch_port.py's WTransform2d / BatchNorm2d in float64 (the reference's operator sequence, pinned to
the reference's own outputs by test_oracle_vs_golden.py), composed as the reference composes a site: the D domain
modules called in order on the site's running buffers (so the EMA runs source -> target -> ...), then * gamma + beta,
+ identity, ReLU.  For the two-site tail of a downsampling Bottleneck the identity is the downsample site's composition
without the ReLU.  The elementwise steps commute with the reference's cat, so the reference runs one domain at a time
and its fp64 graph never holds more than one domain.  Backward: fp64 autograd, with the ReLU derivative taken where the
kernel put it -- the fp64 pre-activation times the kernel's decoded byte map (residual sites) or its out > 0 (plain
sites), as a constant.  The two masks may disagree only on elements within rounding of zero; that is asserted.

Compared for every case, norm-wise with the max-elementwise error beside it: the output, the byte map (bit for bit
against the kernel's own out > 0), dx, dxd, d_identity, dgamma / dbeta of each site, each site's batch mean and
covariance (recovered from the saved W), every running buffer (BN: unbiased variance, momentum=None),
num_batches_tracked and the status word.

Cases:
  * every site geometry of one channels-last training forward of the harness ResNet-50-DWT at 224^2, recorded from
    the model, run at 2 images per domain;
  * launch edges of norm_cl.cu, derived from rpi, the statistics kernel's unroll and the SM count: C/4 < 8 (one column
    shared by up to 256 threads), C = 1024 / 2048 / 4096 (rpi = 1, grid.y = 1 / 2 / 4), group sizes 1 / 2 / 4, fewer
    rows than 8 and than rpi, exactly one chunk, one chunk + 1, a chunk count that is not a multiple of the capped
    grid, 1 to 4 domains, shared / distinct / mixed running buffers;
  * the benchmark's 3 x 64 images per call, where cl_plan caps the grid and every thread sums hundreds of rows;
  * pilot-shift robustness there: |mean| = 50 sigma, and a first image whose top row is 30 sigma off.

Tolerances as in test_gpu_parity_r2.py: 1e-3 norm-wise through a Cholesky factor, 1e-4 on BN outputs and on
statistics; max-elementwise (scaled by max |reference|) below 5x the norm-wise bound.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-3
TOL_STAT = 1e-4
TOL_MAX = 5e-3
GIB = 1 << 30
CL = torch.channels_last
BENCH_PER_DOMAIN = 64            # bench.py's workload: 3 x 64 images per norm-site call
# launch shape of the channels-last kernels (norm_cl.cu, cl_plan in api.cu)
THREADS = 256                    # threads per CTA; a CTA covers min(C/4, 256) float4 columns x rpi row lanes
STATS_UNROLL = 8                 # rows per thread and chunk of cl_stats_kernel
STATS_SLOTS = 3                  # CTAs per SM of cl_stats: grid.x <= 3 * SMs / (grid.y * D)
STAT_KEYS = ("mean", "cov", "running")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst(dev):
    """Worst (norm-wise, max-elementwise) error per (path, size), printed with the peak device memory at the end."""
    torch.cuda.reset_peak_memory_stats(dev)
    table = {}
    yield table
    print("\nworst errors (norm-wise, max-elementwise):")
    for key in sorted(table):
        print("  %-28s %s" % (" / ".join(key), ", ".join(f"{k} {r:.1e} {m:.1e}" for k, (r, m) in sorted(table[key].items()))))
    print(f"peak device memory: {torch.cuda.max_memory_allocated(dev) / GIB:.2f} GiB")


class _Err:
    """||a - b|| / ||b|| and max|a - b| / max|b| (conftest.rel_err / max_err) accumulated over slices, in float64."""

    def __init__(self):
        self.d2 = self.r2 = self.dmax = self.rmax = 0.0

    def add(self, got, ref):
        diff = got.double() - ref
        self.d2 += diff.square().sum().item()
        self.r2 += ref.square().sum().item()
        self.dmax = max(self.dmax, diff.abs().max().item())
        self.rmax = max(self.rmax, ref.abs().max().item())

    def both(self):
        return math.sqrt(self.d2) / max(math.sqrt(self.r2), 1e-30), self.dmax / max(self.rmax, 1e-30)


def _launch(c, d, sms):
    """(rpi, capped grid.x of cl_stats) of a channels-last site with C channels and d domains."""
    cw = min(c // 4, THREADS)
    gridy = (c // 4) // cw
    return THREADS // cw, max(1, STATS_SLOTS * sms // (gridy * d))


def _edge_rows(rows, c, d, sms):
    """Rows per domain of a named launch edge."""
    rpi, cap = _launch(c, d, sms)
    chunk = rpi * STATS_UNROLL
    if rows == "lt_rpi":
        assert 9 < rpi
    n = {"lt8": 4, "lt_rpi": 9, "chunk": chunk, "chunk+1": chunk + 1, "ragged": (2 * cap + 7) * chunk - 5}[rows]
    if rows == "ragged":      # enough work for the capped grid, and a last round in which only some CTAs have a chunk
        assert n // (2 * chunk) >= cap and -(-n // chunk) % cap != 0
    return n


def _activation(gen, shape, d, dev):
    """Channels-last activations: neighbouring channels correlated (inside whitening groups too), per-channel scales,
    a different mean in every domain."""
    n_all, c, h, w = shape
    z = torch.randn(n_all, h, w, c, device=dev, generator=gen).permute(0, 3, 1, 2)
    z.add_(z.roll(1, 1), alpha=0.6)
    z.mul_(0.5 + torch.rand(c, 1, 1, device=dev, generator=gen))
    n = n_all // d
    for k in range(d):
        z[k * n:(k + 1) * n].add_(0.6 * k - 0.5)
    return z


def _f64(t):
    return t.detach().to(torch.float64, memory_format=torch.contiguous_format)


def _decode(mask, shape):
    """The residual tail's byte map (one byte per float4 of the NHWC tensor, bit i = channel 4q + i) -> bool [N,C,H,W]."""
    n, c, h, w = shape
    bits = torch.arange(4, device=mask.device, dtype=torch.uint8)
    b = (mask.view(n, h, w, c // 4, 1) >> bits) & 1
    return b.view(n, h, w, c).permute(0, 3, 1, 2).bool()


class _Site:
    """One norm site twice: CUDA (fp32 modules, DomainTripleNorm) and reference (fp64 torch_port modules), with the same
    initial running buffers, aliased alike: 'shared' (one pair, as in the model), 'distinct' or 'mixed'."""

    def __init__(self, kind, c, gs, d, layout, gen, dev):
        import dwt_b200
        import oracle.torch_port as port
        self.kind, self.gs = kind, gs
        self.owner = {"shared": [0] * d, "distinct": list(range(d)), "mixed": [0] + [1] * (d - 1)}[layout]
        assert layout != "mixed" or d >= 3
        self.buf32, self.buf64 = {}, {}
        for o in sorted(set(self.owner)):
            rm = 0.1 * torch.randn(c, device=dev, generator=gen)
            if kind == "whiten":
                a = torch.randn(c // gs, gs, gs, device=dev, generator=gen)
                rv = a @ a.transpose(1, 2) / gs + 0.5 * torch.eye(gs, device=dev)
                rm = rm.view(1, c, 1, 1)
            else:
                rv = 0.5 + torch.rand(c, device=dev, generator=gen)
            self.buf32[o], self.buf64[o] = (rm, rv), (rm.double(), rv.double())
        if kind == "whiten":
            self.mods = [dwt_b200.WTransform2d(c, gs, running_m=self.buf32[o][0], running_var=self.buf32[o][1]).train()
                         for o in self.owner]
            self.ref = [port.WTransform2d(c, gs, running_m=self.buf64[o][0], running_var=self.buf64[o][1]).train()
                        for o in self.owner]
        else:
            self.mods = [dwt_b200.BatchNorm2d(c, *self.buf32[o], affine=False, momentum=None).train() for o in self.owner]
            self.ref = [port.BatchNorm2d(c, *self.buf64[o], affine=False, momentum=None).train() for o in self.owner]
            for m in self.mods + self.ref:
                m.num_batches_tracked.fill_(2)          # momentum=None: cumulative average, EMA factor 1/3
        self.eps = self.mods[0].eps
        self.gamma = (0.5 + torch.rand(c, 1, 1, device=dev, generator=gen)).requires_grad_(True)
        self.beta = (0.3 * torch.randn(c, 1, 1, device=dev, generator=gen)).requires_grad_(True)
        self.g64 = self.gamma.detach().double().requires_grad_(True)
        self.b64 = self.beta.detach().double().requires_grad_(True)
        self.norm = dwt_b200.DomainTripleNorm(kind, c, gs, n_domains=d)

    def batch_stats(self, x64):
        """fp64 batch mean and (biased) covariance / variance of one domain."""
        mu = x64.mean(dim=(0, 2, 3))
        xc = x64 - mu.view(1, -1, 1, 1)
        if self.kind == "bn":
            return mu, xc.square().mean(dim=(0, 2, 3))
        t = xc.transpose(0, 1).reshape(x64.shape[1] // self.gs, self.gs, -1)
        return mu, t @ t.mT / t.shape[-1]

    def kernel_cov(self, w):
        """The covariance the kernel factored, from its saved W: S = a cov + b I = L L^T, W = L^-1 (BN: W = 1/sqrt(var + eps))."""
        w = w.double()
        if self.kind == "bn":
            return 1.0 / w.reshape(-1).square() - self.eps
        winv = torch.linalg.inv(w)
        eye = torch.eye(self.gs, dtype=torch.float64, device=w.device)
        return (winv @ winv.mT - self.eps * eye) / (1.0 - self.eps)


def _check(dev, worst, label, size, *, kind, c, gs, d, n, h, w, path, fork, layouts=("shared", "shared"), seed=0,
           make_x=None):
    """Run one site on the channels-last kernels and on the fp64 reference; assert every comparison, return the errors."""
    import dwt_b200
    from dwt_b200 import _native
    gen = torch.Generator(device=dev).manual_seed(seed)
    shape = (d * n, c, h, w)
    x = (make_x or _activation)(gen, shape, d, dev).requires_grad_(True)
    xd = _activation(gen, shape, d, dev).requires_grad_(True) if path == "tail2" else None      # downsample input
    r = _activation(gen, shape, d, dev).requires_grad_(True) if path == "residual" else None    # identity branch
    w1 = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=CL)
    w2 = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=CL) if fork else None
    sites = [_Site(kind, c, gs, d, layouts[0], gen, dev)]
    if path == "tail2":
        sites.append(_Site(kind, c, gs, d, layouts[1], gen, dev))
    site = sites[0]
    _native.clear_status(dev)

    # ---- CUDA
    if path == "plain":
        y = site.norm(x, site.mods, site.gamma, site.beta, relu=True)
    elif path == "residual":
        y = site.norm(x, site.mods, site.gamma, site.beta, True, residual=r)
    else:
        down = sites[1]
        y = site.norm.forward_with_downsample(x, site.mods, site.gamma, site.beta, xd, down.norm, down.mods, down.gamma,
                                              down.beta)
    fn = y.grad_fn
    saved = fn.saved_tensors
    if path == "tail2":
        assert type(fn).__name__.startswith("_TailPairFunction")
        mask, stats = saved[2], [(saved[3], saved[4]), (saved[6], saved[7])]
    else:
        assert fn.cfg[3] & _native.LAYOUT_NHWC, "the channels-last kernels did not run"
        mask, stats = (saved[5] if path == "residual" else None), [(saved[1], saved[2])]
    del saved, fn
    assert y.is_contiguous(memory_format=CL)
    if fork:                                         # loss = <u, w1> + <v, w2>: the two gradients reach the kernels apart
        u, v = dwt_b200.fork_for_sum(y)
        torch.autograd.backward([u, v], [w1, w2])
        del u, v
    else:
        y.backward(w1)
    out = y.detach()
    del y
    status = _native.status(dev)
    active = out > 0
    if mask is not None:
        relu_mask = _decode(mask, shape)
        assert torch.equal(relu_mask, active), "byte map != the kernel's own out > 0"
        del active
    else:
        relu_mask = active

    # ---- fp64 reference, one domain at a time
    err = {}

    def add(key, got, ref):
        err.setdefault(key, _Err()).add(got, ref)
    flips, far = 0, 0.0            # far: the flipped element farthest from zero, in units of max |pre-activation|
    for di in range(d):
        sl = slice(di * n, (di + 1) * n)
        x64 = _f64(x[sl]).requires_grad_(True)
        pre = site.ref[di](x64) * site.g64 + site.b64
        if path == "residual":
            r64 = _f64(r[sl]).requires_grad_(True)
            pre = pre + r64
        elif path == "tail2":
            xd64 = _f64(xd[sl]).requires_grad_(True)
            pre = pre + (sites[1].ref[di](xd64) * sites[1].g64 + sites[1].b64)
        with torch.no_grad():
            p, m = pre.detach(), relu_mask[sl]
            flip = m != (p > 0)
            nflip = int(flip.sum())
            if nflip:
                far = max(far, p[flip].abs().max().item() / p.abs().max().item())
            flips += nflip
            add("out", out[sl], p.clamp_min(0))
            seed_grad = _f64(w1[sl])
            if fork:
                seed_grad += _f64(w2[sl])
            seed_grad.mul_(m)
            del p, m, flip
        (pre * seed_grad).sum().backward()
        del pre, seed_grad
        add("dx", x.grad[sl], x64.grad)
        if path == "residual":
            add("d_identity", r.grad[sl], r64.grad)
            del r64
        inputs = [x64]
        if path == "tail2":
            add("dxd", xd.grad[sl], xd64.grad)
            inputs.append(xd64)
        with torch.no_grad():
            for k, (s, inp, (save_mean, save_w)) in enumerate(zip(sites, inputs, stats)):
                mu, cov = s.batch_stats(inp.detach())
                add(f"mean{'_d' * k}", save_mean[di], mu)
                add(f"cov{'_d' * k}", s.kernel_cov(save_w[di]), cov)
        del x64, inputs
        if path == "tail2":
            del xd64
    for k, s in enumerate(sites):
        sfx = "_d" * k
        add("dgamma" + sfx, s.gamma.grad, s.g64.grad)
        add("dbeta" + sfx, s.beta.grad, s.b64.grad)
        for o in s.buf32:
            add("running_mean" + sfx, s.buf32[o][0], s.buf64[o][0])
            add("running_var" + sfx, s.buf32[o][1], s.buf64[o][1])
        if kind == "bn":
            assert [int(m.num_batches_tracked) for m in s.mods] == [int(m.num_batches_tracked) for m in s.ref] == [3] * d

    res = {k: e.both() for k, e in err.items()}
    print(label, size, "flips", flips, "%.1e" % far, {k: "%.1e %.1e" % v for k, v in res.items()})
    table = worst.setdefault((path, size), {})
    for k, (rel, mx) in res.items():
        cls = "stats" if k.startswith(STAT_KEYS) else "values"
        old = table.get(cls, (0.0, 0.0))
        table[cls] = (max(old[0], rel), max(old[1], mx))
    assert status == 0, status
    assert far <= 1e-5, ("the ReLU mask differs from the fp64 sign away from zero", far)
    # the flips are elements within the output's rounding of zero: 10 per million elements covers |mean| = 50 sigma,
    # whose fp32 mean alone is off by up to 3e-5 sigma (773 flips in 154M elements)
    assert flips <= max(4, out.numel() // 10 ** 5), flips
    for k, (rel, mx) in res.items():
        loose = kind == "whiten" and not k.startswith(STAT_KEYS)   # through a Cholesky factor
        assert rel < (TOL if loose else TOL_STAT), (label, k, rel, mx)
        assert mx < (TOL_MAX if loose else 5 * TOL_STAT), (label, k, rel, mx)
    return res


# --------------------------------------------------------------------------- every site of the training step
@pytest.fixture(scope="module")
def model_sites(dev):
    """(kind, C, H, W, gs, path, relu, forked) of every DomainTripleNorm call of one channels-last fused training forward
    of the harness ResNet-50-DWT at 224^2 (one image per domain), in call order, duplicates removed.  Recorded at the
    functional entry points, so the path is the one the model took; forked = the output went through fork_for_sum."""
    import dwt_b200
    from dwt_b200 import functional as F
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    calls, forked = [], []
    norm, tail_pair, fork = F.norm, F.tail_pair, dwt_b200.fork_for_sum

    def rec_norm(x, *args, **kw):
        y = norm(x, *args, **kw)
        calls.append(((kw["kind"], x.shape[1], x.shape[2], x.shape[3], kw["group_size"],
                       "plain" if kw.get("residual") is None else "residual", bool(kw.get("relu"))), x, y))
        return y

    def rec_tail_pair(x, xd, *args, **kw):
        y = tail_pair(x, xd, *args, **kw)
        calls.append(((kw["kind"], x.shape[1], x.shape[2], x.shape[3], kw["group_size"], "tail2", True), x, y))
        return y

    def rec_fork(y):
        forked.append(y)
        return fork(y)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(F, "norm", rec_norm)
        mp.setattr(F, "tail_pair", rec_tail_pair)
        mp.setattr(dwt_b200, "fork_for_sum", rec_fork)          # the Bottlenecks take it at construction
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        model = build_resnet50_dwt(sd, dwt_b200, site_mode="fused", channels_last=True).to(dev).train()
        images, _ = synth_batch(seed=2, per_domain=1, size=224)
        model(images.to(dev).contiguous(memory_format=CL))
    sites = []
    for key, x, y in calls:
        assert x.shape[0] == 3 and x.is_contiguous(memory_format=CL) and not x.is_contiguous(), key
        entry = key + (any(f is y for f in forked),)
        if entry not in sites:
            sites.append(entry)
    return sites


def test_every_model_site_geometry(model_sites, dev, worst):
    """Each distinct site of the training step (stem 64@112^2 down to the 2048@7^2 tails) at 2 images per domain."""
    assert {s[5] for s in model_sites} == {"plain", "residual", "tail2"}, model_sites
    assert model_sites[0] == ("whiten", 64, 112, 112, 4, "plain", True, False), model_sites[0]      # the stem
    assert ("bn", 2048, 7, 7, 1, "residual", True, False) in model_sites                              # the last block
    print(len(model_sites), "distinct sites:", model_sites)
    failures = []
    for i, (kind, c, h, w, gs, path, relu, fork) in enumerate(model_sites):
        assert relu
        label = f"{kind} {c}@{h}x{w} gs{gs} {path}{' forked' if fork else ''}"
        try:
            _check(dev, worst, label, "N=2", kind=kind, c=c, gs=gs, d=3, n=2, h=h, w=w, path=path, fork=fork, seed=100 + i)
        except AssertionError as e:
            failures.append(f"{label}: {e}")
    assert not failures, "\n".join(failures)


# --------------------------------------------------------------------------- launch edges
EDGES = [   # C, path, kind, gs, domains, rows per domain, forked, running buffers (site, downsample site)
    (4, "plain", "whiten", 4, 3, "lt_rpi", False, ("shared", None)),
    (4, "residual", "whiten", 2, 1, "lt8", True, ("shared", None)),
    (4, "tail2", "bn", 1, 4, "ragged", True, ("distinct", "shared")),
    (8, "plain", "bn", 1, 2, "ragged", False, ("distinct", None)),
    (8, "residual", "whiten", 4, 4, "chunk", False, ("mixed", None)),
    (8, "tail2", "whiten", 2, 3, "lt_rpi", True, ("mixed", "distinct")),
    (16, "plain", "whiten", 2, 1, "chunk+1", False, ("shared", None)),
    (16, "residual", "bn", 1, 3, "ragged", True, ("shared", None)),
    (16, "tail2", "whiten", 4, 2, "chunk", False, ("distinct", "shared")),
    (1024, "plain", "bn", 1, 4, "chunk", False, ("shared", None)),
    (1024, "residual", "whiten", 4, 3, "ragged", True, ("shared", None)),
    (1024, "tail2", "whiten", 2, 1, "lt8", True, ("shared", "shared")),
    (2048, "plain", "whiten", 4, 3, "chunk+1", False, ("shared", None)),
    (2048, "residual", "bn", 1, 2, "lt8", True, ("distinct", None)),
    (2048, "tail2", "bn", 1, 3, "ragged", True, ("shared", "mixed")),
    (4096, "plain", "whiten", 2, 3, "ragged", False, ("mixed", None)),
    (4096, "residual", "whiten", 4, 1, "chunk+1", True, ("shared", None)),
    (4096, "tail2", "bn", 1, 4, "chunk+1", True, ("mixed", "distinct")),
]


@pytest.mark.parametrize("c,path,kind,gs,d,rows,fork,layouts", EDGES,
                         ids=[f"c{e[0]}-{e[1]}-{e[2]}-gs{e[3]}-d{e[4]}-{e[5]}{'-forked' if e[6] else ''}" for e in EDGES])
def test_launch_edges(c, path, kind, gs, d, rows, fork, layouts, dev, worst):
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    m = _edge_rows(rows, c, d, sms)
    n, h, w = (1, 2, 2) if m == 4 else (1, 3, 3) if m == 9 else (1, 1, m)
    _check(dev, worst, f"c{c} {path} {kind} gs{gs} d{d} {rows}={m} rows", "edges", kind=kind, c=c, gs=gs, d=d, n=n,
           h=h, w=w, path=path, fork=fork, layouts=layouts, seed=c + d)


# --------------------------------------------------------------------------- the benchmark's size: capped grid
def _bench_case(dev, worst, label, **kw):
    _check(dev, worst, label, "3x64", d=3, n=BENCH_PER_DOMAIN, **kw)
    peak = torch.cuda.max_memory_allocated(dev)
    assert peak < 20 * GIB, f"peak device memory {peak / GIB:.1f} GiB"


@pytest.mark.parametrize("name", ["stem", "layer1.0-tail2", "layer4-residual"])
def test_bench_size_sites(name, dev, worst):
    """3 x 64 images per call: grid.x capped at 3 x SMs / (grid.y x D) CTAs, hundreds of rows summed per thread in fp32,
    and a finalize that adds one partial row per CTA -- more than a warp's 32 lanes each take once."""
    kw = {"stem": dict(kind="whiten", c=64, gs=4, h=112, w=112, path="plain", fork=False),
          "layer1.0-tail2": dict(kind="whiten", c=256, gs=4, h=56, w=56, path="tail2", fork=True),
          "layer4-residual": dict(kind="bn", c=2048, gs=1, h=7, w=7, path="residual", fork=True)}[name]
    _bench_case(dev, worst, name, seed=7, **kw)


def _large_mean(gen, shape, d, dev):
    """|mean| >= 50 sigma in every channel (the channels-last twin of test_whitening_large_mean_is_stable)."""
    x = _activation(gen, shape, d, dev).mul_(0.1).add_(10.0)
    return x.add_(torch.linspace(0.0, 40.0, shape[1], device=dev).view(1, -1, 1, 1))


def _top_row_offset(gen, shape, d, dev):
    """The first image of every domain has its top row 30 sigma off the rest of the domain: the rows an estimate of the
    mean taken from the first pixels of the domain would see."""
    x = _activation(gen, shape, d, dev)
    n = shape[0] // d
    for k in range(d):
        sigma = x[k * n:(k + 1) * n].std(dim=(0, 2, 3))
        x[k * n, :, 0, :] += 30.0 * sigma.view(-1, 1)
    return x


@pytest.mark.parametrize("make_x", [_large_mean, _top_row_offset], ids=["mean_50sigma", "top_row_30sigma"])
def test_pilot_shift_at_bench_size(make_x, dev, worst):
    """One-pass moments around a pilot shift K lose (K - mean)^2 / sigma^2 of fp32's digits: K must land near the
    domain's mean whatever the first pixels hold.  Stem site geometry at the benchmark's size."""
    _bench_case(dev, worst, make_x.__name__, kind="whiten", c=64, gs=4, h=112, w=112, path="plain", fork=False, seed=11,
                make_x=make_x)
