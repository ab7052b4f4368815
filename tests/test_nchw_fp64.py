"""The NCHW norm kernels -- small (group sizes 1 / 2 / 4, every batch norm), tiled (other group sizes, and shapes the
tensor-core kernels cannot take) and tensor-core (group sizes 8..64) -- against an fp64 reference on the GPU.

Reference: oracle/torch_port.py's WTransform2d / BatchNorm1d / 2d / 3d in float64 (the reference's operator sequence,
pinned to the reference's own outputs by test_oracle_vs_golden.py), composed as the reference composes a site: the D
domain modules called in order on the site's running buffers (shared, distinct or mixed, aliased like the kernels'
buffers, so the EMA runs source -> target -> ...), then * gamma + beta, + identity, ReLU where the site has them.
Groups never cross a slab of channels, so the reference runs one domain and one slab of channels at a time and its fp64
autograd graph stays a few GiB even at the full microbench size (N=256 C=256 56^2).  The ReLU derivative is taken where
the kernel put it (its out > 0, as a constant); the two masks may disagree only on elements within rounding of zero.

Compared for every case, norm-wise with the max-elementwise error beside it: the output, dx, d_identity, dgamma / dbeta
where there is an epilogue, each domain's batch mean and covariance (recovered from the saved W; in eval mode the
running statistics the kernel factored instead), every running buffer, num_batches_tracked for batch norm, and the
status word.  Each case also asserts which kernel family ran (small_* / tiled_* / tc_* in the launch profile): a case
that silently takes another path fails.

Cases (sizes derived from the kernels' constants and the SM count, so the edges move with the code):
  * the microbench at full size, input built as bench.py's run_microbench builds it, gs 64 / 32 / 8 (tensor cores) and
    4 (small): train forward + backward and the EMA;
  * tensor-core routing edges: N*HW on either side of 4096, HW = 32 / 36 / 28, a partial 64-pixel apply tile, partial
    64-channel super-blocks, fewer tiles than CTAs, more problems than 2 x SMs, a contiguous input at a 4-byte storage
    offset (routes to the tiled kernels);
  * 1 to 4 domains with shared / distinct / mixed buffers, train / no-grad train / eval (module and DomainTripleNorm) /
    default-constructed buffers, on the tiled and the tensor-core kernels;
  * tiled edges: gs 3 / 5 / 6 / 12 / 24 / 48 / 64 with float4 and scalar loads, one tile, 128 and 129 samples, a grid
    capped at one wave with 7x7 images;
  * small-path edges: gs 1 / 2 / 4 with float4 and scalar loads, 2 / 4 / 8 (the cap) problems per CTA, the AFFINE /
    RELU / RESIDUAL epilogues, BatchNorm1d (HW = 1) and BatchNorm3d, the ResNet stem site at 3 x 64 images;
  * pilot-shift robustness at the microbench shape, the stem size and a BatchNorm1d batch of 256: a first image whose
    pilot window (the mid-image pixels the shift K is estimated from) sits 30 sigma off, and |mean| = 50 sigma.

Tolerances as in test_gpu_parity_r2.py: 1e-3 norm-wise through a Cholesky factor, 1e-4 on batch norm and on statistics;
max-elementwise (scaled by max |reference|) below 5x the norm-wise bound.
"""
import contextlib
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-3
TOL_STAT = 1e-4
TOL_MAX = 5e-3
GIB = 1 << 30
STAT_KEYS = ("mean", "cov", "running")
FAMILIES = ("small", "tiled", "tc")
# routing and launch shaping of the NCHW kernels (norm_tc.cu tc_supports, api.cu make_plan / shape)
TC_CH = 64                  # channels of a tensor-core super-block
TC_BOX = 32                 # pixels of a TMA box: HW >= TC_BOX
TC_MIN_M = 4096             # N * HW below this takes the (exact fp32) tiled kernels
TC_APPLY_PX = 64            # pixels of a tensor-core apply tile
TC_CTAS_PER_SM = 2          # tc_chunks: 2 * SMs CTAs over the (domain, super-block) problems
TILED_TP = 128              # samples per tile of the tiled kernels
TILED_SLOTS = 2             # CTAs per SM of a tiled reduction
SMALL_SLOTS = {1: 4, 2: 4, 4: 3}    # CTAs per SM of small_stats (slots_per_sm)
PILOT_PX = 32               # the NCHW pilot window: <= 32 mid-image pixels of image 0
SLAB_ELEMS = 1 << 25        # fp64 reference: elements of one (domain, channel slab) call
NBT0 = 2                    # batch norm: num_batches_tracked before the call (momentum=None: EMA factor 1/3)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


@pytest.fixture(scope="module")
def worst(dev):
    """Worst (norm-wise, max-elementwise) error per (family, case group), printed with the peak device memory at the end."""
    torch.cuda.reset_peak_memory_stats(dev)
    table = {}
    yield table
    print("\nworst errors (norm-wise, max-elementwise):")
    for key in sorted(table):
        print("  %-20s %s" % (" / ".join(key), ", ".join(f"{k} {r:.1e} {m:.1e}" for k, (r, m) in sorted(table[key].items()))))
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


def _bcast(v, dim):
    """[C] -> [1, C, 1, ...] against a tensor of `dim` dimensions."""
    return v.view(1, -1, *([1] * (dim - 2)))


def _red_dims(t):
    return [0] + list(range(2, t.dim()))


def _f64(t):
    return t.detach().to(torch.float64, memory_format=torch.contiguous_format)


# --------------------------------------------------------------------------- inputs
def _activation(gen, shape, d, dev):
    """Neighbouring channels correlated (inside whitening groups too), per-channel scales, a different mean per domain."""
    z = torch.randn(shape, device=dev, generator=gen)
    z.add_(z.roll(1, 1), alpha=0.6)
    z.mul_(_bcast(0.5 + torch.rand(shape[1], device=dev, generator=gen), z.dim()))
    n = shape[0] // d
    for k in range(d):
        z[k * n:(k + 1) * n].add_(0.6 * k - 0.5)
    return z


def _microbench(gen, shape, d, dev):
    """bench.py's run_microbench input: seed 0, x = mix . randn + 2.0 (BASELINE.json configs[1])."""
    n, c, h, w = shape
    torch.manual_seed(0)
    mix = torch.randn(c, c, device=dev) / c ** 0.5 + torch.eye(c, device=dev)
    return (torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, h, w, device=dev)) + 2.0).contiguous()


def _pilot_window(base):
    """base's input with image 0 of every domain 30 sigma off in the pilot window -- the <= 32 mid-image pixels the NCHW
    statistics kernels estimate their shift K from (a BatchNorm1d batch: its first sample)."""
    def make(gen, shape, d, dev):
        x = base(gen, shape, d, dev)
        n, hw = shape[0] // d, x[0, 0].numel()
        npx = min(hw, PILOT_PX)
        p0 = ((hw - npx) // 2) & ~3
        flat = x.view(shape[0], shape[1], hw)
        for k in range(d):
            sigma = x[k * n:(k + 1) * n].std(dim=_red_dims(x))
            flat[k * n, :, p0:p0 + npx] += 30.0 * sigma.view(-1, 1)
        return x
    make.__name__ = "pilot_30sigma"
    return make


def _mean_50sigma(base):
    """|mean| >= 50 sigma in every channel (the NCHW twin of test_whitening_large_mean_is_stable): the control input."""
    def make(gen, shape, d, dev):
        x = base(gen, shape, d, dev).mul_(0.1).add_(10.0)
        return x.add_(_bcast(torch.linspace(0.0, 40.0, shape[1], device=dev), x.dim()))
    make.__name__ = "mean_50sigma"
    return make


# --------------------------------------------------------------------------- one site, twice
class _Site:
    """One norm site on the CUDA modules (dwt_b200, fp32) and the buffers of its fp64 reference, with the same initial
    running buffers aliased alike: 'shared' (one pair, as in the model), 'distinct', 'mixed' or 'default'
    (default-constructed whitening modules, one pair each)."""

    def __init__(self, kind, c, gs, d, rank, layout, gen, dev):
        import dwt_b200
        self.kind, self.c, self.gs, self.rank = kind, c, gs, rank
        self.owner = {"shared": [0] * d, "distinct": list(range(d)), "mixed": [0] + [1] * (d - 1),
                      "default": list(range(d))}[layout]
        assert layout != "mixed" or d >= 3
        assert layout != "default" or kind == "whiten"
        bn_cls = {2: dwt_b200.BatchNorm1d, 3: dwt_b200.BatchNorm1d, 4: dwt_b200.BatchNorm2d, 5: dwt_b200.BatchNorm3d}
        own = {}
        for o in sorted(set(self.owner)):
            if layout == "default":
                own[o] = dwt_b200.WTransform2d(c, gs).to(dev)
                continue
            rm = 0.1 * torch.randn(c, device=dev, generator=gen)
            if kind == "whiten":
                a = torch.randn(c // gs, gs, gs, device=dev, generator=gen)
                own[o] = (rm.view(1, c, 1, 1), a @ a.transpose(1, 2) / gs + 0.5 * torch.eye(gs, device=dev))
            else:
                own[o] = (rm, 0.5 + torch.rand(c, device=dev, generator=gen))
        self.mods = []
        for o in self.owner:
            if layout == "default":
                m = own[o]
            elif kind == "whiten":
                m = dwt_b200.WTransform2d(c, gs, running_m=own[o][0], running_var=own[o][1])
            else:
                m = bn_cls[rank](c, *own[o], affine=False, momentum=None)
                m.num_batches_tracked.fill_(NBT0)
            self.mods.append(m)
        second = "running_variance" if kind == "whiten" else "running_var"
        self.buf32 = {o: (self.mods[self.owner.index(o)].running_mean, getattr(self.mods[self.owner.index(o)], second))
                      for o in own}
        self.buf64 = {o: (a.double(), b.double()) for o, (a, b) in self.buf32.items()}
        self.eps = self.mods[0].eps
        self.norm = dwt_b200.DomainTripleNorm(kind, c, gs, n_domains=d)

    def ref(self, di, c0, c1, training):
        """The fp64 reference module of domain di on channels [c0, c1): views into the reference's running buffers."""
        import oracle.torch_port as port
        rm, rv = self.buf64[self.owner[di]]
        if self.kind == "whiten":
            m = port.WTransform2d(c1 - c0, self.gs, running_m=rm[:, c0:c1], running_var=rv[c0 // self.gs:c1 // self.gs])
        else:
            cls = {2: port.BatchNorm1d, 3: port.BatchNorm1d, 4: port.BatchNorm2d, 5: port.BatchNorm3d}[self.rank]
            m = cls(c1 - c0, rm[c0:c1], rv[c0:c1], affine=False, momentum=None)
            m.num_batches_tracked.fill_(NBT0)
        return m.train(training)

    def stats(self, x64, di, c0, c1, training):
        """What the kernel factored for domain di, channels [c0, c1): the fp64 batch mean and (biased) covariance /
        variance in training, the running mean and second moment in eval."""
        if not training:
            rm, rv = self.buf64[self.owner[di]]
            return rm.reshape(-1)[c0:c1], rv[c0 // self.gs:c1 // self.gs] if self.kind == "whiten" else rv[c0:c1]
        mu = x64.mean(dim=_red_dims(x64))
        xc = x64 - _bcast(mu, x64.dim())
        if self.kind == "bn":
            return mu, xc.square().mean(dim=_red_dims(xc))
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


@contextlib.contextmanager
def _record_saved_stats(records):
    """Collect (save_mean, save_w) of every norm call, also under no_grad (where autograd keeps nothing)."""
    from dwt_b200 import functional as F
    fwd = F._NormFunction.forward

    def rec(ctx, *args):
        y = fwd(ctx, *args)
        records.append(tuple(t.detach() for t in ctx.to_save[1:3]))
        return y
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(F._NormFunction, "forward", staticmethod(rec))
        yield


def _check(dev, worst, label, group, *, kind, c, gs, d, n, spatial, family, mode="train", layout="shared", via="site",
           epi="relu", make_x=None, offset=0, seed=0):
    """Run one site on the NCHW kernels and on the fp64 reference; assert every comparison and the kernel family.

    mode: train (forward + backward) | nograd (train-mode forward under no_grad) | eval (forward + backward on the
    running statistics); via: site (DomainTripleNorm over d domains) | module (the layer module itself, d = 1);
    epi: None | affine | relu | residual (site only); offset: the input starts `offset` floats into its storage."""
    from dwt_b200 import _native
    assert via == "site" or (d == 1 and epi is None)
    gen = torch.Generator(device=dev).manual_seed(seed)
    shape = (d * n, c, *spatial)
    grad, training = mode != "nograd", mode != "eval"
    x = (make_x or _activation)(gen, shape, d, dev)
    if offset:                                   # contiguous, but not 16-byte aligned: the scalar-load kernels
        store = torch.empty(x.numel() + offset, device=dev)
        store[offset:].copy_(x.reshape(-1))
        x = store[offset:].view(shape)
        del store
    assert x.is_contiguous() and (x.data_ptr() % 16 != 0) == bool(offset % 4)
    x.requires_grad_(grad)
    r = _activation(gen, shape, d, dev).requires_grad_(grad) if epi == "residual" else None
    w1 = torch.randn(shape, device=dev, generator=gen) if grad else None
    site = _Site(kind, c, gs, d, len(shape), layout, gen, dev)
    affine, relu = epi is not None, epi in ("relu", "residual")
    gamma = (0.5 + torch.rand(c, device=dev, generator=gen)).view(c, *([1] * len(spatial))).requires_grad_(grad)
    beta = (0.3 * torch.randn(c, device=dev, generator=gen)).view(c, *([1] * len(spatial))).requires_grad_(grad)
    g64, b64 = _f64(gamma).requires_grad_(grad), _f64(beta).requires_grad_(grad)
    for m in site.mods:
        m.train(training)

    # ---- CUDA
    records = []
    _native.clear_status(dev)
    with _record_saved_stats(records):
        _native.profile_begin()
        try:
            with torch.set_grad_enabled(grad):
                if via == "module":
                    y = site.mods[0](x)
                else:
                    y = site.norm(x, site.mods, gamma if affine else None, beta if affine else None, relu=relu, residual=r)
            if grad:
                y.backward(w1)
        finally:
            prof = _native.by_family(_native.profile_end())
    out = y.detach()
    del y
    status = _native.status(dev)
    ran = {f for f in FAMILIES if any(k.startswith(f + "_") for k in prof)}
    assert ran == {family}, (label, family, sorted(prof))
    assert len(records) == 1, len(records)
    save_mean, save_w = records[0]

    # ---- fp64 reference, one domain and one slab of channels at a time
    err = {}

    def add(key, got, ref):
        err.setdefault(key, _Err()).add(got, ref)
    per_ch = n * out[0, 0].numel()
    slab = max(gs, SLAB_ELEMS // per_ch // gs * gs)
    # far: |pre-activation| of the flipped element farthest from zero; agree: the largest output error where the masks
    # agree; pmax: max |pre-activation|
    flips, far, agree, pmax = 0, 0.0, 0.0, 0.0
    for di in range(d):
        sl = slice(di * n, (di + 1) * n)
        for c0 in range(0, c, slab):
            c1 = min(c, c0 + slab)
            cs, gsl = slice(c0, c1), slice(c0 // gs, c1 // gs)
            x64 = _f64(x[sl, cs]).requires_grad_(grad)
            with torch.set_grad_enabled(grad):
                pre = site.ref(di, c0, c1, training)(x64)
                if affine:
                    pre = pre * g64[cs] + b64[cs]
                if r is not None:
                    r64 = _f64(r[sl, cs]).requires_grad_(True)
                    pre = pre + r64
            with torch.no_grad():
                p = pre.detach()
                if relu:
                    m = out[sl, cs] > 0
                    flip = m != (p > 0)
                    nflip = int(flip.sum())
                    if nflip:
                        far = max(far, p[flip].abs().max().item())
                    flips += nflip
                    pmax = max(pmax, p.abs().max().item())
                    p = p.clamp_min(0)
                    agree = max(agree, (out[sl, cs].double() - p).abs().masked_fill_(flip, 0.0).max().item())
                    del flip
                add("out", out[sl, cs], p)
                del p
            if grad:
                seed_grad = _f64(w1[sl, cs])
                if relu:
                    seed_grad.mul_(m)
                (pre * seed_grad).sum().backward()
                del seed_grad
                add("dx", x.grad[sl, cs], x64.grad)
                if r is not None:
                    add("d_identity", r.grad[sl, cs], r64.grad)
                    del r64
            del pre
            with torch.no_grad():
                mu, cov = site.stats(x64.detach(), di, c0, c1, training)
                add("mean", save_mean[di, cs], mu)
                add("cov", site.kernel_cov(save_w[di, gsl] if kind == "whiten" else save_w[di, cs]), cov)
            del x64
    if grad and affine:
        add("dgamma", gamma.grad, g64.grad)
        add("dbeta", beta.grad, b64.grad)
    for o in site.buf32:
        add("running_mean", site.buf32[o][0], site.buf64[o][0])
        add("running_var", site.buf32[o][1], site.buf64[o][1])
    if kind == "bn":
        assert [int(m.num_batches_tracked) for m in site.mods] == [NBT0 + training] * d

    res = {k: e.both() for k, e in err.items()}
    far, agree = far / max(pmax, 1e-30), agree / max(pmax, 1e-30)
    print(label, "flips", flips, "%.1e %.1e" % (far, agree), {k: "%.1e %.1e" % v for k, v in res.items()})
    table = worst.setdefault((family, group), {})
    for k, (rel, mx) in res.items():
        cls = "stats" if k.startswith(STAT_KEYS) else "values"
        old = table.get(cls, (0.0, 0.0))
        table[cls] = (max(old[0], rel), max(old[1], mx))
    assert status == 0, status
    # a flipped element lies within rounding of zero: within 1e-5 of max |pre-activation|, or within twice the error the
    # kernel makes where the masks agree (at |mean| = 50 sigma the fp32 centring alone is off by ~1e-5 of the output)
    assert far <= max(1e-5, 2 * agree), ("the ReLU mask differs from the fp64 sign away from zero", far, agree)
    assert flips <= max(4, out.numel() // 10 ** 5), flips
    for k, (rel, mx) in res.items():
        loose = kind == "whiten" and not k.startswith(STAT_KEYS)   # through a Cholesky factor
        assert rel < (TOL if loose else TOL_STAT), (label, k, rel, mx)
        assert mx < (TOL_MAX if loose else 5 * TOL_STAT), (label, k, rel, mx)
    peak = torch.cuda.max_memory_allocated(dev)
    assert peak < 16 * GIB, f"peak device memory {peak / GIB:.1f} GiB"
    return res


# --------------------------------------------------------------------------- 1. the microbench at full size
MICRO = dict(kind="whiten", c=256, d=1, n=256, spatial=(56, 56), via="module", layout="default", epi=None)


@pytest.mark.parametrize("gs,family", [(64, "tc"), (32, "tc"), (8, "tc"), (4, "small")], ids=lambda v: str(v))
def test_microbench_full_size(gs, family, dev, worst):
    """BASELINE.json configs[1] (bench.py --workload microbench): N=256 C=256 56^2, M = 802,816 samples per channel, on
    default-constructed buffers like the benchmark's module; train forward + backward and the EMA."""
    _check(dev, worst, f"microbench gs{gs}", "microbench", gs=gs, family=family, make_x=_microbench, **MICRO)


# --------------------------------------------------------------------------- 2. tensor-core routing edges
def _tc_edges(sms):
    """(label, C, gs, D, N, (H, W), family, storage offset in floats)."""
    hw44 = (4, 11)                                          # 44 pixels: 4092 = 93 x 44 samples
    tiles_n = sms // 4                                      # 128-pixel images: 4 tiles each, fewer than 2 x SMs CTAs
    big_c = TC_CH * 2 ** math.ceil(math.log2(sms + 1))      # > SMs super-blocks: x 2 domains > 2 x SMs problems
    return [
        ("m4096", 64, 16, 1, TC_MIN_M // 32, (4, 8), "tc", 0),
        ("m4092", 64, 16, 1, (TC_MIN_M - 4) // 44, hw44, "tiled", 0),
        ("hw32_one_box", 64, 32, 2, 160, (4, 8), "tc", 0),
        ("hw36_partial_box", 64, 64, 1, 120, (6, 6), "tc", 0),
        ("hw28", 64, 16, 1, 160, (4, 7), "tiled", 0),
        ("hw80_partial_apply_tile", 128, 64, 2, 60, (8, 10), "tc", 0),
        ("c40_gs8", 40, 8, 1, 20, (16, 16), "tc", 0),
        ("c80_gs16", 80, 16, 3, 20, (16, 16), "tc", 0),
        ("c96_gs32", 96, 32, 2, 20, (16, 16), "tc", 0),
        ("c200_gs8", 200, 8, 1, 20, (16, 16), "tc", 0),
        ("few_tiles", 64, 64, 1, tiles_n, (8, 16), "tc", 0),
        ("problems_gt_2sms", big_c, 64, 2, 2, (32, 64), "tc", 0),
        ("offset4B", 128, 64, 2, 16, (32, 32), "tiled", 1),
    ]


@pytest.mark.parametrize("case", range(13), ids=[e[0] for e in _tc_edges(132)])
def test_tensor_core_routing_edges(case, dev, sms, worst):
    label, c, gs, d, n, hw, family, offset = _tc_edges(sms)[case]
    m = n * hw[0] * hw[1]
    if label.startswith("m40"):
        assert (m >= TC_MIN_M) == (family == "tc") and TC_MIN_M - 4 <= m <= TC_MIN_M, m
    if label == "few_tiles":
        assert m >= TC_MIN_M and n * (hw[0] * hw[1] // TC_BOX) < TC_CTAS_PER_SM * sms
    if label == "problems_gt_2sms":
        assert (c // TC_CH) * d > TC_CTAS_PER_SM * sms
    _check(dev, worst, label, "tc_edges", kind="whiten", c=c, gs=gs, d=d, n=n, spatial=hw, family=family,
           layout="mixed" if d >= 3 else "distinct" if d == 2 else "shared", epi="relu", offset=offset, seed=c + d + n)


# --------------------------------------------------------------------------- 3. modes and domains
MODES = [   # domains, running buffers, mode, via
    (1, "shared", "train", "module"), (2, "distinct", "train", "site"), (3, "mixed", "train", "site"),
    (4, "shared", "train", "site"), (4, "mixed", "nograd", "site"), (3, "distinct", "nograd", "site"),
    (1, "shared", "eval", "module"), (3, "mixed", "eval", "site"), (2, "shared", "eval", "site"),
    (1, "default", "train", "module"), (3, "default", "nograd", "site"),
]


@pytest.mark.parametrize("family", ["tc", "tiled"])
@pytest.mark.parametrize("d,layout,mode,via", MODES, ids=[f"d{m[0]}-{m[1]}-{m[2]}-{m[3]}" for m in MODES])
def test_modes_and_domains(family, d, layout, mode, via, dev, worst):
    """The gs >= 8 EMA (fwd_factor_kernel's domain loop, fwd_ema_block) with shared (closed form), distinct and mixed
    (ordered) running buffers, and every mode, on the tensor-core and the tiled kernels."""
    c, gs, n, hw = (128, 32, 8, (24, 24)) if family == "tc" else (96, 24, 6, (10, 10))
    _check(dev, worst, f"{family} d{d} {layout} {mode} {via}", "modes", kind="whiten", c=c, gs=gs, d=d, n=n, spatial=hw,
           family=family, mode=mode, layout=layout, via=via, epi=None if via == "module" else "affine", seed=d + len(mode))


# --------------------------------------------------------------------------- 4. tiled edges
def _tiled_edges(sms):
    """(label, C, gs, N, (H, W)); every case routes to the tiled kernels."""
    cap_n = TILED_SLOTS * sms * TILED_TP // 49 + 64       # more 128-sample tiles than the one-wave grid has CTAs
    edges = []
    for gs in (3, 5, 6, 12, 24, 48, 64):
        edges.append((f"gs{gs}_vec4", 2 * gs, gs, 12, (4, 4)))     # HW % 4 == 0 (HW < 32: tiled for gs 64 too)
        edges.append((f"gs{gs}_vec1", 2 * gs, gs, 10, (5, 5)))
    edges += [("m75_one_tile", 24, 12, 3, (5, 5)), ("m128", 16, 8, 8, (4, 4)), ("m129", 16, 8, 3, (1, 43)),
              ("capped_grid_7x7", 8, 8, cap_n, (7, 7))]
    return edges


@pytest.mark.parametrize("case", range(18), ids=[e[0] for e in _tiled_edges(132)])
def test_tiled_edges(case, dev, sms, worst):
    label, c, gs, n, hw = _tiled_edges(sms)[case]
    m = n * hw[0] * hw[1]
    if label == "capped_grid_7x7":
        assert -(-m // TILED_TP) > TILED_SLOTS * sms
    _check(dev, worst, label, "tiled_edges", kind="whiten", c=c, gs=gs, d=3, n=n, spatial=hw, family="tiled",
           layout="mixed", epi="residual" if case % 2 else "relu", seed=case)


# --------------------------------------------------------------------------- 5. small-path edges
def _ppc_channels(gs, d, ppc, sms):
    """Channels that put `ppc` problems in each CTA of small_stats (ppc = 8 is the cap: twice what it needs)."""
    target = SMALL_SLOTS[gs] * sms
    groups = (3 * ppc * target) // (4 * d) if ppc < 8 else (3 * 8 * target) // d
    return groups * gs


SMALL = [   # label, kind, gs, D, N, spatial, epilogue, via
    ("gs1_vec4", "bn", 1, 3, 4, (6, 6), "relu", "site"),
    ("gs1_vec1", "bn", 1, 3, 5, (5, 5), "affine", "site"),
    ("gs2_vec4", "whiten", 2, 3, 4, (4, 8), "residual", "site"),
    ("gs2_vec1", "whiten", 2, 2, 4, (3, 7), "relu", "site"),
    ("gs4_vec4", "whiten", 4, 4, 3, (8, 8), "affine", "site"),
    ("gs4_vec1", "whiten", 4, 3, 6, (5, 5), "residual", "site"),
    ("gs4_none", "whiten", 4, 1, 8, (6, 6), None, "module"),
    ("bn1d_hw1", "bn", 1, 1, 64, (), None, "module"),
    ("bn1d_len7", "bn", 1, 1, 16, (7,), None, "module"),
    ("bn3d", "bn", 1, 1, 4, (3, 5, 6), None, "module"),
]


@pytest.mark.parametrize("case", SMALL, ids=[s[0] for s in SMALL])
def test_small_path_edges(case, dev, worst):
    label, kind, gs, d, n, spatial, epi, via = case
    _check(dev, worst, label, "small_edges", kind=kind, c=48, gs=gs, d=d, n=n, spatial=spatial, family="small", epi=epi,
           via=via, layout="mixed" if d >= 3 else "distinct", seed=len(label) + gs)


@pytest.mark.parametrize("ppc,kind,gs", [(2, "bn", 1), (4, "whiten", 2), (8, "whiten", 4)], ids=["ppc2", "ppc4", "ppc8"])
def test_small_problems_per_cta(ppc, kind, gs, dev, sms, worst):
    """Thousands of tiny (domain, group) problems: 8 / ppc warps per problem, ppc problems per CTA, D = 3."""
    c = _ppc_channels(gs, 3, ppc, sms)
    target, groups = SMALL_SLOTS[gs] * sms, c // gs
    got = 1
    while got < 8 and -(-groups // got) * 3 > target:
        got *= 2
    assert got == ppc, (c, got)
    _check(dev, worst, f"ppc{ppc} c{c}", "small_edges", kind=kind, c=c, gs=gs, d=3, n=2, spatial=(7, 7), family="small",
           epi="residual", layout="mixed", seed=ppc)


def test_stem_site_at_bench_size(dev, worst):
    """The ResNet stem site on NCHW at the benchmark's size: 3 x 64 images, 64 x 112^2, gs 4, ReLU epilogue."""
    _check(dev, worst, "stem 3x64", "bench_size", kind="whiten", c=64, gs=4, d=3, n=64, spatial=(112, 112),
           family="small", epi="relu", seed=5)


# --------------------------------------------------------------------------- 6. pilot robustness
PILOT_SITES = {   # the microbench shape on the tensor-core and (misaligned input) tiled kernels, the stem size, BN1d
    "micro_tc": dict(kind="whiten", c=256, gs=64, d=1, n=256, spatial=(56, 56), family="tc", via="module", epi=None),
    "micro_tiled": dict(kind="whiten", c=256, gs=64, d=1, n=256, spatial=(56, 56), family="tiled", via="module", epi=None,
                        offset=1),
    "stem_small": dict(kind="whiten", c=64, gs=4, d=3, n=64, spatial=(112, 112), family="small", epi="relu"),
    "bn1d_256": dict(kind="bn", c=256, gs=1, d=1, n=256, spatial=(), family="small", via="module", epi=None),
}


@pytest.mark.parametrize("inp", ["pilot_30sigma", "mean_50sigma"])
@pytest.mark.parametrize("where", list(PILOT_SITES))
def test_pilot_shift(where, inp, dev, worst):
    """One-pass moments around a pilot shift K lose (K - mean)^2 / sigma^2 of fp32's digits: K must land near the
    domain's mean whatever image 0's mid pixels (a BatchNorm1d batch: its first sample) hold."""
    kw = dict(PILOT_SITES[where])
    base = _microbench if where.startswith("micro") else _activation
    make_x = (_pilot_window if inp == "pilot_30sigma" else _mean_50sigma)(base)
    _check(dev, worst, f"{where} {inp}", "pilot", make_x=make_x, seed=11, **kw)
