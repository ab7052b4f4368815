"""Eval, no-grad and statistics-collection (replicated) norm sites against an fp64 reference on the GPU.

Before it reports accuracy the reference runs train-mode forwards under no_grad that feed cat((d, d, d)) so that every
domain branch folds the target batch into its running buffers (resnet50_dwt_mec_officehome.py:380-389), then evaluates
through eval-mode modules.  Here that is DomainTripleNorm(replicated=True) and the eval-mode kernels: small_eval_prep
(each domain's own running buffers), the eval branch of bwd_finalize_thread (dgamma / dbeta, the masked residual
backward), small_bwd_prep (eval backward without an affine gradient) and the k-fold EMA per distinct buffer pair.

Reference: oracle/torch_port.py's WTransform2d / BatchNorm1d / 2d / 3d in float64 on fp64 copies of the running buffers,
aliased like the kernels' buffers (shared / distinct / mixed), composed as the reference composes a site: the D domain
modules called in order, then * gamma + beta, + identity, ReLU.  The replicated reference is three sequential module
calls on the same data; its output is the first call's.  Backward: fp64 autograd, with the ReLU derivative taken where
the kernel put it (its out > 0, or the channels-last residual tail's byte map, checked bit for bit against out > 0).

Compared for every case, norm-wise with the max-elementwise error beside it: the output, dx, d_identity, dgamma / dbeta,
the saved mean and the covariance recovered from the saved W (the batch's in training, the running statistics the
kernel factored in eval), every running buffer, num_batches_tracked and the status word.  In eval every running buffer
must be unchanged bit for bit.  Each case asserts from the launch profile which kernels ran.

Cases:
  * every site geometry of the channels-last fused ResNet-50-DWT at 2 images per domain, each in eval (dgamma / dbeta,
    frozen gamma / beta, the residual epilogue with its byte map and masked backward), no-grad train (bit for bit equal
    to a grad-enabled call, nothing saved) and replicated (shared / distinct / mixed buffers, batch norm with
    momentum=None from num_batches_tracked = 2, count_batches=False, the residual epilogue);
  * channels-last launch edges in eval with distinct per-domain buffers (C = 4, 8, 1024, 4096; D = 1..4);
  * the NCHW small family (gs 1 / 2 / 4, vec4 and scalar loads, every epilogue, D = 1..4, BatchNorm1d / 3d,
    track_running_stats=False) in eval, no-grad and replicated;
  * replicated on the tensor-core (NCHW gs 64, channels-last gs 32) and tiled (gs 12) kernels;
  * a running covariance of condition number 1e4, a non-positive-definite running covariance, and replicated eval;
  * the whole statistics-collection chain of the channels-last and the NCHW fused model against an fp64 port model.

Tolerances as in test_nchw_fp64.py: 1e-3 norm-wise through a Cholesky factor, 1e-4 on batch norm and on statistics;
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
CL = torch.channels_last
STAT_KEYS = ("mean", "cov", "running")
NBT0 = 2                    # batch norm: num_batches_tracked before the call (momentum=None: EMA factor 1/3)
# launch shape of the channels-last kernels (norm_cl.cu, cl_plan in api.cu)
THREADS = 256
STATS_UNROLL = 8
STATS_SLOTS = 3
# kernels of one forward / backward call, by family, as the launch profile names them (fp32)
FWD_TRAIN = {"small": {"small_stats", "small_apply"}, "cl": {"cl_stats", "cl_fwd_finalize", "cl_apply"},
             "tc": {"tc_stats", "dense_fwd_finalize", "tc_apply"},
             "tc_nhwc": {"tc_stats_nhwc", "dense_fwd_finalize", "tc_apply_nhwc"}, "tiled": {"tiled_stats", "tiled_apply"}}
FWD_EVAL = {"small": {"eval_prep", "small_apply"}, "cl": {"eval_prep", "cl_apply"}}
BWD_REDUCE = {"small": {"small_bwd_reduce", "small_bwd_apply"}, "cl": {"cl_bwd_reduce", "cl_bwd_finalize", "cl_bwd_apply"}}
BWD_PREP = {"small": {"bwd_prep", "small_bwd_apply"}, "cl": {"bwd_prep", "cl_bwd_apply"}}
APPLY = {"small": "small_apply", "cl": "cl_apply", "tc": "tc_apply", "tc_nhwc": "tc_apply_nhwc", "tiled": "tiled_apply"}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst(dev):
    """Worst (norm-wise, max-elementwise) error per (family, mode), printed with the peak device memory at the end."""
    torch.cuda.reset_peak_memory_stats(dev)
    table = {}
    yield table
    print("\nworst errors (norm-wise, max-elementwise):")
    for key in sorted(table):
        print("  %-26s %s" % (" / ".join(key), ", ".join(f"{k} {r:.1e} {m:.1e}" for k, (r, m) in sorted(table[key].items()))))
    print(f"peak device memory: {torch.cuda.max_memory_allocated(dev) / GIB:.2f} GiB")


class _Err:
    """||a - b|| / ||b|| and max|a - b| / max|b| accumulated over slices, in float64."""

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
    return v.view(1, -1, *([1] * (dim - 2)))


def _f64(t):
    return t.detach().to(torch.float64, memory_format=torch.contiguous_format)


def _activation(gen, shape, d, dev):
    """Neighbouring channels correlated (inside whitening groups too), per-channel scales, a different mean per domain."""
    z = torch.randn(shape, device=dev, generator=gen)
    z.add_(z.roll(1, 1), alpha=0.6)
    z.mul_(_bcast(0.5 + torch.rand(shape[1], device=dev, generator=gen), z.dim()))
    n = shape[0] // d
    for k in range(d):
        z[k * n:(k + 1) * n].add_(0.6 * k - 0.5)
    return z


def _decode(mask, shape):
    """The channels-last residual tail's byte map (bit i of byte q = channel 4q + i of the NHWC tensor) -> bool NCHW."""
    n, c, h, w = shape
    bits = torch.arange(4, device=mask.device, dtype=torch.uint8)
    b = (mask.view(n, h, w, c // 4, 1) >> bits) & 1
    return b.view(n, h, w, c).permute(0, 3, 1, 2).bool()


@contextlib.contextmanager
def _record_saved_stats(records):
    """Collect (save_mean, save_w) of every norm call, also under no_grad (where autograd keeps nothing)."""
    from dwt_b200 import functional as F
    fwd = F._NormFunction.forward

    def rec(ctx, *args):
        y = fwd(ctx, *args)
        records.append(tuple(t.detach().clone() for t in ctx.to_save[1:3]))
        return y
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(F._NormFunction, "forward", staticmethod(rec))
        yield


def _profiled(fn):
    from dwt_b200 import _native
    _native.profile_begin()
    try:
        out = fn()
    finally:
        prof = _native.by_family(_native.profile_end())
    return out, prof


# --------------------------------------------------------------------------- one site, twice
class _Site:
    """One norm site: the CUDA modules (fp32) and the fp64 reference modules, with the same initial running buffers
    aliased alike ('shared', 'distinct', 'mixed').  cond: the running covariances of every group have condition number
    1e4 (eigenvalues 1e2 .. 1e-2) instead of a a^T / gs + 0.5 I.  track=False: modules that track no running statistics."""

    def __init__(self, kind, c, gs, d, rank, layout, gen, dev, cond=False, track=True):
        import dwt_b200
        import oracle.torch_port as port
        self.kind, self.c, self.gs, self.track = kind, c, gs, track
        self.owner = {"shared": [0] * d, "distinct": list(range(d)), "mixed": [0] + [1] * (d - 1)}[layout]
        assert layout != "mixed" or d >= 3
        own = {}
        for o in sorted(set(self.owner)):
            rm = 0.1 * torch.randn(c, device=dev, generator=gen)
            if kind == "whiten":
                if cond:
                    q = torch.linalg.qr(torch.randn(c // gs, gs, gs, device=dev, generator=gen, dtype=torch.float64))[0]
                    ev = torch.logspace(2, -2, gs, device=dev, dtype=torch.float64)
                    rv = (q * ev) @ q.mT
                    rv = (0.5 * (rv + rv.mT)).float()
                else:
                    a = torch.randn(c // gs, gs, gs, device=dev, generator=gen)
                    rv = a @ a.transpose(1, 2) / gs + 0.5 * torch.eye(gs, device=dev)
                own[o] = (rm.view(1, c, 1, 1), rv)
            else:
                own[o] = (rm, 0.5 + torch.rand(c, device=dev, generator=gen))
        bn_cls = {2: "BatchNorm1d", 3: "BatchNorm1d", 4: "BatchNorm2d", 5: "BatchNorm3d"}[rank]
        self.mods, self.ref = [], []
        own64 = {o: (a.double(), b.double()) for o, (a, b) in own.items()}
        for o in self.owner:
            if kind == "whiten":
                m = dwt_b200.WTransform2d(c, gs, running_m=own[o][0], running_var=own[o][1], track_running_stats=track)
                r = port.WTransform2d(c, gs, running_m=own64[o][0], running_var=own64[o][1], track_running_stats=track)
                m.to(dev)                           # default buffers of untracked modules; borrowed ones stay put
                r.to(dev)
            else:
                m = getattr(dwt_b200, bn_cls)(c, *own[o], affine=False, momentum=None, track_running_stats=track)
                r = getattr(port, bn_cls)(c, *own64[o], affine=False, momentum=None, track_running_stats=track)
                if track:
                    m.num_batches_tracked.fill_(NBT0)
                    r.num_batches_tracked.fill_(NBT0)
            self.mods.append(m)
            self.ref.append(r)
        second = "running_variance" if kind == "whiten" else "running_var"
        self.buf32, self.buf64 = {}, {}
        for o in sorted(set(self.owner)):          # the buffers the modules hold (their own, when they track nothing)
            i = self.owner.index(o)
            if getattr(self.mods[i], "running_mean", None) is not None:
                self.buf32[o] = (self.mods[i].running_mean, getattr(self.mods[i], second))
                self.buf64[o] = (self.ref[i].running_mean, getattr(self.ref[i], second))
        self.eps = self.mods[0].eps
        self.norm = dwt_b200.DomainTripleNorm(kind, c, gs, n_domains=d)

    def train(self, mode):
        for m in self.mods + self.ref:
            m.train(mode)

    def batch_stats(self, x64):
        """fp64 batch mean and (biased) covariance / variance."""
        dims = [0] + list(range(2, x64.dim()))
        mu = x64.mean(dim=dims)
        xc = x64 - _bcast(mu, x64.dim())
        if self.kind == "bn":
            return mu, xc.square().mean(dim=dims)
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


def _family(kind, c, gs, cl, n, hw):
    from dwt_b200 import _native as nv
    if gs in (1, 2, 4) or kind == "bn":
        return "cl" if cl and nv.channels_last_supported(c, gs) else "small"
    if cl and nv.tensor_core_nhwc_supported(n, c, hw, gs):
        return "tc_nhwc"
    return "tc" if (gs in (8, 16, 32, 64) and hw >= 32 and n * hw >= 4096) else "tiled"


def _check(dev, worst, label, group, *, kind, c, gs, d, n, spatial, cl=False, mode, layout="shared", epi="relu",
           frozen=False, via="site", cond=False, track=True, count_batches=True, bad_group=None, tol=None, seed=0):
    """Run one site on the kernels and on the fp64 reference; assert every comparison and the kernels that ran.

    mode: eval (forward + backward on the running statistics) | nograd (train-mode forward under no_grad, also checked
    bit for bit against a grad-enabled call) | replicated (train-mode modules, replicated=True, under no_grad, as the
    statistics-collection pass) | replicated_eval (the same with eval-mode modules).  epi: None | affine | relu |
    residual; frozen: gamma / beta need no gradient; via: site (DomainTripleNorm) | module (the layer itself, d = 1);
    bad_group: that group's running covariance is not positive definite (eval, forward only); tol: the norm-wise bound
    of the loose (whitening) comparisons, TOL unless stated."""
    from dwt_b200 import _native
    assert via == "site" or (d == 1 and epi is None)
    replicated = mode.startswith("replicated")
    training = mode in ("nograd", "replicated")
    grad = mode == "eval" and bad_group is None
    batch_stats = training or not track
    gen = torch.Generator(device=dev).manual_seed(seed)
    d_in = 1 if replicated else d
    shape = (d_in * n, c, *spatial)
    hw = math.prod(spatial) if spatial else 1
    fam = _family(kind, c, gs, cl, n, hw)
    fmt = CL if cl else torch.contiguous_format
    x = _activation(gen, shape, d_in, dev).contiguous(memory_format=fmt)
    r = _activation(gen, shape, d_in, dev).contiguous(memory_format=fmt) if epi == "residual" else None
    w1 = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=fmt) if grad else None
    affine, relu = epi is not None, epi in ("relu", "residual")
    gamma = (0.5 + torch.rand(c, device=dev, generator=gen)).view(c, *([1] * len(spatial)))
    beta = (0.3 * torch.randn(c, device=dev, generator=gen)).view(c, *([1] * len(spatial)))
    site_seed = seed + 1000
    site = _Site(kind, c, gs, d, len(shape), layout, torch.Generator(device=dev).manual_seed(site_seed), dev, cond, track)
    site.train(training)
    if bad_group is not None:
        assert kind == "whiten" and mode == "eval"
        for o in site.buf32:                     # fp32: negative definite; the fp64 reference factors the identity
            site.buf32[o][1][bad_group] = -torch.eye(gs, device=dev)
            site.buf64[o][1][bad_group] = torch.eye(gs, device=dev, dtype=torch.float64)
    before = {o: (a.clone(), b.clone()) for o, (a, b) in site.buf32.items()}
    x.requires_grad_(grad)
    if r is not None:
        r.requires_grad_(grad)
    gamma.requires_grad_(grad and not frozen)
    beta.requires_grad_(grad and not frozen)
    g64, b64 = _f64(gamma).requires_grad_(grad and not frozen), _f64(beta).requires_grad_(grad and not frozen)
    if not count_batches:                        # the caller bumps every training counter (the model's one launch)
        for m in site.mods:
            if m.training and kind == "bn" and track:
                m.num_batches_tracked += 1

    def call(s, inp, res, g, b):
        if via == "module":
            return s.mods[0](inp)
        return s.norm(inp, s.mods, g if affine else None, b if affine else None, relu=relu, residual=res,
                      replicated=replicated, count_batches=count_batches)

    # ---- CUDA
    records = []
    _native.clear_status(dev)
    with _record_saved_stats(records), torch.set_grad_enabled(grad):
        y, fprof = _profiled(lambda: call(site, x, r, gamma, beta))
    mask = None
    if grad and fam == "cl" and epi == "residual":
        mask = y.grad_fn.saved_tensors[5]
    bprof = {}
    if grad:
        _, bprof = _profiled(lambda: y.backward(w1))
    out = y.detach()
    assert out.is_contiguous(memory_format=fmt)
    if mode == "nograd" or replicated:
        assert y.grad_fn is None and not y.requires_grad, "a no-grad call recorded a graph"
    del y
    status = _native.status(dev)

    # ---- which kernels ran
    n_calls = 1
    if replicated and training and track:
        n_calls = len(site.buf32)                # one launch per distinct buffer pair
    want_fwd = FWD_TRAIN[fam] if batch_stats else FWD_EVAL[fam]
    assert set(fprof) == want_fwd, (label, sorted(fprof), sorted(want_fwd))
    assert fprof[APPLY[fam]]["launches"] == n_calls == len(records), (label, fprof, len(records))
    if grad:
        reduce = batch_stats or (affine and not frozen) or (fam == "cl" and epi == "residual")
        want_bwd = BWD_REDUCE[fam] if reduce else BWD_PREP[fam]
        assert set(bprof) == want_bwd, (label, sorted(bprof), sorted(want_bwd))

    # ---- no-grad train: the same call with autograd recording, on a twin site, bit for bit
    if mode == "nograd":
        twin = _Site(kind, c, gs, d, len(shape), layout, torch.Generator(device=dev).manual_seed(site_seed), dev, cond,
                     track)
        twin.train(True)
        xg = x.detach().clone().requires_grad_(True)
        gg, bg = gamma.detach().clone().requires_grad_(True), beta.detach().clone().requires_grad_(True)
        yg = call(twin, xg, None if r is None else r.detach().clone().requires_grad_(True), gg, bg)
        assert yg.grad_fn is not None
        assert torch.equal(yg.detach(), out), label
        for o in site.buf32:
            assert torch.equal(site.buf32[o][0], twin.buf32[o][0]) and torch.equal(site.buf32[o][1], twin.buf32[o][1])
        if kind == "bn" and track:
            assert [int(m.num_batches_tracked) for m in site.mods] == [int(m.num_batches_tracked) for m in twin.mods]
        del yg, xg, twin

    # ---- relu mask
    active = out > 0
    if mask is not None:
        relu_mask = _decode(mask, shape)
        assert torch.equal(relu_mask, active), "byte map != the kernel's own out > 0"
    else:
        relu_mask = active
    del active

    # ---- fp64 reference
    err = {}
    keep = torch.ones(c, dtype=torch.bool, device=dev)         # channels compared: all but a non-PD group's
    if bad_group is not None:
        keep[bad_group * gs:(bad_group + 1) * gs] = False
        assert torch.isnan(out[:, ~keep]).all() and not torch.isnan(out[:, keep]).any()
    kept = keep.nonzero()[:, 0]

    def sel(t, dim=1):
        return t if bad_group is None else t.index_select(dim, kept)

    def add(key, got, ref):
        err.setdefault(key, _Err()).add(got, ref)
    running0 = {o: (a.clone(), b.clone()) for o, (a, b) in site.buf64.items()}
    flips, far, agree, pmax = 0, 0.0, 0.0, 0.0
    for di in range(d):
        sl = slice(di * n, (di + 1) * n) if not replicated else slice(0, n)
        x64 = _f64(x[sl]).requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            pre = site.ref[di](x64)
            if replicated and di > 0:             # the other two branches only move their buffers
                continue
            if affine:
                pre = pre * g64 + b64
            if r is not None:
                r64 = _f64(r[sl]).requires_grad_(grad)
                pre = pre + r64
        with torch.no_grad():
            p, o = sel(pre.detach()), sel(out[sl])
            if relu:
                m = sel(relu_mask[sl])
                flip = m != (p > 0)
                nflip = int(flip.sum())
                if nflip:
                    far = max(far, p[flip].abs().max().item())
                flips += nflip
                pmax = max(pmax, p.abs().max().item())
                p = p.clamp_min(0)
                agree = max(agree, (o.double() - p).abs().masked_fill_(flip, 0.0).max().item())
            add("out", o, p)
            del p, o
        if grad:
            seed_grad = _f64(w1[sl])
            if relu:
                seed_grad.mul_(relu_mask[sl])
            (pre * seed_grad).sum().backward()
            add("dx", x.grad[sl], x64.grad)
            if r is not None:
                add("d_identity", r.grad[sl], r64.grad)
        del pre
        with torch.no_grad():
            if batch_stats:
                mu, cov = site.batch_stats(x64.detach())
            else:
                rm, rv = running0[site.owner[di]]
                mu, cov = rm.reshape(-1), rv
            for rec_mean, rec_w in (records if replicated else records[:1]):
                k = 0 if replicated else di
                add("mean", sel(rec_mean[k], 0), sel(mu, 0))
                g_keep = keep.view(-1, gs)[:, 0] if kind == "whiten" else keep
                add("cov", site.kernel_cov(rec_w[k][g_keep]), cov[g_keep])
        del x64
    if grad and affine and not frozen:
        add("dgamma", gamma.grad, g64.grad)
        add("dbeta", beta.grad, b64.grad)
    for o in site.buf32:
        if training and track:
            add("running_mean", site.buf32[o][0], site.buf64[o][0])
            add("running_var", site.buf32[o][1], site.buf64[o][1])
        else:                                    # eval and untracked modules move no buffer, not even by rounding
            assert torch.equal(site.buf32[o][0], before[o][0]) and torch.equal(site.buf32[o][1], before[o][1]), label
            assert torch.equal(site.buf64[o][0], running0[o][0]) and torch.equal(site.buf64[o][1], running0[o][1])
    if kind == "bn" and track:
        got_nbt = [int(m.num_batches_tracked) for m in site.mods]
        assert got_nbt == [int(m.num_batches_tracked) for m in site.ref] == [NBT0 + training] * d, (label, got_nbt)

    res = {k: e.both() for k, e in err.items()}
    far, agree = far / max(pmax, 1e-30), agree / max(pmax, 1e-30)
    print(label, "flips", flips, "%.1e %.1e" % (far, agree), {k: "%.1e %.1e" % v for k, v in res.items()})
    table = worst.setdefault((fam, group), {})
    for k, (rel, mx) in res.items():
        cls = "stats" if k.startswith(STAT_KEYS) else "values"
        old = table.get(cls, (0.0, 0.0))
        table[cls] = (max(old[0], rel), max(old[1], mx))
    if bad_group is None:
        assert status == 0, (label, status)
    else:
        assert status & _native.STATUS_NOT_PD, (label, status)
        _native.clear_status(dev)
    assert far <= max(1e-5, 2 * agree), ("the ReLU mask differs from the fp64 sign away from zero", label, far, agree)
    assert flips <= max(4, out.numel() // 10 ** 5), (label, flips)
    loose_tol = TOL if tol is None else tol
    for k, (rel, mx) in res.items():
        loose = kind == "whiten" and not k.startswith(STAT_KEYS)   # through a Cholesky factor
        assert rel < (loose_tol if loose else TOL_STAT), (label, k, rel, mx)
        assert mx < (5 * loose_tol if loose else 5 * TOL_STAT), (label, k, rel, mx)
    peak = torch.cuda.max_memory_allocated(dev)
    assert peak < 16 * GIB, f"peak device memory {peak / GIB:.1f} GiB"
    return res


# --------------------------------------------------------------------------- 1. every channels-last model site
@pytest.fixture(scope="module")
def model_sites(dev):
    """(kind, C, H, W, gs) of every DomainTripleNorm call of one channels-last fused training forward of the harness
    ResNet-50-DWT at 224^2 (one image per domain), in call order, duplicates removed; recorded at the functional entry
    points, the downsample site of a two-site tail included."""
    import dwt_b200
    from dwt_b200 import functional as F
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    calls = []
    norm, tail_pair = F.norm, F.tail_pair

    def rec_norm(x, *args, **kw):
        calls.append((kw["kind"], x.shape[1], x.shape[2], x.shape[3], kw["group_size"]))
        return norm(x, *args, **kw)

    def rec_tail_pair(x, xd, *args, **kw):
        calls.append((kw["kind"], x.shape[1], x.shape[2], x.shape[3], kw["group_size"]))
        calls.append((kw["kind"], xd.shape[1], xd.shape[2], xd.shape[3], kw["group_size"]))
        return tail_pair(x, xd, *args, **kw)
    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        mp.setattr(F, "norm", rec_norm)
        mp.setattr(F, "tail_pair", rec_tail_pair)
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        model = build_resnet50_dwt(sd, dwt_b200, site_mode="fused", channels_last=True).to(dev).train()
        images, _ = synth_batch(seed=2, per_domain=1, size=224)
        model(images.to(dev).contiguous(memory_format=CL))
    sites = []
    for key in calls:
        if key not in sites:
            sites.append(key)
    return sites


SITE_MODES = [   # label, mode, epilogue, frozen gamma / beta, buffers, count_batches
    ("eval", "eval", "relu", False, "shared", True),
    ("eval_frozen", "eval", "relu", True, "shared", True),
    ("eval_residual", "eval", "residual", False, "mixed", True),
    ("nograd", "nograd", "relu", False, "shared", True),
    ("replicated_shared", "replicated", "relu", False, "shared", True),
    ("replicated_distinct_residual", "replicated", "residual", False, "distinct", False),
    ("replicated_mixed", "replicated", "affine", False, "mixed", True),
]


@pytest.mark.parametrize("smode", SITE_MODES, ids=[m[0] for m in SITE_MODES])
def test_every_model_site_geometry(smode, model_sites, dev, worst):
    """Each distinct site geometry of the channels-last model (stem 64@112^2 down to 2048@7^2) at 2 images per domain."""
    name, mode, epi, frozen, layout, count = smode
    assert model_sites[0] == ("whiten", 64, 112, 112, 4), model_sites[0]                 # the stem
    assert ("bn", 2048, 7, 7, 1) in model_sites and ("whiten", 256, 56, 56, 4) in model_sites
    failures = []
    for i, (kind, c, h, w, gs) in enumerate(model_sites):
        label = f"{name} {kind} {c}@{h}x{w} gs{gs}"
        try:
            _check(dev, worst, label, name, kind=kind, c=c, gs=gs, d=3, n=2, spatial=(h, w), cl=True, mode=mode,
                   layout=layout, epi=epi, frozen=frozen, count_batches=count, seed=100 + i)
        except AssertionError as e:
            failures.append(f"{label}: {e}")
    assert not failures, "\n".join(failures)


# --------------------------------------------------------------------------- 2. channels-last launch edges in eval
def _edge_rows(rows, c, d, sms):
    """Rows per domain of a named launch edge of the channels-last kernels (as test_channels_last_fp64.py)."""
    cw = min(c // 4, THREADS)
    rpi, cap = THREADS // cw, max(1, STATS_SLOTS * sms // (((c // 4) // cw) * d))
    chunk = rpi * STATS_UNROLL
    if rows == "lt_rpi":
        assert 9 < rpi
    return {"lt8": 4, "lt_rpi": 9, "chunk": chunk, "chunk+1": chunk + 1, "ragged": (2 * cap + 7) * chunk - 5}[rows]


CL_EVAL_EDGES = [   # C, kind, gs, domains, rows per domain, epilogue
    (4, "whiten", 4, 3, "lt_rpi", "relu"),
    (4, "whiten", 2, 1, "lt8", "residual"),
    (4, "bn", 1, 4, "ragged", "affine"),
    (8, "bn", 1, 2, "ragged", "relu"),
    (8, "whiten", 4, 4, "chunk", "residual"),
    (1024, "bn", 1, 4, "chunk", "residual"),
    (1024, "whiten", 4, 3, "ragged", "relu"),
    (4096, "whiten", 2, 3, "ragged", "affine"),
    (4096, "whiten", 4, 2, "chunk+1", "residual"),
]


@pytest.mark.parametrize("c,kind,gs,d,rows,epi", CL_EVAL_EDGES,
                         ids=[f"c{e[0]}-{e[1]}-gs{e[2]}-d{e[3]}-{e[4]}-{e[5]}" for e in CL_EVAL_EDGES])
def test_channels_last_eval_edges(c, kind, gs, d, rows, epi, dev, worst):
    """Eval with a distinct running-buffer pair per domain: eval_prep's per-domain indexing of rmean[d] / rcov[d]."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    m = _edge_rows(rows, c, d, sms)
    n, hw = (1, (2, 2)) if m == 4 else (1, (3, 3)) if m == 9 else (1, (1, m))
    _check(dev, worst, f"c{c} {kind} gs{gs} d{d} {rows}={m}", "cl_eval_edges", kind=kind, c=c, gs=gs, d=d, n=n,
           spatial=hw, cl=True, mode="eval", layout="distinct", epi=epi, seed=c + d)


# --------------------------------------------------------------------------- 3. the NCHW small family
SMALL = [   # label, kind, gs, D, N, spatial, epilogue, frozen, buffers, mode, via, track
    ("gs1_vec4_eval", "bn", 1, 3, 4, (6, 6), "relu", False, "mixed", "eval", "site", True),
    ("gs1_vec1_eval_frozen", "bn", 1, 2, 5, (5, 5), "affine", True, "distinct", "eval", "site", True),
    ("gs2_vec4_eval_residual", "whiten", 2, 3, 4, (4, 8), "residual", False, "mixed", "eval", "site", True),
    ("gs2_vec1_eval_frozen_relu", "whiten", 2, 4, 3, (3, 7), "relu", True, "distinct", "eval", "site", True),
    ("gs4_vec4_eval", "whiten", 4, 4, 3, (8, 8), "affine", False, "mixed", "eval", "site", True),
    ("gs4_7x7_eval_residual", "whiten", 4, 3, 2, (7, 7), "residual", False, "distinct", "eval", "site", True),
    ("gs4_7x7_eval_frozen_residual", "whiten", 4, 3, 2, (7, 7), "residual", True, "mixed", "eval", "site", True),
    ("gs4_eval_none", "whiten", 4, 2, 4, (6, 6), None, False, "distinct", "eval", "site", True),
    ("gs4_module_eval", "whiten", 4, 1, 8, (6, 6), None, False, "shared", "eval", "module", True),
    ("bn1d_hw1_eval", "bn", 1, 1, 64, (), None, False, "shared", "eval", "module", True),
    ("bn1d_len7_eval", "bn", 1, 1, 16, (7,), None, False, "shared", "eval", "module", True),
    ("bn3d_eval", "bn", 1, 1, 4, (3, 5, 6), None, False, "shared", "eval", "module", True),
    ("gs4_7x7_nograd", "whiten", 4, 3, 2, (7, 7), "relu", False, "mixed", "nograd", "site", True),
    ("gs1_nograd_residual", "bn", 1, 4, 3, (4, 4), "residual", False, "distinct", "nograd", "site", True),
    ("gs2_vec1_nograd", "whiten", 2, 1, 6, (5, 5), "affine", False, "shared", "nograd", "site", True),
    ("bn3d_nograd", "bn", 1, 1, 4, (3, 5, 6), None, False, "shared", "nograd", "module", True),
    ("gs2_replicated_residual", "whiten", 2, 3, 4, (4, 8), "residual", False, "shared", "replicated", "site", True),
    ("gs4_7x7_replicated", "whiten", 4, 3, 4, (7, 7), "relu", False, "distinct", "replicated", "site", True),
    ("gs1_replicated_mixed", "bn", 1, 3, 4, (5, 5), "affine", False, "mixed", "replicated", "site", True),
    ("gs4_untracked_eval", "whiten", 4, 3, 3, (6, 6), "relu", False, "distinct", "eval", "site", False),
    ("gs1_untracked_eval", "bn", 1, 2, 3, (5, 5), "affine", False, "distinct", "eval", "site", False),
    ("bn1d_untracked_eval", "bn", 1, 1, 32, (), None, False, "shared", "eval", "module", False),
]


@pytest.mark.parametrize("case", SMALL, ids=[s[0] for s in SMALL])
def test_nchw_small_family(case, dev, worst):
    label, kind, gs, d, n, spatial, epi, frozen, layout, mode, via, track = case
    _check(dev, worst, label, mode, kind=kind, c=48, gs=gs, d=d, n=n, spatial=spatial, mode=mode, layout=layout,
           epi=epi, frozen=frozen, via=via, track=track, seed=len(label) + gs)


def test_nchw_replicated_without_counting_batches(dev, worst):
    _check(dev, worst, "bn replicated count_batches=False", "replicated", kind="bn", c=64, gs=1, d=3, n=4,
           spatial=(6, 6), mode="replicated", layout="mixed", epi="residual", count_batches=False, seed=3)


# --------------------------------------------------------------------------- 4. replicated on the other families
OTHER = [   # label, family, C, gs, N, (H, W), channels-last, epilogue, buffers
    ("nchw_gs64_tc", "tc", 128, 64, 16, (16, 16), False, "relu", "mixed"),
    ("cl_gs32_tc", "tc_nhwc", 64, 32, 16, (16, 16), True, "residual", "distinct"),
    ("nchw_gs12_tiled", "tiled", 48, 12, 4, (5, 5), False, "affine", "shared"),
]


@pytest.mark.parametrize("case", OTHER, ids=[o[0] for o in OTHER])
def test_replicated_other_families(case, dev, worst):
    """gamma / beta / ReLU / residual follow the tensor-core and tiled kernels as tensor ops."""
    label, family, c, gs, n, hw, cl, epi, layout = case
    assert _family("whiten", c, gs, cl, n, hw[0] * hw[1]) == family
    _check(dev, worst, label, "replicated", kind="whiten", c=c, gs=gs, d=3, n=n, spatial=hw, cl=cl, mode="replicated",
           layout=layout, epi=epi, seed=c + gs)


# --------------------------------------------------------------------------- 5. conditioning and status
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "channels_last"])
def test_eval_condition_1e4(cl, dev, worst):
    """Running covariances with eigenvalues 1e2 .. 1e-2 (condition number 1e4; about 9e3 after the eps shrinkage)."""
    _check(dev, worst, f"cond1e4 {'cl' if cl else 'nchw'}", "cond1e4", kind="whiten", c=64, gs=4, d=3, n=4,
           spatial=(8, 8), cl=cl, mode="eval", layout="distinct", epi="relu", cond=True, seed=21)


@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "channels_last"])
def test_eval_not_positive_definite(cl, dev, worst):
    """One group's running covariance is negative definite: DWT_STATUS_NOT_PD is set, that group's output is NaN and
    every other group stays within tolerance."""
    _check(dev, worst, f"not_pd {'cl' if cl else 'nchw'}", "not_pd", kind="whiten", c=32, gs=4, d=3, n=2,
           spatial=(8, 8), cl=cl, mode="eval", layout="shared", epi="affine", bad_group=3, seed=22)


@pytest.mark.parametrize("layout", ["distinct", "mixed"])
@pytest.mark.parametrize("kind", ["whiten", "bn"])
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "channels_last"])
def test_replicated_eval(cl, kind, layout, dev, worst):
    """replicated=True through eval-mode modules is the first third of cat((d, d, d)) through them: normalised with the
    first module's running buffers (not the batch's statistics), no buffer or counter moved."""
    _check(dev, worst, f"replicated_eval {kind} {layout} {'cl' if cl else 'nchw'}", "replicated_eval", kind=kind,
           c=64, gs=4 if kind == "whiten" else 1, d=3, n=4, spatial=(8, 8), cl=cl, mode="replicated_eval",
           layout=layout, epi="residual", seed=23)


# --------------------------------------------------------------------------- 6. the whole chain
@contextlib.contextmanager
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# measured on an H100 80GB HBM3 at 700 W: 3.1e-5 (running buffers) and 2.0e-5 (logits) norm-wise
CHAIN_TOL = {"running": TOL_STAT, "logits": TOL_STAT}


@pytest.mark.parametrize("cl", [True, False], ids=["channels_last", "nchw"])
def test_collect_stats_then_eval_chain(cl, dev, worst):
    """collect_stats(replicated=True), 2 passes over 2 batches, then an eval forward of the fused model, against an fp64
    port model (site_mode "modules") that runs the reference form cat((d, d, d)) and then evaluates.  The fp64 model is
    built from a float64 copy of the state dict and converts only its conv / fc parameters: Module.double() would
    re-allocate the borrowed running buffers per module and break the aliasing of the three branches."""
    import dwt_b200
    import oracle.torch_port as port
    from harness.resnet50_dwt import build_resnet50_dwt, collect_stats
    from harness.synth import synth_batch, synth_state_dict
    fmt = CL if cl else torch.contiguous_format
    images, _ = synth_batch(seed=5, per_domain=2, size=96)
    images = images.to(dev)
    batches = [images[0:2], images[2:4]]
    probe = images[4:6]
    sd = synth_state_dict(seed=1)
    with _no_tf32():
        model = build_resnet50_dwt({k: v.to(dev) for k, v in sd.items()}, dwt_b200, site_mode="fused",
                                   channels_last=cl).to(dev).eval()
        collect_stats(model, [b.contiguous(memory_format=fmt) for b in batches], passes=2, replicated=True)
        with torch.no_grad():
            logits = model(probe.contiguous(memory_format=fmt))
        ref = build_resnet50_dwt({k: (v.double() if v.is_floating_point() else v).to(dev) for k, v in sd.items()}, port,
                                 site_mode="modules").to(dev).eval()
        for m in ref.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)):
                for p in m.parameters():
                    p.data = p.data.double()
        collect_stats(ref, [b.double() for b in batches], passes=2, replicated=False)
        with torch.no_grad():
            logits64 = ref(probe.double())
    assert not model.training and not ref.training
    got, want = model.state_dict(), ref.state_dict()
    assert set(got) == set(want)
    bufs = {}                                    # running buffer -> (norm-wise, max-elementwise) error
    for k, v in got.items():
        if k.endswith("num_batches_tracked"):
            assert int(v) == int(want[k]) == 2 * len(batches), (k, int(v), int(want[k]))
        elif "running" in k:
            e = _Err()
            e.add(v, want[k])
            bufs[k] = e.both()
    assert len(bufs) > 100, len(bufs)
    where = max(bufs, key=lambda k: bufs[k][0])
    e = _Err()
    e.add(logits, logits64)
    err = {"running": (bufs[where][0], max(m for _, m in bufs.values()), where), "logits": (*e.both(), "")}
    print(f"chain {'cl' if cl else 'nchw'}:", {k: "%.1e %.1e %s" % v for k, v in err.items()})
    table = worst.setdefault(("model", "chain"), {})
    for k, (rel, mx, _) in err.items():
        old = table.get(k, (0.0, 0.0))
        table[k] = (max(old[0], rel), max(old[1], mx))
    assert dwt_b200._native.status(dev) == 0
    for k, (rel, mx, where) in err.items():
        assert rel < CHAIN_TOL[k] and mx < 5 * CHAIN_TOL[k], (k, rel, mx, where)
    peak = torch.cuda.max_memory_allocated(dev)
    assert peak < 16 * GIB, f"peak device memory {peak / GIB:.1f} GiB"
