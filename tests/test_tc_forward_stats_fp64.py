"""The tensor-core whitening forward statistics (tc_stats, tc_gram_pair at group size 128, dense_partial_reduce and the
dense finalize) against float64, one stage at a time, beside a float32 yardstick.

The batch covariance feeds a Cholesky factor (or the Newton-Schulz iteration of the ZCA basis), so its error comes back
multiplied by the condition number in y, and once more in dx when the output gradient lies mostly along y.  The Gram
kernels accumulate the products of hundreds of tiles per CTA at production sizes (about 380 at BASELINE config 2), so
these tests follow the error along the accumulation length and localise it stage by stage:

  mean   save_mean against the float64 mean, in units of each channel's float64 sigma
  cov    the kernel's un-shrunk batch covariance against the float64 one (two-pass, one slab of images at a time), both
         divided by sigma_i sigma_j: the error on the correlation scale, so that channels of any size count alike
  W      save_w against the float64 factor of (1 - eps) cov_kernel + eps I built from the kernel's own covariance:
         the finalize alone (inverse Cholesky factor; ZCA basis: zca_reference's float64 Newton-Schulz iteration)
  y      end to end, against oracle.torch_port.WTransform2d in float64 (zca_reference.zca_torch for the ZCA basis)

Each stage is norm-wise per (domain, group), the worst group reported, with the maximum elementwise error beside it.
The kernel's covariance is read without any extra hook: with momentum = 1 the whitening EMA is 1 * (cov * 1) + 0 * old
(unbias = 1), so running_variance holds it bit for bit (asserted in test_short_control).

The float32 yardstick is the reference operator sequence in float32 on the GPU with TF32 off in cuBLAS and cuDNN: the
mean, bmm(T, T^T) / M, Cholesky and inverse (y: the torch port in float32).  Mean and covariance must stay within
RATIO x the yardstick's error or FLOOR, whichever is larger, at every accumulation length, and the covariance within
BOUND_COV of float64 as well: cuBLAS's float32 bmm over K = N*HW is itself 2e-5 .. 1e-3 off at 64 .. 760 tiles per CTA
(group sizes 32..128; 3e-7 at 8 and 16), too loose a yardstick to tell one rounding per tile from one per instruction.
W within BOUND_W of float64 at the kernel's covariance; y within BOUND_Y norm-wise and BOUND_Y_MAX max-elementwise, or
RATIO x the yardstick.  bf16 inputs: against float64 of the widened values, plus the error of rounding the float64 y to
bf16; and the statistics bit-identical to the float32 call on the widened values.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit).  A fresh accumulator per 32-pixel tile added into an fp32
register sum (norm_tc.cu): covariance 4.5e-7 .. 1.7e-6 (bf16) in every case and flat along the accumulation length
(7.2e-7 at 2 tiles per CTA, 7.3e-7 at 16, 7.6e-7 at 760); mean at most 1.6e-6 sigma (|mean| = 50 sigma, the
yardstick's 2.6e-6); W at most 4.9e-6 (condition number 1e4), 1.3e-7 elsewhere; y at most 5.5e-6 (condition number
1e4; the yardstick's 8.2e-6), bf16 1.7e-3, its rounding alone.  The single accumulator per CTA this replaced: the
covariance grew with the length, 4.5e-7 / 1.6e-6 / 5.8e-6 / 3.9e-5 / 8.1e-5 at 2 / 16 / 64 / 380 / 760 tiles per CTA,
4.3e-5 at gs 8 (where it failed even the yardstick rule, 3.5e-7) and y 1.0e-4 .. 3.8e-4 at condition numbers 1e2 ..
1e4; mean and W were as now.  It fails every case here at 64 tiles per CTA or more.
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import zca_reference as Z  # noqa: E402
from test_tc_backward_fp64 import _Err, fp32_strict, mixed, ref_forward  # noqa: E402

pytestmark = pytest.mark.gpu

RATIO = 4.0                  # mean and covariance: at most RATIO x the float32 yardstick's error ...
FLOOR = 2e-6                 # ... or FLOOR, whichever is larger
BOUND_COV = 3e-6             # and the covariance within BOUND_COV of float64 at every length (norm-wise)
BOUND_W = 2e-5               # W against float64 at the kernel's own covariance (norm-wise)
BOUND_Y, BOUND_Y_MAX = 1e-3, 5e-3
EPS = 1e-3                   # WTransform2d's default shrinkage
TC_CH = 64                   # channels of a tensor-core super-block (norm_tc.cu kTileCh)
TC_BOX = 32                  # pixels of a Gram tile (norm_tc.cu kTilePx)
TC_MIN_M = 4096              # N * HW per domain below which the tiled kernels take the call (norm_tc.cu tc_supports)
SLAB_ELEMS = 1 << 25         # elements of one float64 slab
CONFIG2 = (256, 256, 56, 56)  # BASELINE.json configs[1]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\ntensor-core forward statistics against float64 (worst group: norm-wise, max-elementwise, (float32 yardstick"
          " norm-wise)):")
    for k in sorted(table):
        print("  %-34s %s" % (k, ", ".join(f"{s} {r:.1e} {m:.1e} ({y:.1e})" for s, (r, m, y) in table[k].items())))


# --------------------------------------------------------------------------- launch shape (api.cu tc_chunks)
def tc_chunks(sms, problems, tiles):
    """CTAs per problem of a Gram kernel: one wave of 2 CTAs per SM over the problems, capped at the tile count."""
    return max(1, min(2 * sms // problems, tiles))


def tiles_per_cta(sms, n, c, hw, d=1, pair=False):
    """Tiles one Gram CTA accumulates: N * ceil(HW / 32) per problem over tc_chunks CTAs.  Problems: (domain,
    super-block) for tc_stats; (domain, pair of super-blocks) for tc_gram_pair (pair = True, group size 128)."""
    tiles = n * -(-hw // TC_BOX)
    sb = -(-c // TC_CH)
    return tiles / tc_chunks(sms, (sb // 2 if pair else sb) * d, tiles)


def n_for_tiles(sms, target, c, hw):
    """The batch size whose tc_stats CTAs accumulate about `target` tiles each (d = 1)."""
    return max(1, round(target * max(1, 2 * sms // -(-c // TC_CH)) / -(-hw // TC_BOX)))


# --------------------------------------------------------------------------- inputs (float32 NCHW on the device)
def conditioned_at_scale(shape, gs, cond, dev, seed=0):
    """zca_reference.conditioned_input in float64 on the device (the numpy version is minutes at config 2): per group,
    the samples whitened exactly, then given the spectrum 1 .. 1/cond under a random rotation, mean 1."""
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    out = torch.empty(shape, device=dev)
    for g0 in range(0, c, gs):
        z = torch.randn(gs, n * h * w, dtype=torch.float64, device=dev, generator=g)
        z -= z.mean(-1, keepdim=True)
        lam, v = torch.linalg.eigh(z @ z.T / z.shape[-1])
        q, _ = torch.linalg.qr(torch.randn(gs, gs, dtype=torch.float64, device=dev, generator=g))
        spec = torch.logspace(0, -math.log10(cond), gs, dtype=torch.float64, device=dev)
        a = q @ torch.diag(spec.sqrt()) @ q.T @ v @ torch.diag(lam.rsqrt()) @ v.T
        out[:, g0:g0 + gs] = (a @ z).view(gs, n, h, w).transpose(0, 1).float() + 1.0
        del z
    return out


def post_relu(shape, dev, seed=0):
    """ReLU of the zero-mean microbench mixture: about half zeros, a positive mean."""
    return torch.relu(mixed(shape, dev, seed, shift=0.0))


def mean_50sigma(shape, dev, seed=0):
    """Every channel's |mean| about 50 of its sigmas (signs alternate)."""
    x = mixed(shape, dev, seed, shift=0.0)
    sigma = x.std(dim=(0, 2, 3))
    sign = torch.tensor([1.0, -1.0], device=dev).repeat(shape[1] // 2)
    return x.add_((50.0 * sign * sigma).view(1, -1, 1, 1))


def spread_scales(shape, dev, seed=0):
    """Per-channel scales log-spread over 1e-3 .. 1e3 inside every group (interleaved over the channels)."""
    c = shape[1]
    scale = torch.logspace(-3, 3, c, device=dev)[torch.randperm(c, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))]
    return mixed(shape, dev, seed).mul_(scale.view(1, -1, 1, 1))


def pilot_30sigma(shape, dev, seed=0):
    """The microbench input with image 0's pilot window (<= 32 mid-image pixels, the NCHW kernels' first shift
    estimate) 30 sigma off: the input of test_nchw_fp64.py's _pilot_window, here at the production length."""
    x = mixed(shape, dev, seed)
    hw = shape[2] * shape[3]
    npx = min(hw, 32)
    p0 = ((hw - npx) // 2) & ~3
    sigma = x.std(dim=(0, 2, 3))
    x.view(shape[0], shape[1], hw)[0, :, p0:p0 + npx] += 30.0 * sigma.view(-1, 1)
    return x


# --------------------------------------------------------------------------- references
def ref_stats(x, d, gs):
    """float64 mean [d, C], sigma [d, C] and covariance [d, G, gs, gs] of x [d*N, C, H, W], two-pass, one slab of
    images at a time (no float64 copy of the whole tensor)."""
    dn, c = x.shape[:2]
    n, hw = dn // d, x[0, 0].numel()
    step = max(1, SLAB_ELEMS // (c * hw))
    f64 = dict(dtype=torch.float64, device=x.device)
    means, covs = [], []
    for di in range(d):
        rng = [(a, min(a + step, (di + 1) * n)) for a in range(di * n, (di + 1) * n, step)]
        s = torch.zeros(c, **f64)
        for a, b in rng:
            s += x[a:b].double().sum((0, 2, 3))
        mean = s / (n * hw)
        cov = torch.zeros(c // gs, gs, gs, **f64)
        for a, b in rng:
            xg = (x[a:b].double() - mean.view(1, c, 1, 1)).transpose(0, 1).reshape(c // gs, gs, -1)
            cov += xg @ xg.mT
            del xg
        means.append(mean)
        covs.append(cov / (n * hw))
    cov = torch.stack(covs)
    return torch.stack(means), cov.diagonal(dim1=-2, dim2=-1).reshape(d, c).sqrt(), cov


def yardstick_stats(x, d, gs):
    """The reference operator sequence in float32 (TF32 off): mean [d, C] and covariance [d, G, gs, gs]."""
    dn, c = x.shape[:2]
    n = dn // d
    restore = fp32_strict()
    try:
        means, covs = [], []
        for di in range(d):
            xg = x[di * n:(di + 1) * n].transpose(0, 1).reshape(c // gs, gs, -1)
            mean = xg.mean(-1)
            t = xg - mean[..., None]
            del xg
            covs.append(torch.bmm(t, t.mT) / t.shape[-1])
            means.append(mean.reshape(c))
            del t
    finally:
        restore()
    return torch.stack(means), torch.stack(covs)


def factor64(cov, T):
    """float64 W of S = (1 - eps) cov + eps I, cov [..., gs, gs]: the inverse Cholesky factor (T = None) or the ZCA
    basis after T Newton-Schulz iterations (zca_reference.zca_torch on the running buffers)."""
    gs = cov.shape[-1]
    cov = cov.double().reshape(-1, gs, gs)
    if T:
        g = cov.shape[0]
        probe = torch.zeros(1, g * gs, 1, 1, dtype=torch.float64, device=cov.device)
        return Z.zca_torch(probe, gs, T, eps=EPS, running_mean=torch.zeros(g * gs, dtype=torch.float64, device=cov.device),
                           running_cov=cov, train=False)[3]
    eye = torch.eye(gs, dtype=torch.float64, device=cov.device)
    low = torch.linalg.cholesky((1 - EPS) * cov + EPS * eye)
    return torch.linalg.solve_triangular(low, eye.expand_as(low), upper=False)


def per_group(got, ref, scale=None):
    """got, ref [G, ...] (scale: divides both): worst (norm-wise, max-elementwise) over the groups."""
    got, ref = got.double(), ref.double()
    if scale is not None:
        got, ref = got / scale, ref / scale
    diff = (got - ref).flatten(1)
    ref = ref.flatten(1)
    r = (diff.norm(dim=1) / ref.norm(dim=1).clamp_min(1e-300)).max().item()
    m = (diff.abs().amax(1) / ref.abs().amax(1).clamp_min(1e-300)).max().item()
    return r, m


def mean_err(got, mean64, sigma, gs):
    """Worst group's RMS and max of (got - mean) / sigma."""
    e = ((got.double() - mean64) / sigma).view(-1, gs)
    return (e.norm(dim=1) / math.sqrt(gs)).max().item(), e.abs().max().item()


# --------------------------------------------------------------------------- one case
def run_case(dev, worst, label, x, gs, d=1, nhwc=False, bf16=False, T=None, tiles=None):
    """x [d*N, C, H, W] float32 NCHW through the kernels (d = 1: the module; d > 1: one DomainTripleNorm site) with
    momentum 1; the four stages against float64 and the float32 yardstick, domain by domain, group by group."""
    import dwt_b200
    from dwt_b200 import _native as nv
    dn, c = x.shape[:2]
    n, hw = dn // d, x[0, 0].numel()
    assert n * hw >= TC_MIN_M and hw >= TC_BOX
    x = x.detach().bfloat16().float() if bf16 else x.detach()     # the reference sees the widened values
    cl = torch.channels_last if nhwc else torch.contiguous_format
    xin = (x.bfloat16() if bf16 else x).contiguous(memory_format=cl).detach().requires_grad_(True)

    def module():
        return (dwt_b200.ZCAWTransform2d(c, gs, momentum=1.0, iterations=T) if T
                else dwt_b200.WTransform2d(c, gs, momentum=1.0)).to(dev).train()

    def run(inp):
        mods = [module() for _ in range(d)]
        y = mods[0](inp) if d == 1 else dwt_b200.DomainTripleNorm("whiten", c, gs, n_domains=d)(inp, mods, None, None)
        save_mean, save_w = (t.detach() for t in y.grad_fn.saved_tensors[1:3])
        cov = torch.stack([m.running_variance for m in mods])
        return y.detach(), save_mean, save_w, cov

    nv.profile_begin()
    y, save_mean, save_w, cov_k = run(xin)
    fam_ran = set(nv.by_family(nv.profile_end()))
    want = "tc_stats" + ("_nhwc" if nhwc else "") + ("_bf16" if bf16 else "")
    assert want in fam_ran and not any(f.startswith(("tiled", "small", "cl_")) for f in fam_ran), (label, fam_ran)
    assert save_mean.shape == (d, c) and save_w.shape == (d, c // gs, gs, gs) and cov_k.shape == save_w.shape
    if bf16:
        # the bf16 kernels transform to exactly the fp32 kernels' operands: the statistics are the fp32 call's on x.float()
        _, m32, w32, c32 = run(x.contiguous(memory_format=cl).detach().requires_grad_(True))
        assert torch.equal(save_mean, m32) and torch.equal(save_w, w32) and torch.equal(cov_k, c32), label
        del m32, w32, c32

    mean64, sigma64, cov64 = ref_stats(x, d, gs)
    mean32, cov32 = yardstick_stats(x, d, gs)
    sig_outer = (sigma64[:, :, None] * sigma64[:, None, :]).view(d, c // gs, gs, c)
    sig_outer = torch.stack([sig_outer[:, g, :, g * gs:(g + 1) * gs] for g in range(c // gs)], 1)   # [d, G, gs, gs]
    res = {}
    for di in range(d):
        st = {
            "mean": mean_err(save_mean[di], mean64[di], sigma64[di], gs) + (mean_err(mean32[di], mean64[di], sigma64[di], gs)[0],),
            "cov": per_group(cov_k[di], cov64[di], sig_outer[di]) + (per_group(cov32[di], cov64[di], sig_outer[di])[0],),
            "W": per_group(save_w[di], factor64(cov_k[di], T)) + (float("nan"),),
        }
        for k, v in st.items():
            res[k] = max(res.get(k, (0.0, 0.0, 0.0)), v)
    del cov64, cov32

    # y end to end: float64 reference and float32 yardstick, one (domain, channel slab) at a time
    x64 = None
    err, yard, rnd = _Err(), _Err(), _Err()
    slab = max(gs, SLAB_ELEMS // (n * hw) // gs * gs)
    restore = fp32_strict()
    try:
        with torch.no_grad():
            for di in range(d):
                rs = slice(di * n, (di + 1) * n)
                for c0 in range(0, c, slab):
                    cs = slice(c0, min(c, c0 + slab))
                    x64 = x[rs, cs].double()
                    y64 = ref_forward(x64, gs, T)
                    err.add(y[rs, cs], y64)
                    yard.add(ref_forward(x[rs, cs].contiguous(), gs, T), y64)
                    if bf16:
                        rnd.add(y64.bfloat16(), y64)
                    del x64, y64
    finally:
        restore()
    (ry, my), yy = err.both(), yard.both()[0]
    fr, fm = rnd.both() if bf16 else (0.0, 0.0)
    res["y"] = (ry, my, yy)
    worst[f"{label} [{tiles:.0f} tiles/CTA]" if tiles else label] = res
    del y, xin

    failures = []
    for k in ("mean", "cov"):
        r, _, yr = res[k]
        if r > max(RATIO * yr, FLOOR):
            failures.append(f"{k}: norm-wise {r:.2e} > max({RATIO} x float32 yardstick {yr:.2e}, {FLOOR:.0e})")
    if res["cov"][0] > BOUND_COV:
        failures.append(f"cov: norm-wise {res['cov'][0]:.2e} against float64 (bound {BOUND_COV:.0e})")
    if res["W"][0] > BOUND_W:
        failures.append(f"W: norm-wise {res['W'][0]:.2e} against float64 at the kernel's covariance (bound {BOUND_W:.0e})")
    if (ry > BOUND_Y + fr or my > BOUND_Y_MAX + fm) and ry > RATIO * yy:
        failures.append(f"y: norm-wise {ry:.2e}, max-elementwise {my:.2e} (bounds {BOUND_Y + fr:.1e}, {BOUND_Y_MAX + fm:.1e};"
                        f" float32 yardstick {yy:.2e})")
    assert not failures, f"{label}: " + "; ".join(failures)


# --------------------------------------------------------------------------- 1. accumulation length
@pytest.mark.parametrize("target", [16, 64, 380, 760])
def test_accumulation_length(target, dev, sms, worst):
    """The microbench input (mixed, shift 2) at C = 256, gs 64, 56^2, N such that every Gram CTA accumulates about 16,
    64, 380 (BASELINE config 2: N = 256) and 760 (N = 512, 1.6 GB) tiles: a covariance rounded once per tile keeps its
    error as the length grows, one rounded once per instruction of a long accumulation does not."""
    c, h, w = CONFIG2[1:]
    n = n_for_tiles(sms, target, c, h * w)
    tiles = tiles_per_cta(sms, n, c, h * w)
    assert abs(tiles - target) <= 0.05 * target, (n, tiles, target)
    run_case(dev, worst, f"length{target} n{n}", mixed((n, c, h, w), dev), 64, tiles=tiles)


# --------------------------------------------------------------------------- 2. inputs at config-2 scale
INPUTS = {
    "cond1e2": lambda dev: conditioned_at_scale(CONFIG2, 64, 1e2, dev, seed=1),
    "cond1e4": lambda dev: conditioned_at_scale(CONFIG2, 64, 1e4, dev, seed=2),
    "post_relu": lambda dev: post_relu(CONFIG2, dev, seed=3),
    "mean_50sigma": lambda dev: mean_50sigma(CONFIG2, dev, seed=4),
    "scales_1e-3_1e3": lambda dev: spread_scales(CONFIG2, dev, seed=5),
    "pilot_30sigma": lambda dev: pilot_30sigma(CONFIG2, dev, seed=6),
}


@pytest.mark.parametrize("inp", list(INPUTS))
def test_config2_inputs(inp, dev, sms, worst):
    n, c, h, w = CONFIG2
    run_case(dev, worst, f"config2 {inp}", INPUTS[inp](dev), 64, tiles=tiles_per_cta(sms, n, c, h * w))


# --------------------------------------------------------------------------- 3. every Gram instantiation, at length
@pytest.mark.parametrize("gs", [8, 16, 32])
def test_group_sizes(gs, dev, sms, worst):
    """gs 8 / 16 / 32 at config 2 (gs 64 is test_accumulation_length): the same Gram, other diagonal blocks kept."""
    n, c, h, w = CONFIG2
    run_case(dev, worst, f"config2 gs{gs}", mixed(CONFIG2, dev, seed=gs), gs, tiles=tiles_per_cta(sms, n, c, h * w))


def test_channels_last(dev, sms, worst):
    n, c, h, w = CONFIG2
    run_case(dev, worst, "config2 nhwc", mixed(CONFIG2, dev, seed=7), 64, nhwc=True, tiles=tiles_per_cta(sms, n, c, h * w))


@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
def test_bf16(nhwc, dev, sms, worst):
    """bf16 x at config 2: the statistics bit-identical to the float32 call on the widened values, and against float64
    of those values."""
    n, c, h, w = CONFIG2
    run_case(dev, worst, f"config2 bf16 {'nhwc' if nhwc else 'nchw'}", mixed(CONFIG2, dev, seed=8), 64, nhwc=nhwc,
             bf16=True, tiles=tiles_per_cta(sms, n, c, h * w))


@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
def test_group_size_128(nhwc, dev, sms, worst):
    """gs 128 at config 2: the diagonal blocks from tc_stats, the off-diagonal block from tc_gram_pair, which
    accumulates about half as many tiles per CTA (C / 128 problems)."""
    n, c, h, w = CONFIG2
    pair = tiles_per_cta(sms, n, c, h * w, pair=True)
    assert pair >= 100, pair
    run_case(dev, worst, f"config2 gs128 {'nhwc' if nhwc else 'nchw'}", mixed(CONFIG2, dev, seed=9), 128, nhwc=nhwc,
             tiles=pair)


def test_three_domains(dev, sms, worst):
    """D = 3 on one DomainTripleNorm site, C = 256, 56^2: 3 x 4 problems, a different mean per domain."""
    n, c, h, w = 86, 256, 56, 56
    tiles = tiles_per_cta(sms, n, c, h * w, d=3)
    assert tiles >= 300, tiles
    x = torch.cat([mixed((n, c, h, w), dev, seed=10 + k, shift=2.0 + 0.7 * k) for k in range(3)])
    run_case(dev, worst, "d3 gs64", x, 64, d=3, tiles=tiles)


def test_zca_basis(dev, sms, worst):
    """The ZCA basis (T = 5 Newton-Schulz iterations) at config 2: the same statistics, the other finalize."""
    n, c, h, w = CONFIG2
    run_case(dev, worst, "config2 zca T5", mixed(CONFIG2, dev, seed=11), 64, T=5, tiles=tiles_per_cta(sms, n, c, h * w))


# --------------------------------------------------------------------------- 4. short control
def test_short_control(dev, sms, worst):
    """N * HW = 4096, the fewest samples the tensor-core kernels take (one or two tiles per CTA): it passes under the
    same bounds, so that they are not simply loose.  Also the identity the file reads the covariance through: with
    momentum 1, running_variance and running_mean are the batch statistics bit for bit, whatever the buffers held."""
    import dwt_b200
    shape = (128, 256, 4, 8)
    x = mixed(shape, dev, seed=12)
    run_case(dev, worst, "short m4096", x, 64, tiles=tiles_per_cta(sms, shape[0], shape[1], 32))
    a = dwt_b200.WTransform2d(256, 64, momentum=1.0).to(dev).train()
    b = dwt_b200.WTransform2d(256, 64, momentum=1.0).to(dev).train()
    b.running_mean.normal_()
    b.running_variance.normal_()
    xg = x.detach().requires_grad_(True)
    ya, yb = a(xg), b(xg)
    assert torch.equal(a.running_variance, b.running_variance) and torch.equal(a.running_mean, b.running_mean)
    assert torch.equal(a.running_mean.view(1, -1), ya.grad_fn.saved_tensors[1])
    assert torch.equal(ya, yb)
