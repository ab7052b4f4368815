"""The tensor-core whitening backward (tc_bwd_reduce: R = sum dy xc^T and the row sums of dy, then the coefficient
algebra and tc_bwd_apply) against float64, under output gradients that are not iid randn.

A gradient with a per-channel mean, or one mostly along the output y, is what a real network sends back: the next
layer's bias and affine weights see exactly those directions.  True R does not depend on a per-channel offset of dy
(sum xc = 0), and a dy along y largely cancels in dx; a contraction that rounds dy to tf32 around zero turns both into
error in dx.  So every case runs these gradient families, each built from (x, y, seed):

  randn                   iid, the control
  offset10 / offset100    randn + 10 / 100 sigma per channel, sign and size drawn per (domain, channel)
  aligned0.1 / 0.01       y s + 0.1 / 0.01 randn, s a per-channel scale
  aligned0.1+offset10     both
  relu                    randn where y > 0.52 (about 70 % zeros)
  head                    y -> gamma, beta -> ReLU -> global average pool -> linear -> cross-entropy, differentiated in
                          float64: constant over the pixels of an (image, channel) apart from the ReLU mask

Reference: oracle/torch_port.WTransform2d in float64 on the device (tests/support/zca_reference.zca_torch for the ZCA
basis), one domain and one slab of whole groups at a time, fed the same fp32 (bf16) x and dy the kernels read.  Beside
it, a float32 yardstick: the same operator sequence in float32 on the GPU with TF32 off in cuBLAS and cuDNN (set and
restored here).

Bounds, for every case and family: dx within 1e-3 norm-wise of float64 and 5e-3 max-elementwise (bf16: plus the error of
rounding the float64 dx to bf16, which the kernel's store cannot avoid); and for the structured families, a norm-wise
error no worse than RATIO x the float32 yardstick's or FLOOR, whichever is larger.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), split and centred contraction, the Gram kernel's fresh
accumulator per tile: worst norm-wise dx error of a float32 family 9.7e-5 (config 2, aligned0.01; the yardstick's
8.7e-5; 5.6e-3 while the Gram kept one accumulator per CTA), worst ratio to the yardstick where the error exceeds FLOOR
2.8 (gs 16 at N*HW = 4096, aligned0.01: 3.7e-5 against 1.3e-5; config 2 offset10 was 4.6 before, now 1.1e-6 against
6.5e-6); backward alone at most 2.9e-4 (D = 3, offset100); bf16 1.7e-3, its rounding alone.  The single tf32
pass this replaced failed all 24 tests here other than test_many_tiles_per_cta (not run on it): 6.4e-3 at gs 64 and
N*HW = 4096 (offset100), 1.1e-2 at condition number 1e3, 9.4e-3 at gs 128, 6.3e-2 in bf16.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import zca_reference as Z  # noqa: E402

pytestmark = pytest.mark.gpu

BOUND, BOUND_MAX = 1e-3, 5e-3
RATIO, FLOOR = 15.0, 2e-5
TC_CH = 64                  # channels of a tensor-core super-block
TC_BOX = 32                 # pixels of a TMA box (the contraction's tile)
TC_MIN_M = 4096             # N * HW per domain below which the tiled kernels take the call
SLAB_ELEMS = 1 << 25        # elements of one (domain, channel slab) reference call
FAMILIES = ("randn", "offset10", "offset100", "aligned0.1", "aligned0.01", "aligned0.1+offset10", "relu", "head")


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
    print("\ntensor-core backward, dx against float64 (norm-wise, max-elementwise, (float32 yardstick norm-wise),"
          " [backward alone at the kernels' statistics]):")
    for k in sorted(table):
        print("  %-28s %s" % (k, ", ".join(f"{f} {r:.1e} {m:.1e} ({y:.1e}) [{b:.1e}]" for f, (r, m, y, b) in table[k].items())))


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
        return math.sqrt(self.d2) / max(math.sqrt(self.r2), 1e-300), self.dmax / max(self.rmax, 1e-300)


# --------------------------------------------------------------------------- inputs
def mixed(shape, dev, seed=0, shift=2.0):
    """bench.py's microbench input: x = mix . randn + 2, mix = randn / sqrt(C) + I over all channels."""
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    mix = torch.randn(c, c, device=dev, generator=g) / c ** 0.5 + torch.eye(c, device=dev)
    return (torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, h, w, device=dev, generator=g)) + shift).contiguous()


def conditioned(shape, gs, cond, dev, seed=0):
    """Per-group batch covariance of condition number `cond` exactly, mean 1 (zca_reference.conditioned_input)."""
    n, c, h, w = shape
    return torch.tensor(Z.conditioned_input(np.random.default_rng(seed), n, c, (h, w), gs, cond, shift=1.0),
                        dtype=torch.float32, device=dev)


def make_dy(fam, y, d, seed):
    """The output gradient of family `fam` in float64 for y [d*N, C, H, W] (float64)."""
    g = torch.Generator(device=y.device).manual_seed(seed)
    dn, c = y.shape[:2]
    r = torch.randn(y.shape, dtype=y.dtype, device=y.device, generator=g)
    if fam == "randn":
        return r
    if fam == "relu":
        return r * (y > 0.52)
    if fam == "head":
        gamma = 0.5 + torch.rand(1, c, 1, 1, dtype=y.dtype, device=y.device, generator=g)
        beta = 0.1 * torch.randn(1, c, 1, 1, dtype=y.dtype, device=y.device, generator=g)
        lin = torch.randn(10, c, dtype=y.dtype, device=y.device, generator=g) / c ** 0.5
        labels = torch.randint(0, 10, (dn,), device=y.device, generator=g)
        yg = y.detach().clone().requires_grad_(True)
        logits = torch.relu(yg * gamma + beta).mean((2, 3)) @ lin.T
        (dy,) = torch.autograd.grad(torch.nn.functional.cross_entropy(logits, labels), yg)
        return dy
    out = torch.zeros_like(y)
    if fam.startswith("aligned"):
        sigma = float(fam[len("aligned"):].split("+")[0])
        s = 0.5 + torch.rand(1, c, 1, 1, dtype=y.dtype, device=y.device, generator=g)
        out += y * s + sigma * r
    else:
        out += r
    if "offset" in fam:
        a = float(fam.split("offset")[1])
        sign = torch.where(torch.rand(d, 1, c, 1, 1, device=y.device, generator=g) < 0.5, -1.0, 1.0).to(y.dtype)
        size = 0.5 + torch.rand(d, 1, c, 1, 1, dtype=y.dtype, device=y.device, generator=g)
        out = (out.view(d, dn // d, c, *y.shape[2:]) + a * sign * size).view(y.shape)
    return out


# --------------------------------------------------------------------------- references
def ref_forward(xs, gs, T):
    """The reference forward of one (domain, slab) xs [N, Cs, H, W] in xs's dtype (train mode, batch statistics)."""
    if T:
        return Z.zca_torch(xs, gs, T)[0]
    import oracle.torch_port as port
    cs = xs.shape[1]
    m = port.WTransform2d(cs, gs, running_m=torch.zeros(1, cs, 1, 1, dtype=xs.dtype, device=xs.device),
                          running_var=torch.eye(gs, dtype=xs.dtype, device=xs.device).repeat(cs // gs, 1, 1))
    return m.train()(xs)


def slabs(d, n, c, per_ch, gs):
    slab = max(gs, SLAB_ELEMS // per_ch // gs * gs)
    for di in range(d):
        for c0 in range(0, c, slab):
            yield di, slice(di * n, (di + 1) * n), slice(c0, min(c, c0 + slab))


def fp32_strict():
    """TF32 off in cuBLAS (the reference's bmm) and cuDNN (its grouped 1x1 convolution); returns a restore function."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False

    def restore():
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    return restore


# --------------------------------------------------------------------------- one case
def backward_at(x64, dy64, mean, w, eps=1e-3):
    """oracle.dwt_oracle.whiten_backward's closed form in float64 for one domain [N, C, H, W], at the given statistics
    (mean [C], W [G, gs, gs]): the exact backward of the forward the kernels ran."""
    g, gs = w.shape[:2]
    grp = lambda t: t.transpose(0, 1).reshape(g, gs, -1)                                     # noqa: E731
    xc, gy = grp(x64) - mean.reshape(g, gs, 1), grp(dy64)
    p = torch.tril(-(gy @ xc.mT) @ w.mT)
    p.diagonal(dim1=1, dim2=2).mul_(0.5)
    sm = w.mT @ p @ w
    dx = w.mT @ (gy - gy.mean(-1, keepdim=True)) + (2 * (1 - eps) / xc.shape[-1]) * (0.5 * (sm + sm.mT)) @ xc
    return dx.reshape(x64.shape[1], x64.shape[0], *x64.shape[2:]).transpose(0, 1)


def run_case(dev, worst, label, x, gs, d=1, nhwc=False, bf16=False, T=None, fams=FAMILIES, seed=0):
    """x [d*N, C, H, W] float32 through the kernels (d = 1: the module; d > 1: one DomainTripleNorm site), then one
    backward per gradient family; dx against float64 and the float32 yardstick, domain by domain.  Cholesky basis: also
    dx against the float64 backward at the kernels' own batch statistics (save_mean, save_w), which isolates the
    backward (contraction, coefficients, apply) from the forward's statistics."""
    import dwt_b200
    from dwt_b200 import _native as nv
    dn, c = x.shape[:2]
    n, per_ch = dn // d, dn // d * x[0, 0].numel()
    assert per_ch >= TC_MIN_M and x.shape[2] * x.shape[3] >= TC_BOX
    dt = torch.bfloat16 if bf16 else torch.float32
    xin = x.to(dt)
    x64 = xin.double()
    cl = torch.channels_last if nhwc else torch.contiguous_format
    # float64 forward: the y the gradient families are built from
    y64 = torch.empty_like(x64)
    with torch.no_grad():
        for di, rs, cs in slabs(d, n, c, per_ch, gs):
            y64[rs, cs] = ref_forward(x64[rs, cs], gs, T)
    # kernels
    mods = [(dwt_b200.ZCAWTransform2d(c, gs, iterations=T) if T else dwt_b200.WTransform2d(c, gs)).to(dev).train()
            for _ in range(d)]
    xg = xin.contiguous(memory_format=cl).requires_grad_(True)
    y = mods[0](xg) if d == 1 else dwt_b200.DomainTripleNorm("whiten", c, gs, n_domains=d)(xg, mods, None, None)
    want = "tc_bwd_reduce" + ("_nhwc" if nhwc else "") + ("_bf16" if bf16 else "")
    save_mean, save_w = (t.detach().double() for t in y.grad_fn.saved_tensors[1:3])
    assert save_mean.shape == (d, c) and save_w.shape == (d, c // gs, gs, gs)
    failures = []
    for fi, fam in enumerate(fams):
        dy64 = make_dy(fam, y64, d, seed + 101 * fi)
        dyin = dy64.to(dt).contiguous(memory_format=cl)
        dyref = dyin.double()
        del dy64
        nv.profile_begin()
        (dx,) = torch.autograd.grad(y, xg, dyin, retain_graph=True)
        fam_ran = set(nv.by_family(nv.profile_end()))
        assert want in fam_ran and not any(f.startswith(("tiled", "small", "cl_")) for f in fam_ran), (label, fam, fam_ran)
        err, yard, rnd, bwd = ([_Err() for _ in range(d)] for _ in range(4))
        restore = fp32_strict()
        try:
            for di, rs, cs in slabs(d, n, c, per_ch, gs):
                xs = x64[rs, cs].clone().requires_grad_(True)
                (dxr,) = torch.autograd.grad(ref_forward(xs, gs, T), xs, dyref[rs, cs])
                xs32 = xin[rs, cs].float().requires_grad_(True)
                (dx32,) = torch.autograd.grad(ref_forward(xs32, gs, T), xs32, dyin[rs, cs].float())
                err[di].add(dx[rs, cs], dxr)
                yard[di].add(dx32.to(dt), dxr)
                rnd[di].add(dxr.to(dt), dxr)
                del xs, dxr, xs32, dx32
        finally:
            restore()
        if not T:
            for di in range(d):
                rs = slice(di * n, (di + 1) * n)
                bwd[di].add(dx[rs], backward_at(x64[rs], dyref[rs], save_mean[di], save_w[di]))
        del dx, dyin, dyref
        # the worst domain
        (r, m), ry, (fr, fm) = max(e.both() for e in err), max(e.both()[0] for e in yard), max(e.both() for e in rnd)
        rb = max(e.both()[0] for e in bwd) if not T else float("nan")
        worst.setdefault(label, {})[fam] = (r, m, ry, rb)
        if not bf16:
            fr = fm = 0.0
        if rb > BOUND + fr:
            failures.append(f"{fam}: backward alone norm-wise {rb:.2e} (bound {BOUND + fr:.1e})")
        if r > BOUND + fr or m > BOUND_MAX + fm:
            failures.append(f"{fam}: norm-wise {r:.2e}, max-elementwise {m:.2e} (bounds {BOUND + fr:.1e}, {BOUND_MAX + fm:.1e})")
        elif fam != "randn" and r > max(RATIO * ry, FLOOR + fr):
            failures.append(f"{fam}: norm-wise {r:.2e} > max({RATIO} x float32 yardstick {ry:.2e}, {FLOOR + fr:.1e})")
    assert not failures, f"{label}: " + "; ".join(failures)


# --------------------------------------------------------------------------- 1. group sizes at the routing edge and above
@pytest.mark.parametrize("gs", [8, 16, 32, 64])
@pytest.mark.parametrize("m", [TC_MIN_M, 8 * TC_MIN_M], ids=["m4096", "m32768"])
def test_group_sizes(gs, m, dev, worst):
    """N * HW = 4096 exactly (the fewest samples the tensor-core kernels take: the error of R falls as 1/sqrt(M)) and
    eight times that; condition number 1e2 per group."""
    hw = (4, 8) if m == TC_MIN_M else (16, 16)
    shape = (m // (hw[0] * hw[1]), 64, *hw)
    run_case(dev, worst, f"gs{gs} m{m}", conditioned(shape, gs, 1e2, dev, seed=gs), gs, seed=gs)


@pytest.mark.parametrize("cond", [1.0, 1e2, 1e3])
def test_condition_numbers(cond, dev, worst):
    """gs 64 at N * HW = 4096, C = 128, per-group condition number 1 / 1e2 / 1e3."""
    run_case(dev, worst, f"gs64 cond{cond:g}", conditioned((128, 128, 4, 8), 64, cond, dev, seed=7), 64, seed=3)


# --------------------------------------------------------------------------- 2. partial tiles and super-blocks, domains
@pytest.mark.parametrize("gs,shape", [(64, (114, 64, 6, 6)), (32, (103, 64, 5, 8))], ids=["hw36_gs64", "hw40_gs32"])
def test_partial_pixel_tile(gs, shape, dev, worst):
    """HW 36 / 40: the last 32-pixel tile of every image is partial (TMA zero fill, n_valid of the tile range)."""
    assert shape[2] * shape[3] % TC_BOX != 0
    run_case(dev, worst, f"hw{shape[2] * shape[3]} gs{gs}", conditioned(shape, gs, 1e2, dev, seed=gs + 1), gs, seed=5)


@pytest.mark.parametrize("gs", [16, 32])
def test_partial_super_block(gs, dev, worst):
    """C = 96: the second 64-channel super-block is half past C (rows and columns zero, K = 0 there)."""
    assert 96 % TC_CH != 0
    run_case(dev, worst, f"c96 gs{gs}", conditioned((16, 96, 16, 16), gs, 1e2, dev, seed=gs + 2), gs, seed=6)


def test_three_domains(dev, worst):
    """D = 3 on one DomainTripleNorm site: every domain its own statistics and its own gradient offsets."""
    x = torch.cat([conditioned((32, 128, 8, 16), 32, 1e2, dev, seed=k) + 0.7 * k for k in range(3)])
    run_case(dev, worst, "d3 gs32", x, 32, d=3, seed=8)


# --------------------------------------------------------------------------- 3. full size, layouts, dtypes, gs 128, ZCA
def test_config2_full_size(dev, worst):
    """BASELINE config 2 (N=256 C=256 56^2, gs 64, the microbench input): about 380 tiles per contraction and Gram CTA,
    the production accumulation regime.  Every family is asserted end to end and the backward alone.  With dy along y,
    dx is about 1 / sigma times smaller than dy, so the forward's statistics count as much as the backward: while the
    Gram kernel kept one tensor-core accumulator per CTA, its covariance (3.9e-5 off, test_tc_forward_stats_fp64.py)
    moved dx by 5.6e-4 (sigma 0.1) and 5.6e-3 (sigma 0.01) even through an exact float64 backward; with a fresh
    accumulator per tile dx lands at 9.7e-6 and 9.7e-5 (the float32 yardstick's 7.7e-6 and 8.7e-5).  Before the per-tile
    accumulator of the contraction the backward alone was 6.3e-3 at sigma 0.01 (now 4.2e-5)."""
    run_case(dev, worst, "config2 gs64", mixed((256, 256, 56, 56), dev), 64, seed=9,
             fams=("offset10", "offset100", "aligned0.1", "aligned0.01", "aligned0.1+offset10"))


def test_many_tiles_per_cta(dev, sms, worst):
    """C = 4096 at N * HW = 8192: 64 super-blocks leave tc_chunks = 2 SMs / 64 CTAs per problem, so every contraction
    CTA accumulates tens of tiles (the other moderate-size cases give 1-4)."""
    c, shape = 4096, (32, 4096, 16, 16)
    chunks = max(1, 2 * sms // (c // TC_CH))
    tiles = shape[0] * (shape[2] * shape[3] // TC_BOX)
    assert tiles // chunks >= 32, (tiles, chunks)
    run_case(dev, worst, "c4096 many tiles", conditioned(shape, 64, 1e2, dev, seed=14), 64, seed=14)


@pytest.mark.parametrize("gs", [16, 64])
def test_channels_last(gs, dev, worst):
    run_case(dev, worst, f"nhwc gs{gs}", conditioned((128, 128, 4, 8), gs, 1e2, dev, seed=10), gs, nhwc=True, seed=10)


@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
def test_bf16(nhwc, dev, worst):
    """bf16 x and dy against float64 of the widened values; one offset and one aligned family."""
    run_case(dev, worst, f"bf16 {'nhwc' if nhwc else 'nchw'} gs32", conditioned((64, 128, 8, 8), 32, 1e2, dev, seed=11), 32,
             nhwc=nhwc, bf16=True, fams=("offset100", "aligned0.01"), seed=11)


@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
def test_group_size_128(nhwc, dev, worst):
    """gs 128: the four-block (PAIR) contraction, dy rows and x columns from different super-blocks."""
    run_case(dev, worst, f"gs128 {'nhwc' if nhwc else 'nchw'}", conditioned((128, 256, 4, 8), 128, 1e2, dev, seed=12), 128,
             nhwc=nhwc, seed=12)


def test_zca_basis(dev, worst):
    """dwt_whiten_zca_bwd (T = 5 Newton-Schulz iterations) at gs 64, N * HW = 4096, condition number 1e2."""
    run_case(dev, worst, "zca gs64 T5", conditioned((128, 128, 4, 8), 64, 1e2, dev, seed=13), 64, T=5, seed=13)
