"""The channels-last max-pool (csrc/pool.cu) and the paired augmentation (csrc/augment.cu) against exact references, at
every launch branch and at the input edges where such kernels go wrong.

Max-pool reference: torch's CPU F.max_pool2d in float32 on the same NCHW data.  It fixes the semantics the kernels
promise: the first maximum in row-major window order over the window's in-image elements, a NaN always taking over (so
the last NaN of a window is kept), and a backward that adds each window's gradient into its argmax in ascending (oh, ow)
order, the kernels' order.  Forward values (bit for bit, the sign of zero included), argmax positions and float32
gradients must therefore be identical.  The gradients are also held to an fp64 scatter-add of the same upstream
gradients, a bound that does not depend on the order of the sums.  bf16 calls are held to the float32 CPU result on the
widened input and gradient, rounded once to nearest-even (the rule of pool.cu's header).  torch's CUDA kernels are not a
reference here: they are another implementation.

Each case names the forward and backward kernels it targets; pool_branches() restates the launch conditions of
maxpool_fwd / maxpool_bwd in pool.cu and checks the label, and test_pool_branch_helper_mirrors_pool_cu pins the restated
conditions to the source text.  The launch profile (one maxpool_fwd[_bf16] and one maxpool_bwd[_bf16] launch) cannot tell
the kernels apart.

Augmentation reference: tests/golden/augment_edges.npz, written by the unmodified reference functions and torchvision
(tests/golden/make_golden_augment_edges.py), and the numpy oracle (oracle/augment_oracle.py) that the CPU part pins to
that fixture.  The bar is equality: the warp is fixed-point and every float step is correctly rounded.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POOL_CU = os.path.join(ROOT, "dwt-domain-adaptation_b200", "dwt_b200", "csrc", "pool.cu")
EDGES = os.path.join(ROOT, "tests", "golden", "augment_edges.npz")
CL = torch.channels_last
BF = torch.bfloat16
gpu = pytest.mark.gpu
GRID_Y = 65535
U32 = 2.0 ** -24
KINDS = ("ties", "neginf", "posinf", "nan", "signed_zero", "constant", "subnormal", "bf16_ties")


# --------------------------------------------------------------------------- max-pool: launch branches
def pool_branches(n, c, h, w, k, s, p):
    """(forward kernel, backward kernel) that maxpool_fwd / maxpool_bwd in csrc/pool.cu launch for this call:
    "3s2" the stem's patch kernel, "fixed" the row kernel compiled for (3, 2, 1), "generic" the row kernel."""
    oh = (h + 2 * p - k) // s + 1
    c4 = c // 4
    stem = (k, s, p) == (3, 2, 1) and c4 & (c4 - 1) == 0
    fwd = "3s2" if stem and h % 4 == 0 and w % 4 == 0 and n * (oh // 2) <= GRID_Y else "fixed" if stem else "generic"
    bwd = "3s2" if stem and h % 2 == 0 and w % 2 == 0 and n * (h // 2) <= GRID_Y else "fixed" if stem else "generic"
    return fwd, bwd


def _gk(k, s, p, n, c, h, w):
    return ("generic", "generic", n, c, h, w, k, s, p)


# (forward kernel, backward kernel, N, C, H, W, k, s, p)
POOL_CASES = [
    # the stem patch kernels both ways; C/4 = 1, 2, 16, 256; wide rows take several CTAs in x
    ("3s2", "3s2", 1, 4, 4, 4, 3, 2, 1), ("3s2", "3s2", 2, 8, 8, 12, 3, 2, 1), ("3s2", "3s2", 3, 64, 12, 16, 3, 2, 1),
    ("3s2", "3s2", 2, 64, 8, 128, 3, 2, 1), ("3s2", "3s2", 1, 1024, 4, 8, 3, 2, 1),
    # one direction on the patch kernel: H = 10, W % 4 == 2, H % 4 == 2 both; odd H (and odd both) on neither
    ("fixed", "3s2", 2, 16, 10, 8, 3, 2, 1), ("fixed", "3s2", 2, 8, 12, 10, 3, 2, 1), ("fixed", "3s2", 2, 8, 6, 6, 3, 2, 1),
    ("fixed", "fixed", 2, 16, 9, 8, 3, 2, 1), ("fixed", "fixed", 3, 8, 9, 7, 3, 2, 1),
    # the grid-y limit: N * (OH/2) forward, N * (H/2) backward, each at, just past and far past 65535
    ("3s2", "3s2", 32767, 4, 4, 4, 3, 2, 1), ("3s2", "fixed", 32768, 4, 4, 4, 3, 2, 1),
    ("3s2", "fixed", 65535, 4, 4, 4, 3, 2, 1), ("fixed", "fixed", 65536, 4, 4, 4, 3, 2, 1),
    # C/4 not a power of two at (3, 2, 1), H % 4 == 0 included
    ("generic", "generic", 2, 12, 8, 8, 3, 2, 1), ("generic", "generic", 2, 24, 16, 12, 3, 2, 1),
    # every window size up to 15 (argmax codes up to 224)
    _gk(1, 1, 0, 2, 8, 5, 6), _gk(2, 1, 1, 2, 8, 7, 6), _gk(3, 1, 0, 2, 4, 9, 11), _gk(4, 2, 2, 1, 8, 10, 9),
    _gk(5, 3, 2, 1, 12, 7, 7), _gk(6, 2, 3, 1, 4, 13, 12), _gk(7, 2, 3, 1, 8, 15, 9), _gk(8, 3, 4, 1, 4, 16, 17),
    _gk(9, 2, 4, 1, 4, 12, 20), _gk(10, 4, 5, 1, 8, 21, 14), _gk(11, 3, 5, 1, 4, 17, 19), _gk(12, 5, 6, 1, 4, 12, 24),
    _gk(13, 2, 6, 1, 8, 20, 13), _gk(14, 5, 7, 1, 4, 14, 22), _gk(15, 4, 7, 1, 4, 30, 15),
    # even k with p = k/2; stride beyond the window (pixels in no window); k = 15 at stride 1 (225 addends per pixel)
    _gk(2, 2, 1, 2, 8, 7, 9), _gk(4, 3, 2, 1, 8, 9, 8), _gk(14, 4, 7, 1, 4, 15, 16),
    _gk(2, 3, 0, 2, 8, 11, 10), _gk(3, 5, 1, 1, 12, 13, 12), _gk(1, 2, 0, 2, 4, 7, 6), _gk(5, 7, 2, 1, 8, 16, 19),
    _gk(15, 1, 7, 1, 8, 17, 17),
    # one output row or column (H or W = k - 2p), and H = W = 1
    _gk(5, 2, 1, 2, 8, 3, 9), _gk(7, 1, 3, 1, 4, 6, 1), _gk(9, 2, 3, 1, 4, 3, 3), _gk(1, 1, 0, 3, 8, 1, 1),
    _gk(2, 1, 1, 2, 4, 1, 1), ("fixed", "fixed", 2, 8, 1, 1, 3, 2, 1),
    # wide rows: OW * C/4 (forward) and W * C/4 (backward) well past 256 threads, C/4 a power of two and not
    _gk(2, 2, 0, 2, 64, 4, 64), _gk(3, 1, 1, 1, 100, 3, 40), ("fixed", "3s2", 1, 256, 10, 16, 3, 2, 1),
    ("fixed", "fixed", 1, 512, 5, 10, 3, 2, 1),
]


def _case_id(cs):
    f, b, n, c, h, w, k, s, p = cs
    return f"{f}-{b}-N{n}C{c}H{h}W{w}-k{k}s{s}p{p}"


# --------------------------------------------------------------------------- max-pool: inputs and the reference
def _planes(n, c):
    return ((torch.arange(n)[:, None] * c + torch.arange(c)[None]))[:, :, None, None]


def pool_input(kind, n, c, h, w, k, gen):
    """float32 NCHW CPU input of one kind; every value is exact in bf16 except where the kind is about bf16 rounding."""
    shape = (n, c, h, w)
    hh = torch.arange(h)[:, None].expand(h, w)
    ww = torch.arange(w)[None, :].expand(h, w)
    q = _planes(n, c).expand(shape)
    rnd = torch.rand(shape, generator=gen)
    base = torch.randn(shape, generator=gen).to(BF).float()
    inf, nan = float("inf"), float("nan")
    if kind == "ties":                     # post-ReLU: windows of zeros
        return torch.relu(base)
    if kind == "neginf":                   # planes of -inf with finite blocks, -inf borders, corners and halves
        keep = [torch.zeros(h, w, dtype=torch.bool), (hh >= h - 2) & (ww >= w - 2), (hh == 0) & (ww == 0),
                (hh >= k) & (hh < h - k) & (ww >= k) & (ww < w - k), None, (hh == h // 2) | (ww == w // 2),
                ww >= w // 2, hh >= h // 2, (hh >= h - 1) | (ww >= w - 1), hh + ww == h + w - 2]
        m = torch.zeros(shape, dtype=torch.bool)
        for i, kp in enumerate(keep):
            m |= (q % len(keep) == i) & (rnd > 0.8 if kp is None else kp)
        return torch.where(m, base, -inf)
    if kind == "posinf":
        return torch.where(rnd < 0.1, inf, torch.where(rnd > 0.9, -inf, base))
    if kind == "nan":                      # NaN on the borders, NaN blocks in the corner, several NaNs in one window
        border = [hh == 0, ww == 0, hh == h - 1, ww == w - 1, (hh < 3) & (ww < 3), None]
        m = torch.zeros(shape, dtype=torch.bool)
        for i, b in enumerate(border):
            m |= (q % len(border) == i) & (rnd < 0.3 if b is None else b)
        return torch.where(m, nan, torch.relu(base))
    if kind == "signed_zero":              # +0 / -0 ties under negative values: -0 must not displace +0 nor the reverse
        return torch.where(rnd < 0.2, -1.0, torch.where(rnd < 0.6, -0.0, 0.0))
    if kind == "constant":
        return torch.full(shape, 0.75) * torch.where(q % 2 == 0, 1.0, -1.0)
    if kind == "subnormal":                # multiples of 2^-133: subnormal in float32 and in bf16
        return torch.randint(-100, 101, shape, generator=gen).float() * 2.0 ** -133
    if kind == "bf16_ties":                # distinct in float32, equal once rounded to bf16 (ulp 2^-7 at 1)
        scale = 2.0 ** torch.randint(-3, 4, shape, generator=gen).float()
        return (1 + torch.randint(0, 4, shape, generator=gen).float() * 2.0 ** -10) * scale
    raise ValueError(kind)


def pool_grad(n, c, oh, ow, gen):
    """Upstream gradient over six decades, so that the order of each pixel's sum shows in its float32 bits."""
    g = torch.randn(n, c, oh, ow, generator=gen) * 2.0 ** torch.randint(-10, 11, (n, c, oh, ow), generator=gen).float()
    return g.to(BF).float()


def pool_reference(x32, dy32, k, s, p):
    """torch CPU float32: (y, flat in-plane argmax h*W+w, dx), and the fp64 sum of each pixel's gradients with the
    float32 bound of summing them in any order."""
    xr = x32.clone().requires_grad_(True)
    y, idx = Fn.max_pool2d(xr, k, s, p, return_indices=True)
    y.backward(dy32)
    n, c, h, w = x32.shape
    plane = (torch.arange(n * c) * (h * w)).view(n, c, 1, 1)
    flat = (idx + plane).reshape(-1)
    dx64 = torch.zeros(n * c * h * w, dtype=torch.float64).index_add_(0, flat, dy32.double().reshape(-1))
    mag = torch.zeros_like(dx64).index_add_(0, flat, dy32.double().abs().reshape(-1))
    cnt = torch.zeros_like(dx64).index_add_(0, flat, torch.ones(flat.numel(), dtype=torch.float64))
    return y.detach(), idx, xr.grad, dx64.view(x32.shape), (cnt * U32 * mag).view(x32.shape)


def _bits(t):
    """Integer view of a float tensor, every NaN mapped to one pattern: equality of these is equality bit for bit."""
    t = t.detach().cpu().contiguous()
    iv = t.view(torch.int32 if t.dtype == torch.float32 else torch.int16).long()
    return torch.where(t.isnan(), -1, iv)


def _codes_to_flat(codes, n, c, oh, ow, h, w, k, s, p):
    """The kernels' window-local argmax bytes (NHWC order) -> in-plane positions h*W + w (NCHW order)."""
    cd = codes.view(n, oh, ow, c).permute(0, 3, 1, 2).long().cpu()
    rows = torch.arange(oh).view(1, 1, oh, 1) * s - p + cd // k
    cols = torch.arange(ow).view(1, 1, 1, ow) * s - p + cd % k
    return rows * w + cols


# --------------------------------------------------------------------------- max-pool: CPU part
def test_pool_branch_helper_mirrors_pool_cu():
    """pool_branches() restates the launch conditions of maxpool_fwd / maxpool_bwd; if pool.cu's dispatch changes, the
    labels of POOL_CASES must be revisited."""
    src = open(POOL_CU).read()
    assert "k == 3 && s == 2 && p == 1 && sh >= 0 && H % 4 == 0 && W % 4 == 0 && (long long)N * (OH / 2) <= 65535" in src
    assert "k == 3 && s == 2 && p == 1 && sh >= 0 && H % 2 == 0 && W % 2 == 0 && (long long)N * (H / 2) <= 65535" in src
    assert src.count("else if (k == 3 && s == 2 && p == 1 && sh >= 0) maxpool_") == 2
    assert "int pow2_shift(int v)" in src


def test_pool_cases_cover_every_branch():
    for cs in POOL_CASES:
        assert pool_branches(*cs[2:]) == cs[:2], _case_id(cs)
    pairs = {cs[:2] for cs in POOL_CASES}
    assert {("3s2", "3s2"), ("fixed", "3s2"), ("3s2", "fixed"), ("fixed", "fixed"), ("generic", "generic")} <= pairs
    ks = {cs[6] for cs in POOL_CASES}
    assert ks == set(range(1, 16))
    assert any(cs[7] > cs[6] for cs in POOL_CASES)                                     # stride beyond the window
    assert any(cs[6] % 2 == 0 and 2 * cs[8] == cs[6] for cs in POOL_CASES)             # even k, p = k/2
    assert any(cs[4] + 2 * cs[8] == cs[6] for cs in POOL_CASES) and any(cs[5] + 2 * cs[8] == cs[6] for cs in POOL_CASES)
    def fwd_items(cs):                                       # threads one forward CTA row needs (256 per CTA)
        ow = (cs[5] + 2 * cs[8] - cs[6]) // cs[7] + 1
        return (ow // 2 if cs[0] == "3s2" else ow) * (cs[3] // 4)
    for br in ("3s2", "fixed", "generic"):
        assert any(cs[0] == br and fwd_items(cs) > 256 for cs in POOL_CASES), br
        assert any(cs[1] == br and cs[5] * cs[3] // 4 > 256 for cs in POOL_CASES), br
    assert any(cs[0] == "generic" and (cs[3] // 4) & (cs[3] // 4 - 1) and fwd_items(cs) > 256 for cs in POOL_CASES)


@pytest.mark.parametrize("kind", KINDS)
def test_pool_reference_semantics(kind):
    """The CPU reference has the rule the kernels claim: the argmax is the first in-image maximum in row-major order, a
    NaN takes over from anything (the last NaN is kept), ties keep the first element; and its float32 gradient is the
    sequential ascending (oh, ow) sum.  Checked against a direct Python loop at one small geometry with padding."""
    gen = torch.Generator().manual_seed(5)
    n, c, h, w, k, s, p = 1, 8, 6, 7, 3, 2, 1
    x = pool_input(kind, n, c, h, w, k, gen)
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    dy = pool_grad(n, c, oh, ow, gen)
    y, idx, dx, dx64, bound = pool_reference(x, dy, k, s, p)
    want = torch.zeros(n, c, h, w)
    for ch in range(c):
        for i in range(oh):
            for j in range(ow):
                best, arg = None, None
                for a in range(max(0, i * s - p), min(h, i * s - p + k)):
                    for b in range(max(0, j * s - p), min(w, j * s - p + k)):
                        v = x[0, ch, a, b].item()
                        if arg is None or v > best or v != v:
                            best, arg = v, (a, b)
                assert idx[0, ch, i, j].item() == arg[0] * w + arg[1]
                assert _bits(y[0, ch, i, j].reshape(1)).item() == _bits(torch.tensor([best])).item()
                want[0, ch, arg[0], arg[1]] += dy[0, ch, i, j]
    assert torch.equal(_bits(dx), _bits(want))
    assert ((dx.double() - dx64).abs() <= bound).all()


# --------------------------------------------------------------------------- max-pool: C ABI refusals (CPU)
_FAKE = 1 << 20        # never dereferenced: every call below is refused before a launch


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


def _pool(lib, fn, n=2, h=8, w=8, c=8, k=3, s=2, p=1, flags=0, a=_FAKE, b=_FAKE, idx=_FAKE):
    call = lib.dwt_maxpool_fwd if fn == "fwd" else lib.dwt_maxpool_bwd
    vp = lambda v: None if v is None else ctypes.c_void_p(v)        # noqa: E731
    if fn == "fwd":
        return call(vp(a), vp(b), vp(idx), n, h, w, c, k, s, p, flags, None)
    return call(vp(a), vp(idx), vp(b), n, h, w, c, k, s, p, flags, None)


@pytest.mark.parametrize("fn", ["fwd", "bwd"])
@pytest.mark.parametrize("kw, code, text", [
    (dict(k=16, p=0), -1, b"k <= 15"), (dict(k=0, p=0), -1, b"bad pooling window"), (dict(s=0), -1, b"bad pooling window"),
    (dict(p=-1), -1, b"bad pooling window"), (dict(k=3, p=2), -1, b"pad <= k/2"), (dict(k=15, p=8), -1, b"pad <= k/2"),
    (dict(c=6), -1, b"multiple of 4"), (dict(c=0), -1, b"bad pooling input"), (dict(n=0), -1, b"bad pooling input"),
    (dict(h=0), -1, b"bad pooling input"), (dict(h=1, k=5, p=1), -1, b"larger than the padded image"),
    (dict(w=2, k=7, p=2), -1, b"larger than the padded image"),
    (dict(n=1 << 20, h=1024, w=1024, c=4), -4, b"too large"),
    (dict(flags=1), -1, b"bad flags"), (dict(flags=0x100), -1, b"bad flags"), (dict(flags=0x300), -1, b"bad flags"),
    (dict(a=None), -1, b"null pointer"), (dict(b=None), -1, b"null pointer"), (dict(idx=None), -1, b"null pointer"),
    (dict(idx=_FAKE + 2), -1, b"aligned"), (dict(a=_FAKE + 4), -1, b"16-byte aligned"),
    (dict(b=_FAKE + 8), -1, b"16-byte aligned"), (dict(a=_FAKE + 4, flags=0x200), -1, b"8-byte aligned (bf16)"),
    (dict(b=_FAKE + 2, flags=0x200), -1, b"8-byte aligned (bf16)"),
])
def test_maxpool_c_abi_refusals(lib, fn, kw, code, text):
    assert _pool(lib, fn, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


def _aug(lib, B=4, sh=8, sw=8, crop=4, plain=_FAKE, out_aug=_FAKE, cp=_FAKE, ca=_FAKE, flip=_FAKE, aff=_FAKE,
         layout=0, std=(0.2, 0.2, 0.2)):
    vp = lambda v: None if v is None else ctypes.c_void_p(v)        # noqa: E731
    mean, sd = (ctypes.c_float * 3)(0.5, 0.5, 0.5), (ctypes.c_float * 3)(*std)
    return lib.dwt_augment_pair(vp(_FAKE), B, sh, sw, crop, vp(cp), vp(ca), vp(flip), vp(aff), mean, sd, vp(plain),
                                vp(out_aug), layout, None)


@pytest.mark.parametrize("kw, text", [
    (dict(B=65536), b"bad image batch"), (dict(B=0), b"bad image batch"), (dict(sh=16385, crop=4), b"bad image batch"),
    (dict(crop=9), b"does not fit"), (dict(sh=6, sw=10, crop=7), b"does not fit"), (dict(crop=0), b"does not fit"),
    (dict(layout=1), b"layout"), (dict(std=(0.2, 0.0, 0.2)), b"non-zero"), (dict(plain=None, out_aug=None), b"at least one"),
    (dict(cp=None), b"needs crop_plain"), (dict(flip=None), b"needs crop_aug, flip and affine"),
    (dict(aff=None), b"needs crop_aug, flip and affine"),
])
def test_augment_c_abi_refusals(lib, kw, text):
    """B is the launch's grid.y: 65535 is the last batch one launch takes (the GPU part runs it)."""
    assert _aug(lib, **kw) == -1
    assert text in lib.dwt_last_error(), lib.dwt_last_error()


# --------------------------------------------------------------------------- augmentation: oracle vs fixture (CPU)
def _edges():
    z = np.load(EDGES)
    return z, [str(c) for c in z["cases"]]


EDGE_CASES = _edges()[1]


def test_edge_fixture_covers_the_edges():
    """The fixture holds what its generator promises: both translation signs up to the crop, negative determinants,
    exactly singular and near-singular matrices, x4 / x0.25 zooms, non-square sources, crop = source and crop = 1,
    all four crop corners with and without flip, saturated images."""
    z, names = _edges()
    aff = np.concatenate([z[f"{c}/affine"] for c in names])
    crop_of = {c: int(z[f"{c}/crop"]) for c in names}
    det = aff[:, 0, 0].astype(np.float64) * aff[:, 1, 1] - aff[:, 0, 1].astype(np.float64) * aff[:, 1, 0]
    assert (aff[:, :, 2] >= 16).any() and (aff[:, :, 2] <= -16).any() and (det < 0).any() and (det == 0).sum() >= 3
    assert ((np.abs(det) > 0) & (np.abs(det) < 0.01)).sum() >= 2
    assert (np.abs(aff[:, 0, 0]) == 4).any() and (np.abs(aff[:, 0, 0]) == 0.25).any()
    shapes = {c: z[f"{c}/images"].shape for c in names}
    assert any(s[1] != s[2] for s in shapes.values())
    assert any(s[1] == s[2] == crop_of[c] for c, s in shapes.items()) and 1 in crop_of.values()
    cz = z["corners/crop_aug"]
    sh, sw, cr = shapes["corners"][1], shapes["corners"][2], crop_of["corners"]
    corners = {(int(t), int(l), int(f)) for (t, l), f in zip(cz, z["corners/flip"])}
    assert corners == {(t, l, f) for t in (0, sh - cr) for l in (0, sw - cr) for f in (0, 1)}
    im = z["saturated/images"]
    assert (im[0] == 0).all() and (im[1] == 255).all()
    assert str(z["versions"][0]).startswith("cv2 ") and str(z["versions"][1]).startswith("torch ")


@pytest.mark.parametrize("case", EDGE_CASES)
def test_augment_oracle_is_bit_exact_vs_edge_fixture(case):
    from oracle import augment_oracle as A
    z, _ = _edges()
    g = lambda k: z[f"{case}/{k}"]                                  # noqa: E731
    plain, aug = A.paired(g("images"), g("crop_plain"), g("crop_aug"), g("flip"), g("affine"), int(g("crop")))
    assert plain.dtype == aug.dtype == np.float32
    assert np.array_equal(plain, g("plain")) and np.array_equal(aug, g("aug"))


# --------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


def _run_pool(x, dy, k, s, p):
    """MaxPool2d forward + backward through autograd, profiled -> (y, argmax bytes, dx, launches per family)."""
    import dwt_b200
    from dwt_b200 import _native as nv
    xr = x.clone().requires_grad_(True)
    nv.profile_begin()
    y = dwt_b200.MaxPool2d(k, s, p)(xr)
    codes = y.grad_fn.saved_tensors[0].clone()
    y.backward(dy)
    fams = {f: v["launches"] for f, v in nv.by_family(nv.profile_end()).items()}
    return y.detach(), codes, xr.grad, fams


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("case", POOL_CASES, ids=[_case_id(cs) for cs in POOL_CASES])
def test_maxpool_exact(case, dtype, dev):
    fwd, bwd, n, c, h, w, k, s, p = case
    assert pool_branches(n, c, h, w, k, s, p) == (fwd, bwd)
    from dwt_b200 import _native as nv
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    sfx = "_bf16" if dtype == BF else ""
    gen = torch.Generator().manual_seed(n * 7919 + c * 31 + h * 17 + w * 13 + k * 5 + s * 3 + p)
    kinds = KINDS if n * c * h * w <= (1 << 21) else ("ties", "neginf", "nan")
    failures = []
    for kind in kinds:
        x32 = pool_input(kind, n, c, h, w, k, gen)
        dy32 = pool_grad(n, c, oh, ow, gen)
        x_dev, dy_dev = x32.to(dtype), dy32.to(dtype)
        y_ref, idx_ref, dx_ref, dx64, bound = pool_reference(x_dev.float(), dy_dev.float(), k, s, p)
        y, codes, dx, fams = _run_pool(x_dev.to(dev).contiguous(memory_format=CL), dy_dev.to(dev).contiguous(memory_format=CL), k, s, p)
        assert fams == {"maxpool_fwd" + sfx: 1, "maxpool_bwd" + sfx: 1}, fams
        assert y.dtype == dx.dtype == dtype and y.is_contiguous(memory_format=CL) and dx.is_contiguous(memory_format=CL)
        checks = dict(values=torch.equal(_bits(y), _bits(y_ref.to(dtype))),
                      argmax=torch.equal(_codes_to_flat(codes, n, c, oh, ow, h, w, k, s, p), idx_ref),
                      grad=torch.equal(_bits(dx), _bits(dx_ref.to(dtype))))
        tol = bound + (2.0 ** -8 * (dx64.abs() + bound) if dtype == BF else 0.0)      # bf16: one more rounding
        checks["grad_fp64"] = bool(((dx.double().cpu() - dx64).abs() <= tol).all())
        bad = [name for name, ok in checks.items() if not ok]
        if bad:
            lost = (dx_ref.to(dtype).float() - dx.float().cpu()).abs().sum().item()
            failures.append(f"{kind}: {bad} (gradient mass lost or moved {lost:.3g})")
    assert nv.status_all(dev) == 0
    assert not failures, failures


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_maxpool_neginf_border_windows(dtype, dev):
    """The documented example: a -inf plane with a 2x2 block of 1.0 at the bottom right, pooled 3/2/1.  The top-left
    windows hold nothing but -inf; ATen gives their argmax to the first in-image element, (0,0), (0,1) and (1,0), and
    their gradients with it."""
    x = torch.full((1, 4, 4, 4), float("-inf"))
    x[:, :, 2:, 2:] = 1.0
    y_ref, idx_ref, dx_ref, _, _ = pool_reference(x, torch.ones(1, 4, 2, 2), 3, 2, 1)
    assert idx_ref[0, 0].tolist() == [[0, 1], [4, 10]]
    for n, c, h, w in ((1, 4, 4, 4), (1, 12, 4, 4), (1, 4, 6, 6)):               # the 3s2, generic and fixed forwards
        xx = torch.full((n, c, h, w), float("-inf"))
        xx[:, :, h - 2:, w - 2:] = 1.0
        oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        y_ref, idx_ref, dx_ref, _, _ = pool_reference(xx, torch.ones(n, c, oh, ow), 3, 2, 1)
        y, codes, dx, _ = _run_pool(xx.to(dtype).to(dev).contiguous(memory_format=CL),
                                    torch.ones(n, c, oh, ow, dtype=dtype, device=dev).contiguous(memory_format=CL), 3, 2, 1)
        assert torch.equal(_codes_to_flat(codes, n, c, oh, ow, h, w, 3, 2, 1), idx_ref), (n, c, h, w)
        assert torch.equal(dx.float().cpu(), dx_ref), (n, c, h, w, pool_branches(n, c, h, w, 3, 2, 1))


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_maxpool_strided_and_misaligned(dtype, dev):
    """Upstream gradients that are not dense channels-last (copied by the wrapper) or dense at an odd offset (cloned:
    the caller of backward() cannot avoid them) give the aligned call's gradient; an input at an odd offset is refused."""
    import dwt_b200
    from dwt_b200 import _native as nv
    gen = torch.Generator().manual_seed(3)
    n, c, h, w, k, s, p = 2, 16, 12, 10, 3, 2, 1
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    x = pool_input("ties", n, c, h, w, k, gen).to(dtype).to(dev).contiguous(memory_format=CL)
    dy = pool_grad(n, c, oh, ow, gen).to(dtype).to(dev)
    _, _, want, _ = _run_pool(x, dy.contiguous(memory_format=CL), k, s, p)
    wide = torch.zeros(n, c, oh, 2 * ow, dtype=dtype, device=dev)
    wide[..., ::2] = dy
    flat = torch.zeros(dy.numel() + 8, dtype=dtype, device=dev)
    odd = flat[1:1 + dy.numel()].view(n, oh, ow, c).permute(0, 3, 1, 2)
    odd.copy_(dy)
    assert odd.is_contiguous(memory_format=CL) and odd.data_ptr() % (8 if dtype == BF else 16)
    for g in (dy.contiguous(), wide[..., ::2], odd):
        _, _, got, _ = _run_pool(x, g, k, s, p)
        assert torch.equal(_bits(got), _bits(want))
    xflat = torch.zeros(x.numel() + 8, dtype=dtype, device=dev)
    xodd = xflat[1:1 + x.numel()].view(n, h, w, c).permute(0, 3, 1, 2)
    xodd.copy_(x)
    assert xodd.is_contiguous(memory_format=CL)
    with pytest.raises(nv.NativeError, match="aligned"):
        dwt_b200.MaxPool2d(k, s, p)(xodd)
    torch.cuda.synchronize(dev)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape, ksp", [((4, 64, 56, 56), (3, 2, 1)), ((3, 12, 9, 10), (5, 1, 2))], ids=["3s2", "generic"])
def test_maxpool_reruns_and_graph_replay(shape, ksp, dtype, dev):
    """Bit-identical reruns (gathers, no atomics) and a CUDA-graph replay equal to the eager call."""
    import dwt_b200
    from dwt_b200 import _native as nv
    k, s, p = ksp
    gen = torch.Generator(device=dev).manual_seed(11)
    x = torch.relu(torch.randn(*shape, device=dev, generator=gen)).to(dtype).contiguous(memory_format=CL).requires_grad_(True)
    oh, ow = (shape[2] + 2 * p - k) // s + 1, (shape[3] + 2 * p - k) // s + 1
    dy = torch.randn(shape[0], shape[1], oh, ow, device=dev, generator=gen).to(dtype).contiguous(memory_format=CL)
    pool = dwt_b200.MaxPool2d(k, s, p)

    def step():
        y = pool(x)
        return y, torch.autograd.grad(y, x, dy)[0]

    y0, dx0 = (t.detach().clone() for t in step())
    for _ in range(2):
        y1, dx1 = step()
        assert torch.equal(_bits(y1), _bits(y0)) and torch.equal(_bits(dx1), _bits(dx0))
    del y1, dx1
    torch.cuda.synchronize(dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y_g, dx_g = step()
    g.replay()
    torch.cuda.synchronize(dev)
    assert torch.equal(_bits(y_g), _bits(y0)) and torch.equal(_bits(dx_g), _bits(dx0))
    assert nv.status_all(dev) == 0


# --------------------------------------------------------------------------- augmentation (GPU)
def _params(d, dev):
    return {k: torch.as_tensor(np.asarray(d[k])).to(dev) for k in ("crop_plain", "crop_aug", "flip", "affine")}


@gpu
@pytest.mark.parametrize("channels_last", [False, True], ids=["nchw", "nhwc"])
@pytest.mark.parametrize("case", EDGE_CASES)
def test_augment_is_bit_exact_vs_edge_fixture(case, channels_last, dev):
    from dwt_b200 import PairedAugment
    z, _ = _edges()
    g = lambda k: z[f"{case}/{k}"]                                  # noqa: E731
    plain, aug = PairedAugment(crop=int(g("crop")))(torch.tensor(g("images"), device=dev), channels_last=channels_last,
                                                     **_params({k: g(k) for k in ("crop_plain", "crop_aug", "flip", "affine")}, dev))
    fmt = CL if channels_last else torch.contiguous_format
    assert plain.is_contiguous(memory_format=fmt) and aug.is_contiguous(memory_format=fmt)
    assert np.array_equal(plain.cpu().numpy(), g("plain")) and np.array_equal(aug.cpu().numpy(), g("aug"))


@gpu
def test_augment_random_sweep_vs_oracle(dev):
    """300 seeded draw_params batches at affine sigmas 0.1 (the reference's), 0.35 and 1.0 (reflections, near-singular
    matrices), over three source / crop geometries and both layouts, against the oracle."""
    from dwt_b200 import PairedAugment, draw_params
    from oracle import augment_oracle as A
    rng = np.random.default_rng(2024)
    geoms = [(33, 24), (9, 7), (16, 16)]
    done = 0
    for sigma in (0.1, 0.35, 1.0):
        for i in range(100):
            src, crop = geoms[i % 3]
            B = 1 + i % 5
            images = rng.integers(0, 256, (B, src, src, 3), dtype=np.uint8)
            if i % 7 == 0:
                images[:, : src // 3] = 255 * (i % 2)
            p = draw_params(B, src, crop, rng, affine_sigma=sigma)
            plain, aug = PairedAugment(crop=crop)(torch.tensor(images, device=dev), channels_last=bool(i % 2), **_params(p, dev))
            o_plain, o_aug = A.paired(images, p["crop_plain"].numpy(), p["crop_aug"].numpy(), p["flip"].numpy(),
                                      p["affine"].numpy(), crop)
            assert np.array_equal(plain.cpu().numpy(), o_plain), (sigma, i)
            assert np.array_equal(aug.cpu().numpy(), o_aug), (sigma, i, p["affine"].numpy())
            done += 1
    assert done == 300


@gpu
def test_augment_grid_y_edge(dev):
    """B = 65535 (the launch's grid.y, the largest batch the C ABI takes) at a 2x2 crop of 3x4 sources, both views, and
    the plain view alone (want_aug=False) into a slice of a larger buffer that must stay untouched around it."""
    from dwt_b200 import PairedAugment
    from oracle import augment_oracle as A
    rng = np.random.default_rng(65535)
    B, sh, sw, crop = GRID_Y, 3, 4, 2
    images = rng.integers(0, 256, (B, sh, sw, 3), dtype=np.uint8)
    cp = np.stack([rng.integers(0, sh - crop + 1, B), rng.integers(0, sw - crop + 1, B)], 1).astype(np.int32)
    ca = np.stack([rng.integers(0, sh - crop + 1, B), rng.integers(0, sw - crop + 1, B)], 1).astype(np.int32)
    flip = (rng.random(B) < 0.5).astype(np.uint8)
    aff = np.zeros((B, 2, 3), np.float32)
    aff[:, 0, 0], aff[:, 1, 1] = 1 + rng.normal(0, 0.3, B), 1 + rng.normal(0, 0.3, B)
    aff[:, 0, 1], aff[:, 1, 0] = rng.normal(0, 0.3, B), rng.normal(0, 0.3, B)
    aff[:, :, 2] = rng.normal(0, 0.6, (B, 2))
    imgs = torch.tensor(images, device=dev)
    params = _params(dict(crop_plain=cp, crop_aug=ca, flip=flip, affine=aff), dev)
    plain, aug = PairedAugment(crop=crop)(imgs, **params)
    o_plain, o_aug = A.paired(images, cp, ca, flip, aff, crop)
    assert np.array_equal(plain.cpu().numpy(), o_plain) and np.array_equal(aug.cpu().numpy(), o_aug)
    buf = torch.full((B + 2, 3, crop, crop), 7.0, device=dev)
    plain2, none = PairedAugment(crop=crop)(imgs, crop_plain=params["crop_plain"], out_plain=buf[1:B + 1], want_aug=False)
    assert none is None and plain2.data_ptr() == buf[1].data_ptr()
    out = buf.cpu().numpy()
    assert np.array_equal(out[1:B + 1], o_plain) and (out[0] == 7).all() and (out[-1] == 7).all()


@gpu
@pytest.mark.parametrize("channels_last", [False, True], ids=["nchw", "nhwc"])
def test_augment_clamps_out_of_range_crop_offsets(channels_last, dev):
    """Crop corners outside [0, S - crop] are clamped into it, for both views (torchvision's TF.crop would pad instead):
    the result equals the oracle at the clamped corner."""
    from dwt_b200 import PairedAugment
    from oracle import augment_oracle as A
    rng = np.random.default_rng(4)
    sh, sw, crop = 13, 17, 8
    offs = np.int32([[-1, -5], [sh - crop + 1, sw - crop + 1], [sh, sw], [-(1 << 30), 1 << 30], [1 << 30, -(1 << 30)],
                     [2, 40], [-3, 4]])
    B = len(offs)
    images = rng.integers(0, 256, (B, sh, sw, 3), dtype=np.uint8)
    flip = np.uint8([b % 2 for b in range(B)])
    aff = np.float32([[[1 + 0.1 * (b % 3), 0.05, 0.5 * b - 1], [-0.05, 0.9, 1 - 0.3 * b]] for b in range(B)])
    p = _params(dict(crop_plain=offs, crop_aug=offs[::-1].copy(), flip=flip, affine=aff), dev)
    plain, aug = PairedAugment(crop=crop)(torch.tensor(images, device=dev), channels_last=channels_last, **p)
    clamp = lambda o: np.stack([np.clip(o[:, 0], 0, sh - crop), np.clip(o[:, 1], 0, sw - crop)], 1)   # noqa: E731
    o_plain, o_aug = A.paired(images, clamp(offs), clamp(offs[::-1]), flip, aff, crop)
    assert np.array_equal(plain.cpu().numpy(), o_plain) and np.array_equal(aug.cpu().numpy(), o_aug)
