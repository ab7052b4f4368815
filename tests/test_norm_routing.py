"""Which kernel family runs a norm call, and what the C ABI refuses.

CPU: the validation table of dwt_whiten_fwd/bwd, dwt_bn_fwd/bwd and dwt_tail2_fwd/bwd over layouts, dtypes, group sizes,
the geometries at every family edge and one-argument variations of a passing call, against the (return code, message)
fixture tests/golden/norm_routing.json (tests/golden/make_norm_routing.py).  Every case stops at an argument check or
at the workspace size, so no call reaches device memory.  Also on the CPU: functional.route predicts the layout and
dtype of every row of the family table.

GPU: the family table -- one row per route a call can take through functional.norm (forward and backward at a small
real shape), with the exact profile families of both directions and the C mode word of the call (ctx.cfg[3]).
"""
import importlib.util
import json
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
BF = torch.bfloat16
CL = torch.channels_last
NHWC, BF16 = 0x100, 0x200


def _table_module():
    spec = importlib.util.spec_from_file_location("make_norm_routing", os.path.join(GOLDEN, "make_norm_routing.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def built():
    import __graft_entry__
    __graft_entry__.build()


# --------------------------------------------------------------------------- CPU: the validation table
def test_validation_table_matches_fixture(built):
    mod = _table_module()
    with open(mod.FIXTURE) as fh:
        doc = json.load(fh)
    ids, results = mod.table()
    assert len(ids) == doc["cases"] and mod.digest(ids) == doc["digest"], "the case grid changed: regenerate the fixture"
    want = [(rc, doc["texts"][i]) for rc, i in doc["results"]]
    bad = [(i, got, exp) for i, got, exp in zip(ids, results, want) if got != exp]
    assert not bad, f"{len(bad)} of {len(ids)} cases differ, e.g.\n" + "\n".join(
        f"{i}\n  got  {g}\n  want {e}" for i, g, e in bad[:5])
    codes = {rc for rc, _ in want}
    assert {-1, -2, -4} <= codes and 0 not in codes


# --------------------------------------------------------------------------- the family table
def _fams(*names, bf16=False):
    return {n + ("_bf16" if bf16 else "") for n in names}


def _small(bf16=False):
    return _fams("small_stats", "small_apply", bf16=bf16), _fams("small_bwd_reduce", "small_bwd_apply", bf16=bf16)


def _tiled():
    return _fams("tiled_stats", "tiled_apply"), _fams("tiled_bwd_reduce", "tiled_bwd_apply")


def _tc(bf16=False, nhwc=False):
    s = "_nhwc" if nhwc else ""
    return (_fams(f"tc_stats{s}", f"tc_apply{s}", bf16=bf16) | _fams("dense_fwd_finalize", bf16=bf16),
            _fams(f"tc_bwd_reduce{s}", f"tc_bwd_apply{s}", bf16=bf16) | _fams("dense_bwd_finalize", bf16=bf16))


def _cl(bf16=False):
    return (_fams("cl_stats", "cl_fwd_finalize", "cl_apply", bf16=bf16),
            _fams("cl_bwd_reduce", "cl_bwd_finalize", "cl_bwd_apply", bf16=bf16))


# name: (dtype, channels-last?, group size, N per domain, C, H, W, storage offset in elements, extra, families, cfg[3])
# extra: "mixed" = a float32 residual with gamma / beta / ReLU.  Two domains per call.
ROWS = {
    "nchw_f32_small":            (torch.float32, False, 4, 4, 16, 8, 8, 0, None, _small(), 0),
    "nchw_f32_tiled":            (torch.float32, False, 8, 2, 16, 8, 8, 0, None, _tiled(), 0),
    "nchw_f32_tc":               (torch.float32, False, 64, 16, 128, 16, 16, 0, None, _tc(), 0),
    "nchw_f32_tc_gs128":         (torch.float32, False, 128, 16, 256, 16, 16, 0, None, _tc(), 0),
    "nchw_bf16_small":           (BF, False, 4, 4, 16, 8, 8, 0, None, _small(True), BF16),
    "nchw_bf16_tc":              (BF, False, 64, 16, 128, 16, 16, 0, None, _tc(True), BF16),
    "nchw_bf16_upcast_hw4":      (BF, False, 4, 4, 16, 5, 5, 0, None, _small(), 0),
    "nchw_bf16_upcast_hw8":      (BF, False, 64, 120, 128, 6, 6, 0, None, _tc(), 0),
    "nchw_bf16_upcast_view":     (BF, False, 4, 4, 16, 8, 8, 1, None, _small(), 0),
    "nchw_bf16_upcast_mixed":    (BF, False, 4, 4, 16, 8, 8, 0, "mixed", _small(), 0),
    "nhwc_f32_cl":               (torch.float32, True, 4, 4, 64, 8, 8, 0, None, _cl(), NHWC),
    "nhwc_bf16_cl":              (BF, True, 4, 4, 64, 8, 8, 0, None, _cl(True), NHWC | BF16),
    "nhwc_f32_cl_width24":       (torch.float32, True, 4, 4, 24, 8, 8, 0, None, _cl(), NHWC),
    "nhwc_bf16_cl_width24":      (BF, True, 4, 4, 24, 8, 8, 0, None, _cl(True), NHWC | BF16),
    "nhwc_f32_tc":               (torch.float32, True, 64, 16, 128, 16, 16, 0, None, _tc(nhwc=True), NHWC),
    "nhwc_bf16_tc":              (BF, True, 64, 16, 128, 16, 16, 0, None, _tc(True, nhwc=True), NHWC | BF16),
    "nhwc_f32_tc_gs128":         (torch.float32, True, 128, 16, 256, 16, 16, 0, None, _tc(nhwc=True), NHWC),
    "nhwc_bf16_gs128_upcast":    (BF, True, 128, 16, 256, 16, 16, 0, None, _tc(nhwc=True), NHWC),
    "nhwc_f32_tc_misaligned":    (torch.float32, True, 64, 16, 128, 16, 16, 2, None, _tc(), 0),
    "nhwc_bf16_tc_misaligned":   (BF, True, 64, 16, 128, 16, 16, 4, None, _tc(nhwc=True), NHWC),
}
D = 2


def _make(row, dev, seed=0):
    """-> (x, residual, gamma, beta) of a row on dev: x a view `offset` elements into its storage."""
    dt, cl, gs, n, c, h, w, offset, extra = row[:9]
    g = torch.Generator().manual_seed(seed)
    numel = D * n * c * h * w
    src = torch.randn(numel, generator=g) + 0.5
    base = torch.empty(numel + offset, dtype=dt, device=dev)
    base[offset:].copy_(src.to(dt))
    flat = base[offset:]
    x = flat.view(D * n, h, w, c).permute(0, 3, 1, 2) if cl else flat.view(D * n, c, h, w)
    if extra != "mixed":
        return x, None, None, None
    res = torch.randn(x.shape, generator=g).to(dev)
    return x, res, torch.rand(c, generator=g).add(0.5).to(dev), torch.randn(c, generator=g).to(dev)


def _running(row, dev):
    gs, c = row[2], row[4]
    return [(torch.zeros(c, device=dev), torch.eye(gs, device=dev).repeat(c // gs, 1, 1)) for _ in range(D)]


def _norm_node(y, prefix):
    node = y.grad_fn
    while not type(node).__name__.startswith(prefix):
        node = node.next_functions[0][0]
    return node


@pytest.mark.parametrize("name", sorted(ROWS))
def test_python_route_predicts_layout_and_dtype(name):
    """functional.route on the CPU tensors of a row (norm() asks again on the float32 copies when it upcasts)."""
    from dwt_b200 import functional as F
    row = ROWS[name]
    x, res, _, _ = _make(row, "cpu")
    r = F.route(x, res, "whiten", row[2], D)
    if r is None:
        x, res = x.float(), None if res is None else res.float()
        r = F.route(x, res, "whiten", row[2], D)
    assert (r.nhwc, r.bf16) == (bool(row[10] & NHWC), bool(row[10] & BF16))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ROWS))
def test_family_table(name, built):
    from dwt_b200 import _native as nv, functional as F
    dev = torch.device("cuda", 0)
    row = ROWS[name]
    (want_fwd, want_bwd), want_mode = row[9], row[10]
    x, res, gamma, beta = _make(row, dev)
    x.requires_grad_(True)
    nv.profile_begin()
    y = F.norm(x, gamma, beta, kind="whiten", group_size=row[2], n_domains=D, training_stats=True, eps=1e-3,
               momentum=0.1, update_running=True, running=_running(row, dev), relu=res is not None, residual=res)
    fwd = set(nv.by_family(nv.profile_end()))
    assert y.dtype == x.dtype and y.shape == x.shape
    mode = _norm_node(y, "_NormFunction").cfg[3]
    nv.profile_begin()
    y.backward(torch.randn_like(y))
    bwd = set(nv.by_family(nv.profile_end()))
    assert (fwd, bwd, mode) == (want_fwd, want_bwd, want_mode), (sorted(fwd), sorted(bwd), hex(mode))
    assert torch.isfinite(x.grad.float()).all()
    assert nv.status_all(dev) == 0


@pytest.mark.gpu
def test_family_table_tail_pair(built):
    """The two-site residual tail, its output used twice through fork_for_sum: the second gradient addend goes to the
    tail's backward kernels (one more tensor read by the reduction)."""
    import dwt_b200
    from dwt_b200 import _native as nv, functional as F
    dev = torch.device("cuda", 0)
    row = (torch.float32, True, 4, 4, 64, 8, 8, 0, None)
    x, _, _, _ = _make(row, dev, seed=1)
    xd, _, _, _ = _make(row, dev, seed=2)
    x.requires_grad_(True)
    xd.requires_grad_(True)
    params = [torch.rand(64, device=dev).add(0.5).requires_grad_(True) for _ in range(4)]
    sites = [(_running(row, dev), 1e-3, 0.1, True) for _ in range(2)]
    nv.profile_begin()
    y = F.tail_pair(x, xd, *params, kind="whiten", group_size=4, n_domains=D, sites=sites)
    fwd = nv.by_family(nv.profile_end())
    assert _norm_node(y, "_TailPairFunction").cfg[0] == nv.KIND_WHITEN
    a, b = dwt_b200.fork_for_sum(y)
    nv.profile_begin()
    torch.autograd.backward([a, b], [torch.randn_like(y), torch.randn_like(y)])
    bwd = nv.by_family(nv.profile_end())
    assert set(fwd) == {"cl_stats", "cl_tail2_fwd_finalize", "cl_tail2_apply"}, sorted(fwd)
    assert set(bwd) == {"cl_tail2_bwd_reduce", "cl_tail2_bwd_finalize", "cl_tail2_bwd_apply"}, sorted(bwd)
    assert fwd["cl_stats"]["launches"] == 2 and all(v["launches"] == 1 for k, v in bwd.items())
    e = 4.0 * x.numel()                              # bytes of one tensor: x, xd, dout, dout2 and the byte map
    assert bwd["cl_tail2_bwd_reduce"]["bytes"] == 5 * e + e / 16
    assert torch.isfinite(x.grad).all() and torch.isfinite(xd.grad).all()
