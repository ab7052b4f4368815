"""Latent-domain batch norm and small-group latent-domain whitening (gs 1, 2, 4) at every edge of their shared work plan
(ldbn_plan / lds_plan, norm_ldbn.cu): segment tails of 1 pixel and of exactly P pixels, the segment count at its cap and
at 1, NCHW scalar loads over several segments, fewer than 8 images, and channels-last slabs whose width qc does not divide
the 256 threads or whose last slab is partial.  The shapes come from tests/support/ldbn_plan.py, which restates the plan
and generates one shape per edge for the device's SM count.

CPU: every generated shape has the plan property its name claims, at 114 and 132 SMs.

GPU: the restated workspace carve equals the library's workspace queries at every case, so a plan that drifts from the
restatement fails here instead of quietly testing other shapes; every case against the float64 composition (the site
harness of test_latent_domain_sites.py, loaded from its file: y, dx, dweights, dgamma, dbeta, dresidual and the running
buffers, train / eval / untracked, AFFINE, AFFINE|RELU, AFFINE|RELU|RESIDUAL, D = 3 and 8) with that file's bounds; bf16
bit for bit against the fp32 call on the widened inputs; the channels-last residual's byte map through its effect
(dresidual == dout where out > 0, else 0); reruns bit for bit; the launch profile naming the family that ran; and each
row's first pixel -- the latent passes' pilot shift -- 30 sigma off its row.
"""
import importlib.util
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import ld_reference as LR  # noqa: E402
import ldbn_plan as PL  # noqa: E402
import ldbn_reference as LB  # noqa: E402

_spec = importlib.util.spec_from_file_location("_latent_sites_harness",
                                               os.path.join(os.path.dirname(__file__), "test_latent_domain_sites.py"))
H = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(H)

gpu = pytest.mark.gpu
EPIS = ["affine", "relu", "residual"]
MOMENTUM = 0.1

# Edge names do not depend on the SM count (their shapes do): parametrize by name, resolve on the device.
_NAMES = [e.name for e in PL.edges(132)]
_LAYOUT = {e.name: (e.layout, e.gs) for e in PL.edges(132)}


def _families(name):
    """(kind, gs) run at an edge: channels-last edges hold for batch norm and every gs; an NCHW edge for its own gs,
    batch norm with the gs 1 ones."""
    layout, gs = _LAYOUT[name]
    if layout == "cl":
        return [("bn", 1), ("whiten", 1), ("whiten", 2), ("whiten", 4)]
    return ([("bn", 1)] if gs == 1 else []) + [("whiten", gs)]


CASES = [(name, kind, gs) for name in _NAMES for kind, gs in _families(name)]
CL_WIDTHS = [n for n in _NAMES if n.startswith("cl_c4_")]       # the odd C/4 and partial-slab widths
_ids = [f"{n}-{k}{'' if k == 'bn' else gs}" for n, k, gs in CASES]


# =========================================================================== CPU: the generator
@pytest.mark.parametrize("sms", [114, 132])
def test_generated_shapes_have_the_claimed_plan(sms):
    edges = PL.edges(sms)
    assert [e.name for e in edges] == _NAMES
    for e in edges:
        bad = [k for k, ok in PL.claims(e, sms).items() if not ok]
        assert not bad, (e, PL.plan(e.shape[0], e.shape[1], e.shape[2] * e.shape[3], sms, e.layout == "cl", e.gs), bad)


def test_the_mislabelled_whitening_edges_run_two_long_segments():
    """test_latent_domain_whitening_small's [2, 8, 257, 1] NCHW and [2, 4, 1025, 1] channels-last cases (gs 4): two
    segments of 132 + 125 and 513 + 512 pixels, at either SM count; the 1-pixel tails are this file's *_tail1 edges."""
    for sms in (114, 132):
        a = PL.plan(2, 8, 257, sms, False, 4)
        b = PL.plan(2, 4, 1025, sms, True, 4)
        assert (a.S, a.P, PL.tail(a, 257)) == (2, 132, 125)
        assert (b.S, b.P, PL.tail(b, 1025)) == (2, 513, 512)


# =========================================================================== GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


@pytest.fixture(scope="module")
def shapes(sms):
    return {e.name: e.shape for e in PL.edges(sms)}


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nlatent-domain plan edges, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-72s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def _layout(name):
    return _LAYOUT[name][0]


def _ref_running(cs, mode):
    """The running buffers after the call, in float64: the EMA of the weighted statistics in train mode (batch norm:
    the unbiased variance, skipped where M s_d <= 1; whitening: the biased second moment of every live domain)."""
    rm, rv = cs.rm.double(), cs.rv.double()
    if mode != "train":
        return rm, rv
    x, w = cs.x.double(), cs.w.double()
    if cs.kind == "bn":
        return LB.running_update(LB.ldbn_torch(x, w, eps=cs.eps), (rm, rv), MOMENTUM, x[0, 0].numel())
    f = LR.ld_torch(x, cs.gs, w, eps=cs.eps)
    for k in f["live"]:
        rm[k] = (1 - MOMENTUM) * rm[k] + MOMENTUM * f["mu"][k].reshape(-1)
        rv[k] = (1 - MOMENTUM) * rv[k] + MOMENTUM * f["sigma"][k]
    return rm, rv


def _against_float64(worst, label, cs, epi, layout, mode):
    got = H.site_call(cs, epi, layout, mode)
    H.compare(worst, label, got, H.ref_call(cs, epi, mode, mask=(got["y"] != 0).double()))
    want = _ref_running(cs, mode)
    for name, a, b, orig in zip(("rmean", "rvar"), got["running"], want, (cs.rm, cs.rv)):
        if mode == "train":
            H.check(worst, label, name, a, b)
        else:
            assert torch.equal(a, orig), f"{label}: {name} changed outside train mode"


@gpu
@pytest.mark.parametrize("name, kind, gs", CASES, ids=_ids)
def test_workspace_query_is_the_restated_carve(dev, sms, shapes, name, kind, gs):
    from dwt_b200 import _native
    lib = _native.lib()
    n, c, h, w = shapes[name]
    for d in (3, 8):
        got = lib.dwt_bn_latent_workspace_bytes(n, c, h * w, d) if kind == "bn" else \
            lib.dwt_latent_small_workspace_bytes(n, c, h * w, gs, d)
        assert got == PL.workspace_bytes(kind, n, c, h * w, gs, d, sms), (name, kind, gs, d)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval", "notrack"])
@pytest.mark.parametrize("d", [3, 8])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("name, kind, gs", CASES, ids=_ids)
def test_edges_against_float64(dev, worst, shapes, name, kind, gs, epi, d, mode):
    shape = shapes[name]
    cs = H.Case(kind, shape, gs, d, dev, seed=d)
    _against_float64(worst, f"{name} {kind} gs{gs} {list(shape)} D{d} {mode} {epi}", cs, epi, _layout(name), mode)


def _bf16_kernels(name, shape):
    """The layout has bf16 kernels at this shape: channels-last always, NCHW at H*W % 4 == 0 (else an fp32 upcast)."""
    return _layout(name) == "cl" or (shape[2] * shape[3]) % 4 == 0


@gpu
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("name, kind, gs", CASES, ids=_ids)
def test_bf16_is_the_fp32_call_on_widened_inputs_rounded(dev, shapes, name, kind, gs, epi):
    shape = shapes[name]
    cs = H.Case(kind, shape, gs, 3, dev, seed=4)
    layout = _layout(name)
    xb, rb, db = cs.x.bfloat16(), cs.res.bfloat16(), cs.dout.bfloat16()
    got = H.site_call(cs, epi, layout, dtype=torch.bfloat16, x=xb, dout=db, res=rb)
    want = H.site_call(cs, epi, layout, x=xb.float(), dout=db.float(), res=rb.float())
    for k in ("y", "dx", "dres"):
        if want[k] is not None:
            assert got[k].dtype == torch.bfloat16 and torch.equal(got[k], want[k].bfloat16()), k
    for k in ("dw", "dgamma", "dbeta"):
        assert torch.equal(got[k], want[k]), k
    for a, b in zip(got["running"], want["running"]):
        assert torch.equal(a, b)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("name, kind, gs", [c for c in CASES if c[0] in CL_WIDTHS + ["cl_tail1"]],
                         ids=[i for c, i in zip(CASES, _ids) if c[0] in CL_WIDTHS + ["cl_tail1"]])
def test_channels_last_byte_map_passes_dout_where_the_output_is_positive(dev, shapes, name, kind, gs, dtype):
    """The forward writes bit k of byte (n HW + p) C/4 + c4 for channel 4 c4 + k of pixel p; the backward reduction reads
    it back to mask dout into dresidual.  A wrong index or bit order moves a gradient to or from an element whose output
    is 0."""
    cs = H.Case(kind, shapes[name], gs, 3, dev, seed=6)
    out = H.site_call(cs, "residual", "cl", dtype=dtype, x=cs.x.to(dtype), dout=cs.dout.to(dtype), res=cs.res.to(dtype))
    dout = cs.dout.to(dtype)
    assert torch.equal(out["dres"], torch.where(out["y"] > 0, dout, torch.zeros_like(dout)))
    assert 0 < int((out["y"] > 0).sum()) < out["y"].numel()


@gpu
@pytest.mark.parametrize("name", ["cl_c4_65_slab1", "cl_c4_257_slab1", "cl_tail1"])
@pytest.mark.parametrize("kind, gs", [("bn", 1), ("whiten", 1), ("whiten", 2), ("whiten", 4)])
def test_reruns_are_bit_identical(dev, shapes, name, kind, gs):
    cs = H.Case(kind, shapes[name], gs, 8, dev, seed=9)
    a, b = (H.site_call(cs, "residual", "cl") for _ in range(2))
    for k in ("y", "dx", "dw", "dgamma", "dbeta", "dres"):
        assert torch.equal(a[k], b[k]), k
    for u, v in zip(a["running"], b["running"]):
        assert torch.equal(u, v)


def _expected_families(kind, layout, bf16, mode):
    p = "ldbn" if kind == "bn" else "lds"
    sfx = ("_nhwc" if layout == "cl" else "") + ("_bf16" if bf16 else "")
    passes = (["stats"] if mode != "eval" else []) + ["apply", "bwd_reduce", "bwd_apply"]
    return {f"{p}_{q}{sfx}" for q in passes} | {f"{p}_fwd_finalize", f"{p}_bwd_finalize"}


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("name, kind, gs", CASES, ids=_ids)
def test_route_is_the_layout_and_dtype_family(dev, shapes, name, kind, gs, dtype):
    """The launch profile names the family that ran: ldbn_* / lds_*, _nhwc for channels-last, _bf16 for bf16 kernels --
    so a case that fell back to an NCHW copy or an fp32 upcast fails here.  NCHW bf16 at H*W % 4 != 0 is the documented
    upcast: the fp32 NCHW kernels."""
    from dwt_b200 import _native
    shape = shapes[name]
    bf16 = dtype == torch.bfloat16 and _bf16_kernels(name, shape)
    cs = H.Case(kind, shape, gs, 3, dev, seed=2)
    layout = _layout(name)
    torch.cuda.synchronize()
    _native.profile_begin()
    H.site_call(cs, "relu", layout, dtype=dtype, x=cs.x.to(dtype), dout=cs.dout.to(dtype))
    fams = {f for f, v in _native.by_family(_native.profile_end()).items() if v["launches"]}
    assert fams == _expected_families(kind, layout, bf16, "train"), fams


def _pilot_30_sigma(x):
    """x with the first pixel of every (image, channel) row -- the latent passes' pilot shift -- 30 sigma off the row's
    mean."""
    n, c = x.shape[:2]
    flat = x.reshape(n, c, -1).clone()
    flat[:, :, 0] = flat.mean(-1) + 30.0 * flat.std(-1)
    return flat.reshape(x.shape)


@gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("layout", ["nchw", "cl"])
@pytest.mark.parametrize("kind, gs", [("bn", 1), ("whiten", 1), ("whiten", 2), ("whiten", 4)])
def test_pilot_30_sigma_off_against_float64(dev, worst, kind, gs, layout, mode):
    shape = (16, 64, 28, 28)
    cs = H.Case(kind, shape, gs, 3, dev, seed=11)
    cs.x = _pilot_30_sigma(cs.x)
    _against_float64(worst, f"pilot 30 sigma {kind} gs{gs} {list(shape)} {layout} {mode} residual", cs, "residual",
                     layout, mode)
