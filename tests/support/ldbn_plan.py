"""The work plan of latent-domain batch norm and small-group latent-domain whitening, restated in plain Python, and a
generator of shapes that each land on one edge of it.

Restated from dwt_b200/csrc/norm_ldbn.cu -- ldbn_plan, lds_plan (a group of gs channels in place of a channel: NCHW plans
N x C/gs rows, channels-last C channels), the slab count of ldbn_reduce_nhwc / lds_reduce_nhwc / lds_apply_nhwc and their
launches, ldbn_scratch_floats, lds_partial_floats, lds_coef_floats -- and from dwt_b200/csrc/api.cu -- kOffScratch, the
carves carve_ldbn and carve_lds, larger_layout_workspace_bytes.

    NCHW: S = clamp(min(ceil(64 SMs / rows), ceil(HW / 256)), 1), P = ceil(ceil(HW / S) / 4) * 4 (whole float4s);
          a warp per (row, segment); HW % 4 != 0 runs the scalar loads.
    channels-last: qc = min(C/4, 64) float4 columns, pr = 256 // qc pixel rows (threads past qc * pr sit out), slabs =
          ceil(C/4 / qc) (the last one partial when C/4 > 64 and C/4 % 64 != 0), a CTA per (image, slab, segment);
          S = clamp(min(ceil(8 SMs / (N slabs)), ceil(HW / (4 pr))), 1), P = ceil(HW / S).
    both: S = ceil(HW / P) after P is set; the last segment holds HW - (S - 1) P pixels.

The workspace queries dwt_bn_latent_workspace_bytes / dwt_latent_small_workspace_bytes return the larger of the two
layouts' carves.  The carves differ only in the segment partials, so the query pins the segment count of the layout with
the larger carve exactly (up to the 256-byte rounding of each array) and only bounds the other from above.
"""
from collections import namedtuple

THREADS = 256                       # kThreads (dwt_common.cuh)
MAX_DOMAINS = 4                     # DWT_MAX_DOMAINS (dwt_b200.h): the arrival counters of the common workspace head
MAX_GROUPS = 65536                  # kMaxGroups (api.cu)
OFF_SCRATCH = 256 + 4 * MAX_DOMAINS * MAX_GROUPS + 4 * MAX_GROUPS + 4 * MAX_GROUPS   # kOffScratch (api.cu)
LDS_MAX_DOMAINS = 8                 # kLdsMaxDomains (norm_launch.h): dweights shares per (image, group)

Plan = namedtuple("Plan", "nhwc S P qc pr slabs want cap")


def _cdiv(a, b):
    return -(-a // b)


def plan(n, c, hw, sms, nhwc, gs=1):
    """ldbn_plan (gs 1) / lds_plan (gs 1, 2, 4).  want / cap: the segment count asked for by the occupancy target and
    its per-segment minimum."""
    if nhwc:
        c4 = c // 4
        qc = min(c4, 64)
        pr = THREADS // qc
        slabs = _cdiv(c4, qc)
        want = _cdiv(8 * sms, n * slabs)
        cap = _cdiv(hw, 4 * pr)                       # at least 4 pixels per thread and segment
        s = max(min(want, cap), 1)
        p = _cdiv(hw, s)
    else:
        qc = pr = slabs = 0
        want = _cdiv(64 * sms, n * (c // gs))          # one full load of warps
        cap = _cdiv(hw, 256)                          # at least 256 pixels per warp and segment
        s = max(min(want, cap), 1)
        p = _cdiv(_cdiv(hw, s), 4) * 4
    return Plan(nhwc, _cdiv(hw, p), p, qc, pr, slabs, want, cap)


def tail(pl, hw):
    """Pixels of the last segment."""
    return hw - (pl.S - 1) * pl.P


def last_slab_columns(c):
    """float4 columns of the last channels-last slab."""
    c4 = c // 4
    return c4 - (_cdiv(c4, min(c4, 64)) - 1) * min(c4, 64)


def _align(v):
    return _cdiv(v, 256) * 256


def _carve(arrays):
    off = OFF_SCRATCH
    for nbytes in arrays:
        off = _align(off + nbytes)
    return off


def carve_ldbn(n, c, pl, d):
    """carve_ldbn: pa, pb [N][S][C]; pilot, c0, c1, c2 [N][C]; the dweights shares [N][D][ceil(C / 32)] (floats)."""
    part, nc, dw = n * pl.S * c, n * c, n * d * _cdiv(c, 32)
    return _carve(4 * k for k in (part, part, nc, nc, nc, nc, dw))


def carve_lds(n, c, pl, gs, k):
    """carve_lds: the segment partials, pilot, fp64 image moments, backward sums, P_k | mubar_k, <P_k, Sigma_k>, the
    apply coefficients, the dweights shares."""
    ng, kg = n * (c // gs), k * (c // gs)
    return _carve([4 * ng * pl.S * (gs + gs * gs), 4 * n * c, 8 * ng * (gs + gs * (gs + 1) // 2), 4 * ng * (gs + gs * gs),
                   4 * kg * (gs * gs + gs), 4 * kg, 4 * ng * (gs * (gs + 1) // 2 + gs * gs + 2 * gs),
                   4 * ng * LDS_MAX_DOMAINS])


def workspace_bytes(kind, n, c, hw, gs, d, sms):
    """dwt_bn_latent_workspace_bytes (kind "bn") / dwt_latent_small_workspace_bytes (kind "whiten") of a valid
    geometry: the larger of the two layouts' carves, channels-last counted only at C % 4 == 0."""
    most = 0
    for nhwc in (False, True):
        if nhwc and c % 4:
            continue
        pl = plan(n, c, hw, sms, nhwc, gs)
        most = max(most, carve_ldbn(n, c, pl, d) if kind == "bn" else carve_lds(n, c, pl, gs, d))
    return most


# ---------------------------------------------------------------------------------------------------- plan edges
Edge = namedtuple("Edge", "name layout gs shape")     # gs: the NCHW rows' group size (channels-last: any of 1, 2, 4)

ODD_WIDTHS = (3, 5, 25)             # C/4 with qc not dividing 256
SLAB_WIDTHS = (65, 80, 257)         # C/4 > 64: a last slab of 1, 16 and 1 columns


def _hw_shape(hw):
    """[H, W] of hw pixels: the most square split with H >= W (a prime hw is [hw, 1])."""
    w = max(k for k in range(1, int(hw ** 0.5) + 1) if hw % k == 0)
    return (hw // w, w)


def _first(cands, ok):
    for n, c, hw in cands:
        if ok(n, c, hw):
            return (n, c) + _hw_shape(hw)
    raise AssertionError("no shape found for a plan edge")


def _multi_segment(sms, nhwc, gs=1):
    return lambda n, c, hw: plan(n, c, hw, sms, nhwc, gs).S > 1


def claims(edge, sms):
    """{property: holds} for what the edge's name claims about its plan."""
    n, c = edge.shape[:2]
    hw = edge.shape[2] * edge.shape[3]
    nhwc = edge.layout == "cl"
    pl = plan(n, c, hw, sms, nhwc, edge.gs)
    t = tail(pl, hw)
    out = {}
    name = edge.name
    if nhwc:
        out["C % 4 == 0"] = c % 4 == 0
    else:
        out["C % gs == 0"] = c % edge.gs == 0
    if name.startswith("cl_c4_") and name.endswith("_qc_odd"):
        out["qc does not divide 256"] = THREADS % pl.qc != 0 and c // 4 == int(name.split("_")[2])
        out["S > 1"] = pl.S > 1
    if name.startswith("cl_c4_") and "_slab" in name:
        want = int(name.split("slab")[1])
        out["partial last slab"] = c // 4 > 64 and pl.slabs > 1 and last_slab_columns(c) == want
        out["S > 1"] = pl.S > 1
    if name.endswith("_tail1"):
        out["S > 1 and a 1-pixel last segment"] = pl.S > 1 and t == 1
    if name.endswith("_tail_exact"):
        out["S > 1 and a last segment exactly P long"] = pl.S > 1 and t == pl.P
    if name.endswith("_s_cap"):
        out["S at its cap below the occupancy target"] = pl.S == pl.cap > 1 and pl.want > pl.cap
    if name.endswith("_s1_full"):
        rows = n * (c // edge.gs) if not nhwc else n * pl.slabs
        full = 64 * sms if not nhwc else 8 * sms
        out["S == 1 from a full load of rows"] = pl.S == 1 and rows >= full and pl.cap > 1
    if name.endswith("_scalar_multi"):
        out["HW % 4 != 0 and S > 1"] = hw % 4 != 0 and pl.S > 1 and not nhwc
    if name.endswith("_n1"):
        out["N == 1 and S > 1"] = n == 1 and pl.S > 1
    if name.endswith("_n5"):
        out["1 < N < 8 and S > 1"] = 1 < n < 8 and pl.S > 1
    assert len(out) > 1, f"no claim checked for {name}"
    return out


def edges(sms):
    """The plan edges at this SM count: Edge(name, layout, gs, [N, C, H, W]).  Channels-last edges hold for batch norm and
    every group size (the channels-last plan does not depend on gs); an NCHW edge is made for its gs (NCHW rows are
    N x C/gs) and batch norm runs the gs 1 ones."""
    out = []
    # channels-last widths: qc not dividing 256; a partial last slab -- each over more than one segment
    for c4 in ODD_WIDTHS:
        out.append(Edge(f"cl_c4_{c4}_qc_odd", "cl", 1,
                        _first(((n, 4 * c4, hw) for hw in (49, 100, 196, 400, 784, 1600) for n in (4, 8)),
                               _multi_segment(sms, True))))
    for c4 in SLAB_WIDTHS:
        cols = last_slab_columns(4 * c4)
        out.append(Edge(f"cl_c4_{c4}_slab{cols}", "cl", 1,
                        _first(((n, 4 * c4, hw) for hw in (49, 100, 196, 400) for n in (2, 4)), _multi_segment(sms, True))))

    def cl_first(cands, ok):
        return _first(cands, lambda n, c, hw: ok(n, c, hw, plan(n, c, hw, sms, True)))

    out.append(Edge("cl_tail1", "cl", 1, cl_first(((3, c, hw) for c in (260, 20) for hw in range(17, 4000)),
                                                  lambda n, c, hw, p: p.S > 1 and tail(p, hw) == 1)))
    out.append(Edge("cl_tail_exact", "cl", 1, cl_first(((3, c, hw) for c in (100, 260) for hw in range(17, 4000)),
                                                       lambda n, c, hw, p: p.S > 2 and tail(p, hw) == p.P)))
    out.append(Edge("cl_s_cap", "cl", 1, cl_first(((2, 20, hw) for hw in range(100, 4000)),
                                                  lambda n, c, hw, p: p.S == p.cap > 1 and p.want > p.cap)))
    out.append(Edge("cl_s1_full", "cl", 1, cl_first(((n, 256, hw) for hw in (17, 20, 25) for n in range(8 * sms, 16 * sms)),
                                                    lambda n, c, hw, p: p.S == 1 and p.cap > 1)))
    out.append(Edge("cl_n1", "cl", 1, cl_first(((1, 260, hw) for hw in (100, 196, 400)), lambda n, c, hw, p: p.S > 1)))
    out.append(Edge("cl_n5", "cl", 1, cl_first(((5, 20, hw) for hw in (100, 196, 400)), lambda n, c, hw, p: p.S > 1)))

    # NCHW, one set per group size (batch norm: gs 1)
    for gs in (1, 2, 4):
        def nc_first(cands, ok):
            return _first(cands, lambda n, c, hw: ok(n, c, hw, plan(n, c, hw, sms, False, gs)))

        small = [(2, 4 * gs), (2, 8 * gs), (4, 8 * gs)]
        out.append(Edge(f"nchw_gs{gs}_tail1", "nchw", gs,
                        nc_first(((n, c, hw) for n, c in small for hw in range(257, 40000, 4)),
                                 lambda n, c, hw, p: p.S > 1 and tail(p, hw) == 1)))
        out.append(Edge(f"nchw_gs{gs}_tail_exact", "nchw", gs,
                        nc_first(((n, c, hw) for n, c in small for hw in range(260, 40000, 4)),
                                 lambda n, c, hw, p: p.S > 2 and tail(p, hw) == p.P)))
        out.append(Edge(f"nchw_gs{gs}_scalar_multi", "nchw", gs,
                        nc_first(((n, c, hw) for n, c in small for hw in range(771, 40000, 4)),
                                 lambda n, c, hw, p: p.S > 2 and hw % 4 == 3 and 1 < tail(p, hw) < p.P)))
        out.append(Edge(f"nchw_gs{gs}_s_cap", "nchw", gs,
                        nc_first(((n, 4 * gs, hw) for n in (2, 4) for hw in (300, 784, 1000)),
                                 lambda n, c, hw, p: p.S == p.cap > 1 and p.want > p.cap)))
        out.append(Edge(f"nchw_gs{gs}_s1_full", "nchw", gs,
                        nc_first(((n, 64 * gs, 260) for n in range(sms, 4 * sms)),
                                 lambda n, c, hw, p: p.S == 1 and p.cap > 1 and n * (c // gs) >= 64 * sms)))
        out.append(Edge(f"nchw_gs{gs}_n1", "nchw", gs,
                        nc_first(((1, 4 * gs, hw) for hw in (784, 1000, 3000)), lambda n, c, hw, p: p.S > 1)))
        out.append(Edge(f"nchw_gs{gs}_n5", "nchw", gs,
                        nc_first(((5, 4 * gs, hw) for hw in (784, 1000, 3000)), lambda n, c, hw, p: p.S > 1)))
    return out
