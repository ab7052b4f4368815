"""Whitening in the ZCA basis (ZCAWTransform2d, dwt_whiten_zca_*) on the tensor-core kernels, against the float64
ATen restatement of its definition (tests/support/zca_reference.py) and against itself.

Tolerances as in test_nchw_fp64.py: outputs and input gradients within 1e-3 norm-wise of float64, max-elementwise
error within 5x that; statistics and running buffers within 1e-4.  Where the bound holds: the iteration is not
self-correcting past convergence (test_zca_oracle.py), so T = 16 is checked on well-conditioned groups (iid inputs:
condition number below about 2 at >= 4096 samples per group) and groups of condition number 1e3 at T <= 5;
test_ill_conditioned_accuracy prints the error it measures at T = 5..16 across condition numbers.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import zca_reference as Z  # noqa: E402

pytestmark = pytest.mark.gpu
BOUND, STAT_BOUND = 1e-3, 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst():
    table = {}
    yield table
    print("\nZCA basis, worst errors against float64 (norm-wise, max-elementwise):")
    for k in sorted(table):
        print("  %-34s %s" % (k, ", ".join(f"{n} {r:.1e} {m:.1e}" for n, (r, m) in sorted(table[k].items()))))


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check(worst, label, name, a, b, bound=BOUND):
    r, m = rel(a, b)
    worst.setdefault(label, {})[name] = (r, m)
    assert r <= bound and m <= 5 * bound, f"{label} {name}: norm-wise {r:.2e}, max-elementwise {m:.2e}"


def iid(shape, dev, seed=0, shift=1.5):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, device=dev, generator=g) + shift


def mixed(shape, dev, seed=0, shift=2.0):
    """bench.py's microbench input: x = mix . randn + 2, mix = randn / sqrt(C) + I over all channels."""
    n, c, h, w = shape
    g = torch.Generator(device=dev).manual_seed(seed)
    mix = torch.randn(c, c, device=dev, generator=g) / c ** 0.5 + torch.eye(c, device=dev)
    return (torch.einsum("dc,nchw->ndhw", mix, torch.randn(n, c, h, w, device=dev, generator=g)) + shift).contiguous()


def ema_ref(rm, rc, mean, cov, m):
    return (1 - m) * rm.double() + m * mean.reshape(rm.shape), (1 - m) * rc.double() + m * cov.reshape(rc.shape)


def families(prof):
    return {k.split("|")[0] for k in prof}


def run_case(dev, worst, label, x, gs, T, d=1, mode="train", layout="shared", via="module", check_profile=False):
    """x [d*N, C, H, W] through d ZCAWTransform2d modules (via='module': d sequential calls) or one DomainTripleNorm
    site (via='site'), forward + backward, against float64 per domain; running buffers through the ordered EMA."""
    import dwt_b200
    from dwt_b200 import _native as nv
    c = x.shape[1]
    n = x.shape[0] // d
    gen = torch.Generator(device=dev).manual_seed(1)
    dy = torch.randn(x.shape, device=dev, generator=gen)
    default = mode == "default"
    # running buffers: one shared pair, one per domain, or domains 0 and 2 sharing
    pairs = []
    for k in range({"shared": 1, "distinct": d, "mixed": 2}[layout]):
        rm = torch.randn(1, c, 1, 1, device=dev, generator=gen) * 0.1
        a = torch.randn(c // gs, gs, 2 * gs, device=dev, generator=gen)
        rc = 0.25 * torch.bmm(a, a.transpose(1, 2)) / (2 * gs) + torch.eye(gs, device=dev)   # condition number < 2
        pairs.append((rm, rc))
    which = {"shared": [0] * d, "distinct": list(range(d)), "mixed": [0, 1, 0, 1][:d]}[layout]
    mods = []
    for k in range(d):
        rm, rc = pairs[which[k]]
        m = (dwt_b200.ZCAWTransform2d(c, gs, iterations=T) if default else
             dwt_b200.ZCAWTransform2d(c, gs, running_m=rm, running_var=rc, iterations=T)).to(dev)
        mods.append(m.train(mode in ("train", "nograd", "default")))
    before = [(m.running_mean.clone(), m.running_variance.clone()) for m in mods]
    xg = x.clone().requires_grad_(mode != "nograd")
    nv.profile_begin()
    with torch.set_grad_enabled(mode != "nograd"):
        if via == "site":
            y = dwt_b200.DomainTripleNorm("whiten", c, gs, n_domains=d)(xg, mods, None, None)
        else:
            y = torch.cat([mods[k](xg[k * n:(k + 1) * n]) for k in range(d)])
        dx = torch.autograd.grad(y, xg, dy)[0] if mode != "nograd" else None
    prof = nv.profile_end()
    if check_profile:
        fam = families(prof)
        want = {"dense_fwd_zca"} | ({"dense_bwd_zca", "tc_bwd_apply"} if dx is not None else set())
        want |= {"tc_stats", "tc_apply"} if mode != "eval" else {"tc_apply"}
        assert want <= fam and not any(f.startswith(("dense_fwd_finalize", "tiled", "small")) for f in fam), fam
    # float64, domain by domain, with the EMA in order on (possibly shared) running buffers
    train = mode != "eval"
    ref_buf = {}
    for k in range(d):
        key = which[k] if not default else k
        rm0, rc0 = ref_buf.get(key, tuple(t.double() for t in before[k]))
        xd = x[k * n:(k + 1) * n].double().requires_grad_(True)
        yr, mean, cov, _ = Z.zca_torch(xd, gs, T, eps=1e-3, running_mean=rm0, running_cov=rc0, train=train)
        tag = f"{label} d{k}"
        check(worst, tag, "y", y[k * n:(k + 1) * n].detach(), yr.detach())
        if dx is not None:
            (dxr,) = torch.autograd.grad(yr, xd, dy[k * n:(k + 1) * n].double())
            check(worst, tag, "dx", dx[k * n:(k + 1) * n], dxr)
        if train:
            ref_buf[key] = ema_ref(rm0, rc0, mean.detach(), cov.detach(), 0.1)
    if train:
        for k in range(d):
            key = which[k] if not default else k
            check(worst, f"{label} d{k}", "running_mean", mods[k].running_mean, ref_buf[key][0], STAT_BOUND)
            check(worst, f"{label} d{k}", "running_var", mods[k].running_variance, ref_buf[key][1], STAT_BOUND)
    else:
        for k in range(d):
            assert torch.equal(mods[k].running_mean, before[k][0]) and torch.equal(mods[k].running_variance, before[k][1])


# --------------------------------------------------------------------------- 1. float64 reference
def test_config2_full_size(dev, worst):
    """N=256 C=256 56^2 at group size 64, T = 5, the microbench input, default-constructed buffers."""
    run_case(dev, worst, "config2 gs64 T5", mixed((256, 256, 56, 56), dev), 64, 5, mode="default", check_profile=True)


EDGES = [
    # label, (N, C, H, W), gs, T, domains, mode, buffer layout, via
    ("gs8 c64 hw32 T16", (128, 64, 4, 8), 8, 16, 1, "train", "shared", "module"),
    ("gs16 c96 partial-sb T5", (16, 96, 16, 16), 16, 5, 1, "train", "shared", "module"),
    ("gs32 c96 partial-sb T1", (16, 96, 16, 16), 32, 1, 1, "train", "shared", "module"),
    ("gs64 c512 T16", (8, 512, 24, 24), 64, 16, 1, "train", "shared", "module"),
    ("gs64 hw36 d2 distinct T5", (2 * 114, 128, 6, 6), 64, 5, 2, "train", "distinct", "site"),
    ("gs32 hw40 d3 mixed T16", (3 * 103, 64, 5, 8), 32, 16, 3, "train", "mixed", "site"),
    ("gs16 hw3136 d4 shared T5", (4 * 2, 64, 56, 56), 16, 5, 4, "train", "shared", "site"),
    ("gs64 m4096 nograd T5", (128, 128, 4, 8), 64, 5, 1, "nograd", "shared", "module"),
    ("gs64 eval T5", (16, 128, 16, 16), 64, 5, 1, "eval", "shared", "module"),
    ("gs8 eval d3 site T16", (3 * 16, 64, 16, 16), 8, 16, 3, "eval", "distinct", "site"),
    ("gs32 default d3 site T1", (3 * 16, 128, 16, 16), 32, 1, 3, "default", "shared", "site"),
]


@pytest.mark.parametrize("case", EDGES, ids=[e[0] for e in EDGES])
def test_edges(case, dev, worst):
    label, shape, gs, T, d, mode, layout, via = case
    run_case(dev, worst, label, iid(shape, dev, seed=len(label)), gs, T, d, mode, layout, via, check_profile=True)


@pytest.mark.parametrize("gs", [8, 64])
@pytest.mark.parametrize("T", [1, 5])
def test_ill_conditioned(gs, T, dev, worst):
    """Condition number 1e3 in every group (exact batch covariance spectrum from 1 to 1e-3)."""
    import numpy as np
    x = torch.tensor(Z.conditioned_input(np.random.default_rng(gs), 64, 128, (8, 8), gs, 1e3, shift=1.0),
                     dtype=torch.float32, device=dev)
    run_case(dev, worst, f"cond1e3 gs{gs} T{T}", x, gs, T)


def test_ill_conditioned_accuracy(dev, capsys):
    """Past the range asserted above: report (not assert) the forward error against float64 at T = 5, 8, 12, 16 per
    group size and condition number."""
    import numpy as np
    import dwt_b200
    lines = []
    for gs in (8, 64):
        for cond in (1.0, 2.0, 10.0, 100.0, 1e3):
            x = torch.tensor(Z.conditioned_input(np.random.default_rng(3), 64, 64, (8, 8), gs, cond, shift=1.0),
                             dtype=torch.float32, device=dev)
            row = []
            for T in (5, 8, 12, 16):
                y = dwt_b200.ZCAWTransform2d(64, gs, iterations=T).to(dev)(x)
                yr, *_ = Z.zca_torch(x.double(), gs, T)
                r, mx = rel(y.detach(), yr)
                row.append(f"T={T} {r:.1e}/{mx:.1e}")
            lines.append(f"  gs {gs:2d} cond {cond:6g}: " + "  ".join(row))
    with capsys.disabled():
        print("\nZCA basis forward against float64 (norm-wise/max-elementwise):\n" + "\n".join(lines))


# --------------------------------------------------------------------------- 2. statistics
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_statistics_equal_cholesky(layout, dev):
    """Running buffers and save_mean bit for bit those of WTransform2d on the same input (the shared prologue and EMA)."""
    import dwt_b200
    from dwt_b200 import functional as F
    x = mixed((32, 128, 16, 16), dev)
    if layout == "nhwc":
        x = x.contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    zm, wm = dwt_b200.ZCAWTransform2d(128, 32).to(dev), dwt_b200.WTransform2d(128, 32).to(dev)
    yz, yw = zm(x), wm(x)
    assert torch.equal(zm.running_mean, wm.running_mean) and torch.equal(zm.running_variance, wm.running_variance)
    assert torch.equal(yz.grad_fn.saved_tensors[1], yw.grad_fn.saved_tensors[1])          # save_mean
    # three domains on shared buffers through one call
    bufs = [(torch.zeros(1, 128, 1, 1, device=dev), torch.eye(32, device=dev).repeat(4, 1, 1)) for _ in range(2)]
    for it, (rm, rc) in zip((5, 0), bufs):
        _ = F.norm(x.detach().repeat(3, 1, 1, 1), None, None, kind="whiten", group_size=32, n_domains=3, training_stats=True, eps=1e-3,
               momentum=0.1, update_running=True, running=[(rm, rc)] * 3, iterations=it)
    assert torch.equal(bufs[0][0], bufs[1][0]) and torch.equal(bufs[0][1], bufs[1][1])


# --------------------------------------------------------------------------- 3. layouts, dtypes, determinism, graphs
def _fwd_bwd(m, x, dy):
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    (dx,) = torch.autograd.grad(y, xg, dy)
    return y.detach(), dx


@pytest.mark.parametrize("gs", [16, 64])
def test_channels_last_equals_nchw(gs, dev):
    import dwt_b200
    x, dy = mixed((16, 128, 16, 16), dev), iid((16, 128, 16, 16), dev, seed=5, shift=0.0)
    a, b = dwt_b200.ZCAWTransform2d(128, gs).to(dev), dwt_b200.ZCAWTransform2d(128, gs).to(dev)
    y0, dx0 = _fwd_bwd(a, x, dy)
    cl = torch.channels_last
    y1, dx1 = _fwd_bwd(b, x.contiguous(memory_format=cl), dy.contiguous(memory_format=cl))
    assert y1.is_contiguous(memory_format=cl) and dx1.is_contiguous(memory_format=cl)
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    assert torch.equal(a.running_variance, b.running_variance)


@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_bf16_equals_float32_on_widened_input(layout, dev):
    import dwt_b200
    from dwt_b200 import _native as nv
    x, dy = mixed((16, 128, 16, 16), dev).bfloat16(), iid((16, 128, 16, 16), dev, seed=5, shift=0.0).bfloat16()
    if layout == "nhwc":
        x, dy = x.contiguous(memory_format=torch.channels_last), dy.contiguous(memory_format=torch.channels_last)
    a, b = dwt_b200.ZCAWTransform2d(128, 32).to(dev), dwt_b200.ZCAWTransform2d(128, 32).to(dev)
    nv.profile_begin()
    y16, dx16 = _fwd_bwd(a, x, dy)
    fam = families(nv.profile_end())
    assert {"dense_fwd_zca_bf16", "dense_bwd_zca_bf16"} <= fam, fam
    y32, dx32 = _fwd_bwd(b, x.float(), dy.float())
    assert y16.dtype == torch.bfloat16 and torch.equal(y16, y32.bfloat16()) and torch.equal(dx16, dx32.bfloat16())
    assert torch.equal(a.running_variance, b.running_variance)


def test_bf16_nchw_hw_not_multiple_of_8_upcasts(dev):
    import dwt_b200
    from dwt_b200 import _native as nv
    x = mixed((120, 64, 6, 6), dev).bfloat16()                               # HW 36: a multiple of 4, not of 8
    m = dwt_b200.ZCAWTransform2d(64, 32).to(dev)
    nv.profile_begin()
    y = m(x)
    fam = families(nv.profile_end())
    assert y.dtype == torch.bfloat16 and "dense_fwd_zca" in fam and "dense_fwd_zca_bf16" not in fam, fam


def test_reruns_and_graph_replay_are_bit_identical(dev):
    import dwt_b200
    x, dy = mixed((16, 128, 16, 16), dev), iid((16, 128, 16, 16), dev, seed=5, shift=0.0)
    m = dwt_b200.ZCAWTransform2d(128, 64).to(dev)
    outs = []
    for _ in range(2):
        m.running_mean.zero_()
        m.running_variance.fill_(1.0)
        outs.append(_fwd_bwd(m, x, dy) + (m.running_variance.clone(),))
    assert all(torch.equal(p, q) for p, q in zip(*outs))
    m, m_eager = dwt_b200.ZCAWTransform2d(128, 64).to(dev), dwt_b200.ZCAWTransform2d(128, 64).to(dev)
    leaf = x.clone().requires_grad_(True)

    def step(mod):
        y = mod(leaf)
        (dx,) = torch.autograd.grad(y, leaf, dy)
        return y, dx

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(m)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        step(m_eager)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y_g, dx_g = step(m)
    g.replay()
    torch.cuda.synchronize()
    y_e, dx_e = step(m_eager)
    assert torch.equal(y_g, y_e) and torch.equal(dx_g, dx_e)
    assert torch.equal(m.running_variance, m_eager.running_variance) and torch.equal(m.running_mean, m_eager.running_mean)


# --------------------------------------------------------------------------- 4. failure handling and refusals
def test_nan_group_sets_status_and_skips_ema(dev):
    import dwt_b200
    from dwt_b200 import _native as nv
    x = mixed((16, 128, 16, 16), dev)
    x[3, 70] = float("nan")                                                   # group 1 of 2 at group size 64
    m = dwt_b200.ZCAWTransform2d(128, 64).to(dev)
    rv0 = m.running_variance.clone()
    nv.clear_status(dev)
    y = m(x)
    torch.cuda.synchronize()
    assert nv.status(dev) & nv.STATUS_NOT_PD
    assert torch.equal(m.running_variance[1], rv0[1]) and not torch.equal(m.running_variance[0], rv0[0])
    assert torch.isfinite(y[:, :64]).all()
    with pytest.raises(dwt_b200.NotPositiveDefiniteError):
        nv.check_status(dev)
    nv.raise_on_status(1)
    try:
        with pytest.raises(dwt_b200.NotPositiveDefiniteError):
            m(x)
    finally:
        nv.raise_on_status(0)
        nv.clear_status(dev)


@pytest.mark.parametrize("c, gs, shape, cl", [
    (64, 4, (8, 64, 32, 32), False), (64, 2, (8, 64, 32, 32), True), (64, 1, (8, 64, 32, 32), False),
    (256, 128, (8, 256, 32, 32), False),
    (64, 64, (512, 64, 4, 4), False),                                          # HW 16: only the tiled kernels
    (64, 64, (64, 64, 6, 6), True),                                            # N*HW < 4096
    (64, 32, (512, 64, 2, 17), False),                                         # HW % 4 != 0
])
def test_refusals(c, gs, shape, cl, dev):
    import dwt_b200
    x = torch.randn(shape, device=dev)
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    with pytest.raises(dwt_b200._native.NativeError, match="ZCA basis|tensor-core"):
        dwt_b200.ZCAWTransform2d(c, gs).to(dev)(x)


# --------------------------------------------------------------------------- 5. fused site
@pytest.mark.parametrize("layout", ["shared", "distinct"])
def test_domain_site_equals_three_module_calls(layout, dev, worst):
    import dwt_b200
    x = mixed((3 * 16, 128, 16, 16), dev)
    dy = iid(x.shape, dev, seed=9, shift=0.0)
    ra = (torch.zeros(1, 128, 1, 1, device=dev), torch.eye(32, device=dev).repeat(4, 1, 1))
    bufs = {"shared": [ra] * 3, "distinct": [(ra[0].clone(), ra[1].clone()) for _ in range(3)]}[layout]
    clone = {id(b): (b[0].clone(), b[1].clone()) for b in bufs}
    mk = lambda rs: [dwt_b200.ZCAWTransform2d(128, 32, running_m=a, running_var=b).to(dev) for a, b in rs]   # noqa: E731
    site_mods, seq_mods = mk(bufs), mk([clone[id(b)] for b in bufs])
    xs = x.clone().requires_grad_(True)
    ys = dwt_b200.DomainTripleNorm("whiten", 128, 32)(xs, site_mods, None, None)
    (dxs,) = torch.autograd.grad(ys, xs, dy)
    xq = x.clone().requires_grad_(True)
    yq = torch.cat([seq_mods[k](xq[16 * k:16 * (k + 1)]) for k in range(3)])
    (dxq,) = torch.autograd.grad(yq, xq, dy)
    check(worst, f"site vs modules {layout}", "y", ys.detach(), yq.detach(), 1e-5)
    check(worst, f"site vs modules {layout}", "dx", dxs, dxq, 1e-5)
    for a, b in zip(site_mods, seq_mods):
        check(worst, f"site vs modules {layout}", "running_var", a.running_variance, b.running_variance, 1e-6)


def test_domain_site_replicated_and_fork(dev):
    import dwt_b200
    x = mixed((16, 128, 16, 16), dev)
    site = dwt_b200.DomainTripleNorm("whiten", 128, 32)
    mods = [dwt_b200.ZCAWTransform2d(128, 32).to(dev) for _ in range(3)]
    ref = [dwt_b200.ZCAWTransform2d(128, 32).to(dev) for _ in range(3)]
    with torch.no_grad():
        site(x, mods, None, None, replicated=True)
        for m in ref:
            m(x)
    for a, b in zip(mods, ref):
        assert torch.allclose(a.running_variance, b.running_variance, rtol=1e-5, atol=1e-6)
    xg = mixed((48, 128, 16, 16), dev).requires_grad_(True)
    y = site(xg, mods, None, None)
    a, b = dwt_b200.fork_for_sum(y)
    (g1,) = torch.autograd.grad((a * 2 + b).sum(), xg)
    y = site(xg, mods, None, None)
    (g2,) = torch.autograd.grad((y * 3).sum(), xg)
    assert torch.allclose(g1, g2, rtol=1e-4, atol=1e-5)


# --------------------------------------------------------------------------- 6. model
def test_conv_zca_conv_training_step(dev, worst):
    """conv(64 -> 256, 3x3) -> ZCAWTransform2d(256, 64) -> conv(256 -> 32, 1x1): loss and every parameter gradient of one
    training step against the same network in float64 on the ATen restatement."""
    import dwt_b200
    torch.manual_seed(0)
    c1 = torch.nn.Conv2d(64, 256, 3, padding=1, bias=False).to(dev)
    c2 = torch.nn.Conv2d(256, 32, 1, bias=False).to(dev)
    norm = dwt_b200.ZCAWTransform2d(256, 64).to(dev)
    x = torch.randn(32, 64, 16, 16, device=dev)
    target = torch.randn(32, 32, 16, 16, device=dev)
    loss = ((c2(norm(c1(x))) - target) ** 2).mean()
    g = torch.autograd.grad(loss, [c1.weight, c2.weight])
    w1, w2 = c1.weight.detach().double().requires_grad_(True), c2.weight.detach().double().requires_grad_(True)
    h, *_ = Z.zca_torch(torch.nn.functional.conv2d(x.double(), w1, padding=1), 64, 5)
    loss_r = ((torch.nn.functional.conv2d(h, w2) - target.double()) ** 2).mean()
    gr = torch.autograd.grad(loss_r, [w1, w2])
    check(worst, "conv-zca-conv", "loss", loss.detach().reshape(1), loss_r.detach().reshape(1))
    check(worst, "conv-zca-conv", "dconv1", g[0], gr[0])
    check(worst, "conv-zca-conv", "dconv2", g[1], gr[1])
