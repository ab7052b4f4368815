"""Whitening at group size 128 (two 64-channel super-blocks per group) on the tensor-core kernels, fp32, NCHW and
channels-last, against the fp64 reference and against itself.

fp64 comparisons run through the site harness of test_nchw_fp64.py (loaded from its file, not modified): the
reference's operator sequence (oracle/torch_port.py) in float64, one domain and one slab of whole groups at a time,
with the same tolerances -- 1e-3 norm-wise on outputs and gradients, 1e-4 on statistics and running buffers, the
max-elementwise error below 5x the bound -- and the launch profile asserting that the tensor-core family (tc_*) ran.

Cases: BASELINE config 2 (N=256 C=256 56^2) at full size; C = 128 / 256 / 384 / 512; HW = 32 / 36 / 40 (a partial
64-pixel apply tile) / 3136; N*HW = 4096 exactly; fewer tiles than CTAs; 1-4 domains on shared, distinct and mixed
running buffers in train / no-grad / eval / default-buffer modes via the module and DomainTripleNorm, and replicated=True;
the pilot-shift inputs; an ill-conditioned covariance next to the same input at group size 64.  Then: channels-last ==
NCHW bit for bit, determinism, CUDA-graph replay, DWT_STATUS_NOT_PD from a NaN group, the C ABI's refusals, the bf16
routes, and a conv -> WTransform2d(256, 128) -> conv model against an fp64 training step.
"""
import ctypes
import importlib.util
import math
import os

import pytest
import torch

_spec = importlib.util.spec_from_file_location("_nchw_fp64_harness", os.path.join(os.path.dirname(__file__), "test_nchw_fp64.py"))
H = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(H)

GS = 128
TC_CH = 64                  # channels of a tensor-core super-block: a group of 128 spans two
TC_MIN_M = 4096             # N * HW per domain the tensor-core kernels need
TC_BOX = 32                 # HW >= one TMA box of pixels
TC_CTAS_PER_SM = 2          # contraction CTAs per SM over the (domain, super-block) problems


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
    table = {}
    yield table
    print("\nworst errors at group size 128 (norm-wise, max-elementwise):")
    for key in sorted(table):
        print("  %-20s %s" % (" / ".join(key), ", ".join(f"{k} {r:.1e} {m:.1e}" for k, (r, m) in sorted(table[key].items()))))


def _families(prof):
    return {k.split("|")[0] for k in prof}


# --------------------------------------------------------------------------- 1. fp64 reference
@pytest.mark.gpu
def test_config2_full_size(dev, worst):
    """BASELINE config 2 (N=256 C=256 56^2, M = 802,816 samples per channel) at group size 128: train forward + backward
    and the EMA on default-constructed buffers, input built as bench.py's microbench builds it."""
    H._check(dev, worst, "config2 gs128", "config2", gs=GS, family="tc", make_x=H._microbench, **H.MICRO)


def _edges(sms):
    """(label, C, D, N, (H, W), layout)"""
    few = sms // 4                                           # 128-pixel images: 4 tiles each, fewer tiles than CTAs
    return [
        ("c128", 128, 1, 16, (16, 16), "shared"),
        ("c256_d2", 256, 2, 16, (16, 16), "distinct"),
        ("c384_d3", 384, 3, 8, (24, 24), "mixed"),
        ("c512", 512, 1, 12, (20, 20), "shared"),
        ("hw32", 256, 1, 160, (4, 8), "shared"),
        ("hw36", 128, 2, 120, (6, 6), "distinct"),
        ("hw40_partial_apply_tile", 256, 1, 120, (5, 8), "shared"),
        ("hw3136", 128, 1, 8, (56, 56), "shared"),
        ("m4096", 256, 1, TC_MIN_M // 32, (4, 8), "shared"),
        ("few_tiles", 128, 1, few, (8, 16), "shared"),
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(10), ids=[e[0] for e in _edges(132)])
def test_shapes(case, dev, sms, worst):
    label, c, d, n, hw, layout = _edges(sms)[case]
    m = n * hw[0] * hw[1]
    assert m >= TC_MIN_M and hw[0] * hw[1] >= TC_BOX and hw[0] * hw[1] % 4 == 0
    if label == "m4096":
        assert m == TC_MIN_M
    if label == "few_tiles":
        assert n * (hw[0] * hw[1] // TC_BOX) < TC_CTAS_PER_SM * sms
    H._check(dev, worst, label, "shapes", kind="whiten", c=c, gs=GS, d=d, n=n, spatial=hw, family="tc", layout=layout,
             via="site", epi="relu", seed=c + d + n)


@pytest.mark.gpu
@pytest.mark.parametrize("d,layout,mode,via", H.MODES, ids=[f"d{m[0]}-{m[1]}-{m[2]}-{m[3]}" for m in H.MODES])
def test_modes_and_domains(d, layout, mode, via, dev, worst):
    """fwd_factor128's ordered domain loop on shared, distinct and mixed buffers, in every mode."""
    H._check(dev, worst, f"d{d} {layout} {mode} {via}", "modes", kind="whiten", c=256, gs=GS, d=d, n=8, spatial=(24, 24),
             family="tc", mode=mode, layout=layout, via=via, epi=None if via == "module" else "affine", seed=d + len(mode))


@pytest.mark.gpu
@pytest.mark.parametrize("make", ["pilot_30sigma", "mean_50sigma"])
def test_pilot_shift_inputs(make, dev, worst):
    base = H._activation
    make_x = H._pilot_window(base) if make == "pilot_30sigma" else H._mean_50sigma(base)
    H._check(dev, worst, make, "pilot", kind="whiten", c=256, gs=GS, d=2, n=32, spatial=(28, 28), family="tc",
             layout="distinct", via="site", epi=None, make_x=make_x, seed=7)


@pytest.mark.gpu
def test_replicated_site(dev):
    """DomainTripleNorm(replicated=True) at group size 128: one batch stands for the three branches; equals each module
    called on it, running buffers included."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(3)
    x = H._activation(gen, (16, 256, 16, 16), 1, dev)
    mods = [dwt_b200.WTransform2d(256, GS).to(dev).train() for _ in range(3)]
    ref = [dwt_b200.WTransform2d(256, GS).to(dev).train() for _ in range(3)]
    g = torch.ones(256, 1, 1, device=dev)
    b = torch.zeros(256, 1, 1, device=dev)
    site = dwt_b200.DomainTripleNorm("whiten", 256, GS)
    out = site(x, mods, g, b, replicated=True)
    want = [r(x) for r in ref]
    for w in want:
        assert torch.equal(w, want[0])
    err = (out - want[0]).norm() / want[0].norm()
    assert err < 1e-6, err.item()
    for m, r in zip(mods, ref):
        assert torch.allclose(m.running_variance, r.running_variance, rtol=1e-5, atol=1e-6)


def _ill_conditioned(gen, shape, d, dev, scale_hi=10.0, scale_lo=0.01):
    """Channels mixed by a random orthogonal matrix per 128-channel group with standard deviations log-spaced from
    scale_hi to scale_lo: covariance eigenvalues 1e2 .. 1e-4."""
    n, c, h, w = shape
    s = torch.logspace(math.log10(scale_hi), math.log10(scale_lo), GS, device=dev, dtype=torch.float64)
    z = torch.randn(n, c, h * w, device=dev, generator=gen, dtype=torch.float64)
    out = torch.empty_like(z)
    for g in range(c // GS):
        q, _ = torch.linalg.qr(torch.randn(GS, GS, device=dev, generator=gen, dtype=torch.float64))
        out[:, g * GS:(g + 1) * GS] = torch.einsum("ij,njp->nip", q * s, z[:, g * GS:(g + 1) * GS])
    return (out + 1.0).float().view(shape)


@pytest.mark.gpu
def test_ill_conditioned_covariance(dev):
    """Covariance eigenvalues spanning 1e6: the shrunk S = 0.999 cov + 1e-3 I has condition number 9.4e4 at group size
    128 and 6.9e3 in the 64-channel halves the same input forms at group size 64.  On an H100 the worst norm-wise errors
    were y 4.0e-4, dx 1.0e-3, W 3.5e-4 at 128 against y 2.9e-5, dx 1.3e-4, W 1.5e-4 at 64: per unit of condition number
    the two group sizes are alike, which is what is asserted.  W is compared with LAPACK's fp64 inverse Cholesky factor
    of the kernel's own covariance (recovered from the running buffer, momentum 1)."""
    import dwt_b200
    import oracle.torch_port as port
    gen = torch.Generator(device=dev).manual_seed(11)
    shape = (64, 256, 16, 16)
    x = _ill_conditioned(gen, shape, 1, dev)
    dy = torch.randn(shape, device=dev, generator=gen)
    res = {}
    for gs in (64, GS):
        m = dwt_b200.WTransform2d(256, gs, momentum=1.0).to(dev).train()
        xt = x.clone().requires_grad_(True)
        y = m(xt)
        y.backward(dy)
        x64 = x.double().requires_grad_(True)
        ref = port.WTransform2d(256, gs, momentum=1.0).to(dev).double().train()
        y64 = ref(x64)
        y64.backward(dy.double())
        cov = m.running_variance.double()
        s = 0.999 * cov + 1e-3 * torch.eye(gs, dtype=torch.float64, device=dev)
        cond = torch.linalg.cond(s).max().item()
        w64 = torch.linalg.inv(torch.linalg.cholesky(s))
        records = []
        with H._record_saved_stats(records), torch.no_grad():
            dwt_b200.WTransform2d(256, gs, running_m=m.running_mean.clone(), running_var=m.running_variance.clone()).to(dev).eval()(x)
        wk = records[0][1][0].double()
        res[gs] = dict(cond=cond, y=((y.double() - y64).norm() / y64.norm()).item(),
                       dx=((xt.grad.double() - x64.grad).norm() / x64.grad.norm()).item(),
                       w=((wk - w64).norm() / w64.norm()).item())
    print("ill-conditioned covariance:", res)
    assert res[GS]["cond"] > 1e4
    for k in ("y", "dx", "w"):
        # error per unit of condition number no worse than twice group size 64's on the same input; bounded outright
        assert res[GS][k] / res[GS]["cond"] < 2 * res[64][k] / res[64]["cond"] and res[GS][k] < 1e-2, (k, res)


# --------------------------------------------------------------------------- 2. layouts, determinism, graphs
def _run(mod_state, x, dy, cl):
    """One train forward + backward of a fresh WTransform2d(C, 128) from mod_state -> (y, dx, running buffers)."""
    import dwt_b200
    c = x.shape[1]
    m = dwt_b200.WTransform2d(c, GS, running_m=mod_state[0].clone(), running_var=mod_state[1].clone()).to(x.device).train()
    fmt = torch.channels_last if cl else torch.contiguous_format
    dy = dy.contiguous(memory_format=fmt)
    xt = x.detach().clone(memory_format=fmt).requires_grad_(True)
    y = m(xt)
    y.backward(dy)
    return y.detach(), xt.grad, m.running_mean.clone(), m.running_variance.clone()


def _state(c, dev, gen):
    a = torch.randn(c // GS, GS, GS, device=dev, generator=gen)
    return 0.1 * torch.randn(1, c, 1, 1, device=dev, generator=gen), a @ a.mT / GS + 0.5 * torch.eye(GS, device=dev)


LAYOUT_CASES = [(256, 8, (56, 56)), (128, 160, (4, 8)), (256, 120, (5, 8)), (384, 8, (24, 24)), (512, 12, (20, 20))]


@pytest.mark.gpu
@pytest.mark.parametrize("c,n,hw", LAYOUT_CASES, ids=[f"c{c}_n{n}_{h}x{w}" for c, n, (h, w) in LAYOUT_CASES])
def test_channels_last_equals_nchw_and_determinism(c, n, hw, dev):
    from dwt_b200 import _native
    gen = torch.Generator(device=dev).manual_seed(c + n)
    x = H._activation(gen, (n, c, *hw), 1, dev)
    dy = torch.randn(x.shape, device=dev, generator=gen)
    st = _state(c, dev, gen)
    _native.clear_status(dev)
    _native.profile_begin()
    a = _run(st, x, dy, False)
    fam_nchw = _families(_native.profile_end())
    _native.profile_begin()
    b = _run(st, x, dy, True)
    fam_nhwc = _families(_native.profile_end())
    a2 = _run(st, x, dy, False)
    assert {"tc_stats", "tc_apply", "tc_bwd_reduce", "tc_bwd_apply"} <= fam_nchw and not any(f.startswith("tiled") for f in fam_nchw)
    assert {"tc_stats_nhwc", "tc_apply_nhwc", "tc_bwd_reduce_nhwc", "tc_bwd_apply_nhwc"} <= fam_nhwc, fam_nhwc
    assert b[0].is_contiguous(memory_format=torch.channels_last) and b[1].is_contiguous(memory_format=torch.channels_last)
    for u, v, w in zip(a, b, a2):
        assert torch.equal(u, v.contiguous())
        assert torch.equal(u, w)
    assert _native.status(dev) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "nhwc"])
def test_cuda_graph_replay(cl, dev):
    """Capture forward + backward (a fresh leaf per step, as tools/cl_tc_micro.py does), replay, compare with eager."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(5)
    fmt = torch.channels_last if cl else torch.contiguous_format
    x = H._activation(gen, (16, 256, 16, 16), 1, dev).contiguous(memory_format=fmt)
    dy = torch.randn(x.shape, device=dev, generator=gen).contiguous(memory_format=fmt)
    m = dwt_b200.WTransform2d(256, GS).to(dev).train()
    m_eager = dwt_b200.WTransform2d(256, GS).to(dev).train()
    xs, dys = x.clone(memory_format=fmt), dy.clone(memory_format=fmt)

    def step(mod):
        leaf = xs.detach().requires_grad_(True)
        y = mod(leaf)
        (dx,) = torch.autograd.grad(y, leaf, dys)
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


# --------------------------------------------------------------------------- 3. status
@pytest.mark.gpu
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "nhwc"])
def test_nan_group_sets_not_pd(cl, dev):
    """A NaN in group 1 of 2: DWT_STATUS_NOT_PD, only group 1's outputs are NaN, only group 0's running buffers move."""
    import dwt_b200
    from dwt_b200 import _native
    gen = torch.Generator(device=dev).manual_seed(9)
    x = H._activation(gen, (16, 256, 16, 16), 1, dev)
    x[3, GS + 5, 2, 2] = float("nan")
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    m = dwt_b200.WTransform2d(256, GS).to(dev).train()
    rm0, rv0 = m.running_mean.clone(), m.running_variance.clone()
    _native.clear_status(dev)
    y = m(x)
    assert _native.status(dev) & _native.STATUS_NOT_PD
    _native.clear_status(dev)
    assert torch.isfinite(y[:, :GS]).all() and torch.isnan(y[:, GS:]).all()
    assert not torch.equal(m.running_variance[0], rv0[0]) and torch.equal(m.running_variance[1], rv0[1])
    assert torch.equal(m.running_mean[:, GS:], rm0[:, GS:]) and not torch.equal(m.running_mean[:, :GS], rm0[:, :GS])


# --------------------------------------------------------------------------- 4. C ABI refusals and routing
def _abi_fwd(dev, n, c, hw, gs, *, mode=0, epi=0, x_off=0, bf16=False):
    from dwt_b200 import _native as nv
    lib = nv.lib()
    dt = torch.bfloat16 if bf16 else torch.float32
    store = torch.randn(n * c * hw + 8, device=dev).to(dt)
    x = store[x_off:x_off + n * c * hw]
    y = torch.empty(n * c * hw + 8, device=dev, dtype=dt)[x_off:x_off + n * c * hw]
    gb = torch.ones(c, device=dev)
    save_mean = torch.empty(c, device=dev)
    save_w = torch.empty(c * max(gs, 1), device=dev)
    ws_gs = gs if gs in (GS,) or gs <= 64 else 64
    ws = nv.workspace(dev, n, c, hw, ws_gs, 1)
    rc = lib.dwt_whiten_fwd(nv.ptr(x), nv.ptr(y), n, c, hw, gs, 1, mode | (nv.DTYPE_BF16 if bf16 else 0), 1e-3, 0.1, 0,
                            None, None, nv.ptr(gb) if epi else None, nv.ptr(gb) if epi else None, None, None, epi,
                            nv.ptr(save_mean), nv.ptr(save_w), nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
    torch.cuda.synchronize(dev)
    return rc, lib.dwt_last_error().decode()


@pytest.mark.gpu
def test_abi_codes(dev):
    from dwt_b200 import _native as nv
    assert nv.lib().dwt_abi_version() == 10
    assert _abi_fwd(dev, 16, 256, 256, GS)[0] == 0
    assert _abi_fwd(dev, 16, 256, 256, GS, mode=nv.LAYOUT_NHWC)[0] == 0
    assert _abi_fwd(dev, 16, 256, 256, GS, mode=nv.LAYOUT_NHWC, x_off=1)[0] == -1          # misaligned channels-last
    for kw in (dict(epi=nv.EPI_AFFINE), dict(bf16=True), dict(bf16=True, mode=nv.LAYOUT_NHWC)):
        assert _abi_fwd(dev, 16, 256, 256, GS, **kw)[0] == -4, kw
    for gs in (96, 192, 256):
        rc, msg = _abi_fwd(dev, 16, 768, 256, gs)
        assert rc == -4 and "group_size" in msg, (gs, rc, msg)
    for n, hw, off in ((2, 16, 0), (160, 34, 0), (127, 32, 0), (16, 256, 1)):   # HW < 32, HW % 4, N*HW < 4096, vec != 4
        rc, msg = _abi_fwd(dev, n, 256, hw, GS, x_off=off)
        assert rc == -4 and "group_size" in msg, (n, hw, off, rc, msg)
    # dout2 at group size 128 is refused like at 8..64
    lib = nv.lib()
    n, c, hw = 16, 256, 256
    t = [torch.randn(n * c * hw, device=dev) for _ in range(4)]
    sm, sw = torch.zeros(c, device=dev), torch.zeros(c * GS, device=dev)
    ws = nv.workspace(dev, n, c, hw, GS, 1)
    rc = lib.dwt_whiten_bwd(nv.ptr(t[0]), nv.ptr(t[1]), nv.ptr(t[2]), nv.ptr(t[3]), n, c, hw, GS, 1, 0, 1e-3, nv.ptr(sm), nv.ptr(sw),
                            None, None, None, None, 0, None, None, nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
    assert rc == -4
    assert lib.dwt_workspace_bytes(n, c, hw, GS, 1) == 0 and lib.dwt_workspace_bytes(n, 768, hw, 96, 1) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "nhwc"])
def test_bf16_upcasts(cl, dev):
    """A bf16 call at group size 128 under autocast runs the fp32 kernels on x.float() (channels-last stays
    channels-last) and equals them rounded to bf16; no bf16 kernel family is launched."""
    import dwt_b200
    from dwt_b200 import _native
    gen = torch.Generator(device=dev).manual_seed(21)
    x = H._activation(gen, (16, 256, 16, 16), 1, dev).bfloat16()
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    m1, m2 = dwt_b200.WTransform2d(256, GS).to(dev).train(), dwt_b200.WTransform2d(256, GS).to(dev).train()
    _native.profile_begin()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = m1(x)
    fams = _families(_native.profile_end())
    want = m2(x.float()).to(torch.bfloat16)
    assert y.dtype == torch.bfloat16 and torch.equal(y, want)
    assert not any(f.endswith("_bf16") for f in fams), fams
    assert ("tc_apply_nhwc" if cl else "tc_apply") in fams, fams


@pytest.mark.gpu
def test_model_training_matches_fp64(dev):
    """conv -> WTransform2d(256, 128) -> conv, three SGD steps, against the same model in float64 on the reference layer."""
    import dwt_b200
    import oracle.torch_port as port
    torch.manual_seed(0)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # the convolutions in full fp32: the comparison is of the norm layer
    try:
        _train_three_steps(dev, dwt_b200, port)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _train_three_steps(dev, dwt_b200, port):
    def model(norm, dtype):
        m = torch.nn.Sequential(torch.nn.Conv2d(16, 256, 3, padding=1), norm, torch.nn.Conv2d(256, 8, 1))
        return m.to(dev, dtype)
    a = model(dwt_b200.WTransform2d(256, GS), torch.float32)
    b = model(port.WTransform2d(256, GS), torch.float64)
    b.load_state_dict({k: v.double() for k, v in a.state_dict().items()})
    oa, ob = torch.optim.SGD(a.parameters(), lr=0.05), torch.optim.SGD(b.parameters(), lr=0.05)
    gen = torch.Generator(device=dev).manual_seed(1)
    for step in range(3):
        x = torch.randn(32, 16, 16, 16, device=dev, generator=gen)
        t = torch.randn(32, 8, 16, 16, device=dev, generator=gen)
        for m, o, dt in ((a, oa, torch.float32), (b, ob, torch.float64)):
            o.zero_grad()  # noqa
            loss = (m(x.to(dt)) - t.to(dt)).square().mean()
            loss.backward()
        for (k, pa), pb in zip(a.named_parameters(), b.parameters()):
            if k == "0.bias":            # a per-channel shift before whitening: its gradient is zero up to rounding
                assert pa.grad.abs().max() < 1e-6 * a[0].weight.grad.abs().max(), step
                continue
            err = ((pa.grad.double() - pb.grad).norm() / pb.grad.norm()).item()
            assert err < 1e-3, (step, k, err)
        oa.step()
        ob.step()
        for (k, pa), pb in zip(a.named_parameters(), b.parameters()):
            err = ((pa.double() - pb).norm() / pb.norm()).item()
            assert err < 1e-4, (step, k, err)
    for k in ("1.running_mean", "1.running_variance"):
        va, vb = a.state_dict()[k].double(), b.state_dict()[k]
        assert ((va - vb).norm() / vb.norm()).item() < 1e-4, k


# --------------------------------------------------------------------------- 5. Python mirrors (no GPU)
def test_python_routing_mirrors():
    from dwt_b200 import _native as nv
    assert nv.tensor_core_nhwc_supported(16, 256, 256, GS)
    assert not nv.tensor_core_nhwc_supported(16, 192, 256, GS)          # C not a multiple of 128
    assert not nv.tensor_core_nhwc_supported(2, 256, 16, GS)
    assert not nv.tensor_core_nhwc_supported(16, 768, 256, 96)
    assert not nv.tensor_core_bf16_supported(16, 256, 256, GS)


def test_workspace_rule_covers_group_size_128():
    """dwt_workspace_bytes keeps its range (0 at group size 128, as at 96 / 192 / 256); a group-size-128 call on C
    channels is sized by the group-size-64 query on 2C channels (dwt_b200.h, _native.workspace).  The forward call
    reports what it needs ("need N bytes", DWT_E_WORKSPACE) before it touches any memory, so this runs without a GPU;
    the geometries include more problems than two waves of CTAs."""
    import re
    from dwt_b200 import _native as nv
    lib = nv.lib()
    for gs in (96, GS, 192, 256):
        assert lib.dwt_workspace_bytes(64, 768, 3136, gs, 1) == 0
    fake = ctypes.c_void_p(1 << 20)                   # never dereferenced: the call stops at the workspace check
    for n, c, hw, d in ((256, 256, 3136, 1), (8, 128, 1024, 4), (64, 512, 256, 3), (1, 16384, 4096, 4), (64, 32768, 64, 2)):
        for layout in (0, nv.LAYOUT_NHWC):
            rc = lib.dwt_whiten_fwd(fake, fake, n, c, hw, GS, d, layout, 1e-3, 0.1, 0, None, None, None, None, None, None, 0,
                                    fake, fake, fake, 1, None)
            msg = lib.dwt_last_error().decode()
            assert rc == -2, (n, c, hw, d, rc, msg)
            need = int(re.search(r"need (\d+) bytes", msg).group(1))
            rule = lib.dwt_workspace_bytes(n, 2 * c, hw, 64, d)
            assert 0 < need <= rule, (n, c, hw, d, need, rule)
