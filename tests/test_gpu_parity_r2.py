"""GPU parity, round 2: the holes the round-1 suite left (VERDICT r1 "what's weak").

  * tensor-core (TMA + wgmma) path in EVERY mode -- train with external buffers, no-grad train (statistics
    collection), eval forward + backward, default buffers -- at M = N*H*W >= 4096, where tc_supports() really
    routes to it (the round-1 goldens for gs >= 8 have M = 108..144 and take the tiled FFMA path);
  * ill-conditioned and far-from-zero-mean inputs on that path: cond(Sigma) ~ 1e3 at activation scale 10 (so the
    eps = 1e-3 shrinkage does not hide the conditioning) and |mean| / sigma = 50;
  * the whole reference model at the REAL site shapes (3 x 4 images of 224 x 224: 112^2 / 56^2 / 28^2 / 14^2 / 7^2),
    golden made by tests/golden/make_golden.py from the unmodified reference;
  * every comparison reports the max-elementwise error next to the norm-wise one;
  * failure surfacing: raise_on_status(), label validation of the head loss, pointer-argument validation.

Tolerances as in test_gpu_parity.py: 1e-3 norm-wise through a Cholesky factor (BASELINE.json), 1e-4 on plain
statistics; max-elementwise error (scaled by max|ref|) below 5x the norm-wise bound.
"""
import os

import numpy as np
import pytest
import torch

from conftest import max_err, rel_err
from oracle import dwt_oracle as O

pytestmark = pytest.mark.gpu

TOL = 1e-3
TOL_STAT = 1e-4
TOL_MAX = 5e-3
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda", 0)


def t(a, dev):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device=dev)


def n(a):
    return a.detach().double().cpu().numpy()


def both(a, b):
    return rel_err(a, b), max_err(a, b)


def _correlated(rng, nimg, c, h, w, offset=2.0):
    z = rng.standard_normal((nimg, c, h, w))
    mix = rng.standard_normal((c, c)) / np.sqrt(c) + np.eye(c)
    return np.einsum("dc,nchw->ndhw", mix, z) + offset


def _spd(rng, g, gs):
    a = rng.standard_normal((g, gs, gs))
    return a @ a.transpose(0, 2, 1) / gs + 0.5 * np.eye(gs)


# N, C, H, W, gs -- all with N*H*W >= 4096 and HW % 4 == 0, HW >= 32: the wgmma path (norm_tc.cu tc_supports)
TC_CASES = [(6, 128, 28, 28, 64), (20, 192, 16, 16, 8), (12, 64, 20, 20, 32), (48, 48, 10, 10, 16)]


@pytest.mark.parametrize("case", TC_CASES, ids=lambda c: "n{}c{}h{}w{}g{}".format(*c))
def test_tensor_core_path_all_modes(case, dev):
    import whitening
    nimg, c, h, w, gs = case
    assert nimg * h * w >= 4096 and (h * w) % 4 == 0
    rng = np.random.default_rng(1000 + c + gs)
    x1, x2 = _correlated(rng, nimg, c, h, w), _correlated(rng, nimg, c, h, w, offset=-1.0)
    dy = rng.standard_normal(x1.shape)
    rm0, rv0 = 0.1 * rng.standard_normal(c), _spd(rng, c // gs, gs)
    m = whitening.WTransform2d(c, gs, running_m=t(rm0.reshape(1, c, 1, 1), dev), running_var=t(rv0, dev)).train()
    # (1) train, external buffers, forward + backward + EMA
    y_o, mean_o, w_o, rm1, rv1, _ = O.whiten_forward(x1, gs, running_mean=rm0, running_cov=rv0)
    xt = t(x1, dev).requires_grad_(True)
    y = m(xt)
    (dx,) = torch.autograd.grad(y, xt, t(dy, dev))
    e = dict(y=both(n(y), y_o), dx=both(n(dx), O.whiten_backward(x1, dy, mean_o, w_o)),
             rm=both(n(m.running_mean).reshape(-1), rm1), rv=both(n(m.running_variance), rv1))
    # (2) train under no_grad (statistics collection, resnet50_dwt_mec_officehome.py:382-389): second EMA step
    y2_o, _, _, rm2, rv2, _ = O.whiten_forward(x2, gs, running_mean=rm1, running_cov=rv1)
    with torch.no_grad():
        y2 = m(t(x2, dev))
    e.update(y_nograd=both(n(y2), y2_o), rm2=both(n(m.running_mean).reshape(-1), rm2), rv2=both(n(m.running_variance), rv2))
    # (3) eval: running statistics, forward + backward (dx = W^T dy), buffers untouched
    m.eval()
    ye_o, _, we_o, *_ = O.whiten_forward(x1, gs, running_mean=rm2, running_cov=rv2, training=False)
    xe = t(x1, dev).requires_grad_(True)
    ye = m(xe)
    (dxe,) = torch.autograd.grad(ye, xe, t(dy, dev))
    e.update(y_eval=both(n(ye), ye_o), dx_eval=both(n(dxe), O.whiten_backward_eval(dy, we_o)),
             rm_after_eval=both(n(m.running_mean).reshape(-1), rm2))
    # (4) default-constructed buffers (zeros / all-ones matrix, whitening.py:23-24), one training step
    d = whitening.WTransform2d(c, gs).to(dev).train()
    with torch.no_grad():
        d(t(x1, dev))
    _, _, _, rmd, rvd, _ = O.whiten_forward(x1, gs, running_mean=np.zeros(c), running_cov=np.ones((c // gs, gs, gs)))
    e.update(rm_default=both(n(d.running_mean).reshape(-1), rmd), rv_default=both(n(d.running_variance), rvd))
    print(case, {k: ("%.2e" % v[0], "%.2e" % v[1]) for k, v in e.items()})
    for k, (rel, mx) in e.items():
        stat = k.startswith(("rm", "rv"))
        assert rel < (TOL_STAT if stat else TOL), (k, rel)
        assert mx < (5 * TOL_STAT if stat else TOL_MAX), (k, mx)
    from dwt_b200 import _native
    assert _native.status(dev) == 0


@pytest.mark.parametrize("case", [(64, 256, 28, 28, 64), (6, 128, 28, 28, 64), (5, 64, 30, 30, 8)],
                         ids=lambda c: "n{}c{}h{}w{}g{}".format(*c))
def test_tensor_core_path_is_run_to_run_identical(case, dev):
    """The TMA / transform / wgmma pipelines (two consumer warpgroups, ring barriers) hold no atomics and
    reduce their partials in a fixed order: 40 repetitions of forward + backward on one input must agree BIT FOR BIT --
    a stage or tensor-memory slot overwritten before its reader is done shows up here as a run that differs."""
    import whitening
    nimg, c, h, w, gs = case
    gen = torch.Generator(device=dev).manual_seed(7)
    x = (torch.randn(nimg, c, h, w, device=dev, generator=gen) * 1.5 + 0.7).requires_grad_(True)
    dy = torch.randn(nimg, c, h, w, device=dev, generator=gen)
    first = None
    for rep in range(40):
        m = whitening.WTransform2d(c, gs).to(dev).train()
        y = m(x)
        (dx,) = torch.autograd.grad(y, x, dy)
        got = (y.detach(), dx, m.running_mean.clone(), m.running_variance.clone())
        if first is None:
            first = [g.clone() for g in got]
            continue
        for name, a, b in zip(("y", "dx", "running_mean", "running_variance"), got, first):
            assert torch.equal(a, b), (name, rep, (a - b).abs().max().item())
    from dwt_b200 import _native
    assert _native.status(dev) == 0


def _conditioned(rng, nimg, c, h, w, gs, cond, scale, mean_over_sigma=0.0):
    """Channels whose per-group covariance has eigenvalues scale^2 * logspace(0, -log10(cond)) in a random
    orthogonal basis, plus a per-channel mean of mean_over_sigma standard deviations."""
    g = c // gs
    z = rng.standard_normal((nimg, g, gs, h * w))
    out = np.empty_like(z)
    for k in range(g):
        q, _ = np.linalg.qr(rng.standard_normal((gs, gs)))
        a = q * (scale * np.sqrt(np.logspace(0, -np.log10(cond), gs)))[None, :]
        out[:, k] = np.einsum("ij,njm->nim", a, z[:, k])
    x = out.reshape(nimg, c, h, w)
    sd = x.std(axis=(0, 2, 3), keepdims=True)
    sign = np.where(rng.random((1, c, 1, 1)) < 0.5, -1.0, 1.0)
    return x + mean_over_sigma * sd * sign


@pytest.mark.parametrize("name,case,cond,scale,mos", [
    ("cond1e3_scale10", (6, 128, 28, 28, 64), 1e3, 10.0, 0.0),
    ("cond1e3_scale10_g16", (48, 48, 10, 10, 16), 1e3, 10.0, 0.0),
    ("cond1e4_scale30", (6, 128, 28, 28, 64), 1e4, 30.0, 0.0),
    ("mean50sigma", (6, 128, 28, 28, 64), 1e1, 1.0, 50.0),
    ("mean50sigma_cond1e3", (12, 64, 20, 20, 32), 1e3, 10.0, 50.0),
])
def test_tensor_core_path_ill_conditioned(name, case, cond, scale, mos, dev):
    """The covariance contraction runs on tf32 tensor cores; the operands are split hi + lo so that the Gram matrix
    keeps ~fp32 accuracy (ADVICE r1: a single tf32 pass loses 1e-3 .. 5e-3 in y once eps stops regularising)."""
    import whitening
    nimg, c, h, w, gs = case
    rng = np.random.default_rng(abs(hash(name)) % (2 ** 31))
    x = _conditioned(rng, nimg, c, h, w, gs, cond, scale, mos)
    dy = rng.standard_normal(x.shape)
    y_o, mean_o, w_o, _, _, cov_o = O.whiten_forward(x, gs)
    dx_o = O.whiten_backward(x, dy, mean_o, w_o)
    m = whitening.WTransform2d(c, gs).to(dev).train()
    xt = t(x, dev).requires_grad_(True)
    y = m(xt)
    (dx,) = torch.autograd.grad(y, xt, t(dy, dev))
    # fp32 yardstick: the reference's own operator sequence in fp32 on this GPU (what "the reference layer outputs"
    # are at this conditioning) against the same fp64 oracle
    import oracle.torch_port as port
    r = port.WTransform2d(c, gs).to(dev).train()
    xr = t(x, dev).requires_grad_(True)
    yr = r(xr)
    (dxr,) = torch.autograd.grad(yr, xr, t(dy, dev))
    e = dict(y=both(n(y), y_o), dx=both(n(dx), dx_o), ref_y=both(n(yr), y_o), ref_dx=both(n(dxr), dx_o),
             y_vs_ref=both(n(y), n(yr)))
    print(name, {k: ("%.2e" % v[0], "%.2e" % v[1]) for k, v in e.items()})
    # within the bar against fp64, or -- where fp32 itself cannot hold 1e-3 at this conditioning -- no worse than
    # twice the fp32 reference
    assert e["y"][0] < max(TOL, 2 * e["ref_y"][0]), e
    assert e["dx"][0] < max(TOL, 2 * e["ref_dx"][0]), e
    assert e["y"][1] < max(TOL_MAX, 2 * e["ref_y"][1]), e


# --------------------------------------------------------------------------- whole model at the real site shapes
@pytest.mark.parametrize("fmt,site_mode,stem", [("nchw", "modules", "direct"), ("nchw", "fused", "direct"), ("nhwc", "fused", "direct"),
                                                ("nhwc", "fused", "s2d"), ("nchw", "fused", "s2d")])
def test_resnet_224_vs_reference_golden(fmt, site_mode, stem, dev):
    """Harness model + CUDA layers vs the UNMODIFIED reference ResNet (CPU fp32, tests/golden/make_golden.py) on
    3 x 4 images of 224 x 224: the site shapes of BASELINE configs[2] (stem 64 x 112^2 ... layer4 2048 x 7^2)."""
    import torch.nn.functional as Fn
    import dwt_b200
    import oracle.torch_port as port
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    z = np.load(os.path.join(HERE, "resnet_224.npz"))
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
    x, labels = synth_batch(seed=2, per_domain=4, size=224)
    x, labels = x.to(dev), labels.to(dev)
    cl = fmt == "nhwc"
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    # stem = "s2d": the 7x7 / 2 stem convolution evaluated as a 4x4 / 1 convolution of the space-to-depth image (harness option)
    model = build_resnet50_dwt(sd, dwt_b200, site_mode=site_mode, channels_last=cl, stem_s2d=stem == "s2d").to(dev).train()
    logits = model(x)
    s, tt, a = torch.split(logits, logits.shape[0] // 3, dim=0)
    cls = Fn.nll_loss(Fn.log_softmax(s, dim=1), labels)
    mec = 0.1 * dwt_b200.MinEntropyConsensusLoss(65, dev)(tt, a)
    (cls + mec).backward()
    # yardstick: the same topology on stock ATen ops on this GPU (fp32 convolutions, cuDNN instead of the golden's
    # MKLDNN): how far apart two correct fp32 implementations of the reference are on this input
    ref = build_resnet50_dwt({k: v.clone() for k, v in synth_state_dict(seed=1).items()}, port, site_mode="modules").to(dev).train()
    rl = ref(x.contiguous())
    rs, rt, ra = torch.split(rl, rl.shape[0] // 3, dim=0)
    (Fn.nll_loss(Fn.log_softmax(rs, dim=1), labels) + 0.1 * port.MinEntropyConsensusLoss(65, dev)(rt, ra)).backward()
    e = dict(logits=both(n(logits), z["logits"]), yard_logits=both(n(rl), z["logits"]))
    params, rparams = dict(model.named_parameters()), dict(ref.named_parameters())
    for k in [k[5:] for k in z.files if k.startswith("grad/")]:
        e["grad/" + k] = both(n(params[k].grad), z["grad/" + k])
        e["yard/" + k] = both(n(rparams[k].grad), z["grad/" + k])
    gn = np.array([params[k].grad.norm().item() for k in z["gradnames"]])
    e["gradnorms"] = both(gn, z["gradnorms"])
    bufs = model.state_dict()
    for k in [k[4:] for k in z.files if k.startswith("buf/")]:
        e["buf/" + k] = both(n(bufs[k]), z["buf/" + k])
    model.eval()
    with torch.no_grad():
        e["logits_eval"] = both(n(model(x)), z["logits_eval"])
    print(fmt, site_mode, stem, {k: ("%.2e" % v[0], "%.2e" % v[1]) for k, v in e.items()})
    assert e["logits"][0] < 2e-4 and e["logits"][1] < 5e-4, e["logits"]
    assert abs(cls.item() - float(z["cls_loss"])) < 2e-3 and abs(mec.item() - float(z["mec_loss"])) < 2e-3
    for k in [k for k in e if k.startswith("grad/")]:
        yard = e["yard/" + k[5:]][0]
        assert e[k][0] < max(1e-2, 1.5 * yard), (k, e[k], yard)       # measured: 2e-2 for both (cuDNN vs MKLDNN golden)
    for k in [k for k in e if k.startswith("buf/")]:
        assert e[k][0] < 1e-3, (k, e[k])
    assert e["logits_eval"][0] < 5e-4, e["logits_eval"]
    assert e["gradnorms"][0] < 5e-3, e["gradnorms"]                           # measured 5e-4 .. 7e-4


# --------------------------------------------------------------------------- residual tail: byte map vs out > 0
def test_residual_mask_matches_output_sign(dev):
    """Channels-last residual tail: backward through the saved (out > 0) byte map == backward of the ATen composition
    relu(site(x) + identity), for dx, d(identity), dgamma, dbeta -- and nothing of the forward output is saved."""
    import dwt_b200
    torch.manual_seed(3)
    c, hw, nper = 64, 14, 6
    x = (torch.randn(3 * nper, c, hw, hw, device=dev) * 2 + 0.5).contiguous(memory_format=torch.channels_last)
    idt = torch.randn_like(x).contiguous(memory_format=torch.channels_last)
    dout = torch.randn_like(x)
    gamma0, beta0 = 0.5 + torch.rand(c, 1, 1, device=dev), 0.1 * torch.randn(c, 1, 1, device=dev)
    out = {}
    for mode in ("fused_tail", "separate"):
        mods = [dwt_b200.WTransform2d(c, 4).to(dev).train() for _ in range(3)]
        site = dwt_b200.DomainTripleNorm("whiten", c, 4)
        g, b = gamma0.clone().requires_grad_(True), beta0.clone().requires_grad_(True)
        xi, ii = x.clone().requires_grad_(True), idt.clone().requires_grad_(True)
        if mode == "fused_tail":
            o = site(xi, mods, g, b, relu=True, residual=ii)
            assert all(s_.data_ptr() != o.data_ptr() for s_ in o.grad_fn.saved_tensors if torch.is_tensor(s_))
        else:
            o = torch.relu(site(xi, mods, g, b, relu=False) + ii)
        o.backward(dout)
        out[mode] = (o.detach(), xi.grad, ii.grad, g.grad, b.grad)
    for a, r, name in zip(out["fused_tail"], out["separate"], ("out", "dx", "d_identity", "dgamma", "dbeta")):
        assert rel_err(n(a), n(r)) < 1e-5, name
    assert torch.equal(out["fused_tail"][2] != 0, (out["fused_tail"][0] > 0) & (dout != 0))


# --------------------------------------------------------------------------- failure surfacing
def test_raise_on_status_reports_non_pd(dev):
    """The reference raises from torch.cholesky (utils/whitening.py:53).  With raise_on_status(k) the drop-in raises a
    LinAlgError subclass at the next poll, and the poisoned group's EMA never reaches the shared buffers."""
    import dwt_b200
    import whitening
    from dwt_b200 import _native
    _native.clear_status(dev)
    x = torch.randn(4, 8, 5, 5, device=dev)
    x[0, 0, 0, 0] = float("nan")
    m = whitening.WTransform2d(8, 4).to(dev).train()
    rv0 = m.running_variance.clone()
    dwt_b200.raise_on_status(every=1)
    try:
        with pytest.raises(torch.linalg.LinAlgError, match="not positive definite"):
            m(x)
        assert _native.status(dev) == 0                                      # the check cleared the word
        assert torch.equal(m.running_variance[0], rv0[0])                    # poisoned group: EMA skipped
        assert not torch.equal(m.running_variance[1], rv0[1]) and torch.isfinite(m.running_variance).all()
        m(torch.randn(4, 8, 5, 5, device=dev))                               # healthy input: no raise
    finally:
        dwt_b200.raise_on_status(every=0)


@pytest.mark.parametrize("gs", [4, 8, 64])
def test_non_pd_skips_ema_every_family(gs, dev):
    """small / tiled / tensor-core finalize: a NaN covariance sets the status bit and leaves that group's buffers alone."""
    import whitening
    from dwt_b200 import _native
    _native.clear_status(dev)
    c, hw, nimg = 2 * gs, 16, 20 if gs >= 8 else 4
    x = torch.randn(nimg, c, hw, hw, device=dev)
    x[0, 0, 0, 0] = float("nan")
    m = whitening.WTransform2d(c, gs).to(dev).train()
    rv0, rm0 = m.running_variance.clone(), m.running_mean.clone()
    with torch.no_grad():
        m(x)
    assert _native.status(dev) & _native.STATUS_NOT_PD
    assert torch.equal(m.running_variance[0], rv0[0]) and torch.equal(m.running_mean.reshape(-1)[:gs], rm0.reshape(-1)[:gs])
    assert torch.isfinite(m.running_variance[1]).all() and not torch.equal(m.running_variance[1], rv0[1])
    _native.clear_status(dev)


def test_head_loss_label_semantics(dev):
    """F.nll_loss semantics of the fused head loss: ignore_index=-100 rows leave sum and denominator; any other
    out-of-range label is never dereferenced, sets STATUS_BAD_LABEL and is dropped."""
    import torch.nn.functional as Fn
    import dwt_b200
    from dwt_b200 import _native
    _native.clear_status(dev)
    torch.manual_seed(0)
    B, K = 8, 65
    logits = torch.randn(3 * B, K, device=dev, requires_grad=True)
    labels = torch.randint(0, K, (B,), device=dev)
    labels[2] = -100
    head = dwt_b200.HeadLoss(K, 0.1)
    loss = head(logits, labels)
    loss.backward()
    ref_logits = logits.detach().clone().requires_grad_(True)
    s, tt, a = torch.split(ref_logits, B, dim=0)
    ref = Fn.nll_loss(Fn.log_softmax(s, dim=1), labels) + 0.1 * dwt_b200.MinEntropyConsensusLoss(K, dev)(tt, a)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5 and rel_err(n(logits.grad), n(ref_logits.grad)) < 1e-5
    assert _native.status(dev) == 0
    bad = labels.clone()
    bad[0], bad[5] = K + 7, -3                                                # F.nll_loss would device-assert
    loss_bad = head(logits.detach(), bad)
    keep = torch.ones(B, dtype=torch.bool, device=dev)
    keep[[0, 2, 5]] = False
    want = Fn.nll_loss(Fn.log_softmax(logits.detach()[:B][keep], dim=1), labels[keep])
    assert abs(head.parts[1].item() - want.item()) < 1e-5 and torch.isfinite(loss_bad)
    assert _native.status(dev) & _native.STATUS_BAD_LABEL
    with pytest.raises(IndexError, match="label"):
        _native.check_status(dev)
    assert _native.status(dev) == 0


def test_pointer_arguments_are_validated(dev):
    """A strided or mis-sized buffer would be read / written out of bounds through the raw-pointer ABI: refuse it."""
    import batch_norm
    import whitening
    x = torch.randn(4, 8, 6, 6, device=dev)
    wide = torch.zeros(1, 16, 1, 1, device=dev)
    m = whitening.WTransform2d(8, 4, running_m=wide[:, ::2], running_var=torch.ones(2, 4, 4, device=dev)).train()
    with pytest.raises(ValueError, match="contiguous"):
        m(x)
    m = whitening.WTransform2d(8, 4, running_m=torch.zeros(1, 8, 1, 1, device=dev), running_var=torch.ones(2, 4, 2, device=dev)).train()
    with pytest.raises(ValueError, match="elements"):
        m(x)
    bn = batch_norm.BatchNorm2d(8, torch.zeros(4, device=dev), torch.ones(8, device=dev), affine=False).train()
    with pytest.raises(ValueError, match="elements"):
        bn(x)
    v0 = torch.zeros(8, device=dev)
    bn = batch_norm.BatchNorm2d(8, v0, torch.ones(8, device=dev), affine=False).train()
    ver = v0._version
    bn(x)
    assert v0._version > ver                                                  # the in-place EMA is visible to autograd


# --------------------------------------------------------------------------- fork_for_sum: gradient sum inside the kernels
@pytest.mark.parametrize("fmt", ["nhwc", "nchw"])
def test_fork_for_sum_equals_autograd_add(fmt, dev):
    """A fused residual-tail site whose output feeds two consumers: with fork_for_sum the two gradients reach the
    site's backward as dout and dout2 and are summed where they are read (channels-last kernels; the NCHW path adds them
    with one ATen op inside backward).  fp32 addition of the same two numbers either way: bit-identical gradients."""
    import dwt_b200
    import whitening
    torch.manual_seed(11)
    c, gs, nper, hw = 64, 4, 4, 12
    cl = fmt == "nhwc"

    def tensor(*shape):
        v = torch.randn(*shape, device=dev)
        return v.contiguous(memory_format=torch.channels_last) if cl else v
    x0, res0, w1, w2 = tensor(3 * nper, c, hw, hw), tensor(3 * nper, c, hw, hw), tensor(3 * nper, c, hw, hw), tensor(3 * nper, c, hw, hw)
    g0, b0 = torch.rand(c, 1, 1, device=dev) + 0.5, 0.1 * torch.randn(c, 1, 1, device=dev)

    def run(use_fork):
        mods = [whitening.WTransform2d(c, gs).to(dev).train() for _ in range(3)]
        site = dwt_b200.DomainTripleNorm("whiten", c, gs)
        x, res = x0.clone().requires_grad_(True), res0.clone().requires_grad_(True)
        gamma, beta = g0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
        y = site(x, mods, gamma, beta, True, residual=res)
        a, b = dwt_b200.fork_for_sum(y) if use_fork else (y, y)
        if use_fork:
            assert a is not y and a.data_ptr() == y.data_ptr()
        ((a * w1).sum() + (b * b * w2).sum()).backward()
        return x.grad, res.grad, gamma.grad, beta.grad
    ref, got = run(False), run(True)
    for name, r, g in zip(("dx", "dres", "dgamma", "dbeta"), ref, got):
        assert torch.equal(r, g), (name, (r - g).abs().max().item())
    # not the output of a site of this package: plain aliases, autograd adds as usual
    t = torch.randn(4, device=dev, requires_grad=True) * 2
    a, b = dwt_b200.fork_for_sum(t)
    assert a is t and b is t
    with torch.no_grad():
        y = dwt_b200.DomainTripleNorm("whiten", c, gs)(x0, [whitening.WTransform2d(c, gs).to(dev).train() for _ in range(3)], g0, b0, True, residual=res0)
        a, b = dwt_b200.fork_for_sum(y)
        assert a is y and b is y


def test_resnet_block_gradients_with_and_without_fork(dev):
    """Whole harness model (fused sites, channels-last): every parameter gradient with the in-kernel gradient sum equals
    the one with autograd's add."""
    import dwt_b200
    from harness.resnet50_dwt import Bottleneck, build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    x, labels = synth_batch(seed=5, per_domain=2, size=64)
    x = x.to(dev).contiguous(memory_format=torch.channels_last)

    def grads(fork):
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        model = build_resnet50_dwt(sd, dwt_b200, site_mode="fused", channels_last=True).to(dev).train()
        if not fork:
            for m in model.modules():
                if isinstance(m, Bottleneck):
                    object.__setattr__(m, "_fork", None)
        model(x).square().mean().backward()
        return {k: p.grad.clone() for k, p in model.named_parameters()}
    det, bm = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False     # same cuDNN algorithms in both runs
    try:
        a, b = grads(True), grads(False)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = det, bm
    worst = max(((a[k] - b[k]).abs().max().item() / (b[k].abs().max().item() + 1e-30), k) for k in a)
    print("fork vs add: worst relative difference", worst)
    assert worst[0] < 1e-6, worst          # measured: 0.0 (the same additions in another place)


# --------------------------------------------------------------------------- channels-last max-pool (stem tail)
@pytest.mark.parametrize("shape,k,s,p", [((6, 64, 112, 112), 3, 2, 1), ((3, 8, 9, 7), 3, 2, 1), ((2, 16, 8, 8), 2, 2, 0),
                                          ((2, 4, 5, 6), 3, 1, 1), ((1, 12, 7, 7), 5, 3, 2),
                                          ((2, 8, 10, 6), 3, 2, 1), ((3, 4, 2, 2), 3, 2, 1), ((2, 12, 8, 8), 3, 2, 1),
                                          ((2, 8, 8, 12), 3, 2, 1), ((1, 4, 4, 4), 3, 2, 1)])
def test_maxpool_is_bit_exact_vs_torch(shape, k, s, p, dev):
    """dwt_b200.MaxPool2d == F.max_pool2d forward AND backward, bit for bit: post-ReLU inputs are full of ties (windows
    of zeros), and the gradient must go to the same element (first maximum in row-major window order)."""
    import torch.nn.functional as Fn
    import dwt_b200
    torch.manual_seed(sum(shape) + k)
    x = torch.relu(torch.randn(*shape, device=dev)).contiguous(memory_format=torch.channels_last)   # ~50 % exact zeros
    x[0, 0, 0, 0] = float("nan")
    g = torch.randn(shape[0], shape[1], (shape[2] + 2 * p - k) // s + 1, (shape[3] + 2 * p - k) // s + 1, device=dev)
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    ya = dwt_b200.MaxPool2d(k, s, p)(xa)
    yb = Fn.max_pool2d(xb, k, s, p)
    assert ya.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(torch.nan_to_num(ya, nan=-7.0), torch.nan_to_num(yb, nan=-7.0))
    ya.backward(g); yb.backward(g)
    assert torch.equal(xa.grad, xb.grad)
    from dwt_b200 import _native
    with pytest.raises(_native.NativeError, match="channels_last"):
        dwt_b200.MaxPool2d(k, s, p)(x.contiguous())


# --------------------------------------------------------------------------- launch-shape switches (read once per process)
_SWITCH_SCRIPT = r"""
import sys, numpy as np, torch
sys.path[:0] = [{plugin!r}, {root!r}]
import dwt_b200
from oracle import dwt_oracle as O
dev = torch.device("cuda", 0)
rng = np.random.default_rng(7)
c, hw, nper, gs = 64, 12, 4, 4
x = rng.standard_normal((3 * nper, c, hw, hw)) * 1.5 + 0.3
dout = rng.standard_normal(x.shape)
gamma, beta = 0.5 + rng.random(c), 0.2 * rng.standard_normal(c)
outs, dxs = [], []
for d in range(3):
    xd, dd = x[d * nper:(d + 1) * nper], dout[d * nper:(d + 1) * nper]
    y, mean, w, *_ = O.whiten_forward(xd, gs)
    pre = O.scale_shift_relu(y, gamma, beta, False)
    dz = dd * (pre > 0)
    dxs.append(O.whiten_backward(xd, dz * gamma.reshape(1, c, 1, 1), mean, w)); outs.append(np.maximum(pre, 0))
t = lambda a: torch.tensor(a, dtype=torch.float32, device=dev)
mods = [dwt_b200.WTransform2d(c, gs).to(dev).train() for _ in range(3)]
xt = t(x).contiguous(memory_format=torch.channels_last).requires_grad_(True)
g, b = t(gamma.reshape(c, 1, 1)).requires_grad_(True), t(beta.reshape(c, 1, 1)).requires_grad_(True)
out = dwt_b200.DomainTripleNorm("whiten", c, gs)(xt, mods, g, b, relu=True)
out.backward(t(dout).contiguous(memory_format=torch.channels_last))
rel = lambda a, r: float(np.linalg.norm(a - r) / np.linalg.norm(r))
e = (rel(out.detach().double().cpu().numpy(), np.concatenate(outs)), rel(xt.grad.double().cpu().numpy(), np.concatenate(dxs)))
assert e[0] < 1e-3 and e[1] < 1e-3, e
assert dwt_b200._native.status_all(dev) == 0
print("OK", e)
"""


@pytest.mark.parametrize("env", [{"DWT_CL_SEQ_MB": "0"}, {"DWT_PDL": "1"}, {"DWT_CL_SEQ_MB": "0", "DWT_PDL": "1"}],
                         ids=["domains_in_sequence", "pdl", "both"])
def test_channels_last_launch_switches(env, dev):
    """The experiment switches of the channels-last family -- all CTAs sweeping the domains one after the other
    (grid.z = 1) and programmatic dependent launch of the finalize / elementwise kernels -- give the same results as the
    default launch shapes (fused site, forward + backward, against the fp64 oracle).  They are read once per process,
    hence the subprocess."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = _SWITCH_SCRIPT.format(plugin=os.path.join(root, "dwt-domain-adaptation_b200"), root=root)
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, **env), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
