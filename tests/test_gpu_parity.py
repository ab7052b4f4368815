"""GPU parity: the CUDA path (through the drop-in modules -> ctypes -> C ABI) against
  (1) golden outputs of the unmodified reference (tests/golden/*.npz), and
  (2) the fp64 CPU oracle (oracle/dwt_oracle.py) on seeded inputs at sizes it finishes in seconds.

Tolerance: BASELINE.json's bar is 1e-3 relative (fp32, norm-wise ||a-b||/||b||).  These tests
assert TOL = 1e-3 on activations/gradients that pass through a Cholesky factor and TOL_STAT =
1e-4 on plain statistics (means, covariances, running buffers, BN outputs).
"""
import glob
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import dwt_oracle as O

pytestmark = pytest.mark.gpu

TOL = 1e-3
TOL_STAT = 1e-4
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WHITEN = sorted(glob.glob(os.path.join(HERE, "w_*.npz")))


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


# --------------------------------------------------------------------------- whitening
@pytest.mark.parametrize("path", WHITEN, ids=[os.path.basename(p)[:-4] for p in WHITEN])
def test_whitening_vs_reference_golden(path, dev):
    import whitening                       # the drop-in shim -> dwt_b200.whitening
    assert "dwt_b200" in whitening.WTransform2d.__module__
    z = np.load(path)
    gs, c = int(z["gs"]), z["x1"].shape[1]
    m = whitening.WTransform2d(c, gs, running_m=t(z["rm0"], dev), running_var=t(z["rv0"], dev)).train()
    x = t(z["x1"], dev).requires_grad_(True)
    y = m(x)
    (dx,) = torch.autograd.grad(y, x, t(z["dy"], dev))
    assert rel_err(n(y), z["y1"]) < TOL
    assert rel_err(n(dx), z["dx1"]) < TOL
    assert rel_err(n(m.running_mean), z["rm1"]) < TOL_STAT and rel_err(n(m.running_variance), z["rv1"]) < TOL_STAT
    with torch.no_grad():                                   # stats-collection forward
        y2 = m(t(z["x2"], dev))
    assert rel_err(n(y2), z["y2"]) < TOL
    assert rel_err(n(m.running_mean), z["rm2"]) < TOL_STAT and rel_err(n(m.running_variance), z["rv2"]) < TOL_STAT
    m.eval()
    xe = t(z["x1"], dev).requires_grad_(True)
    ye = m(xe)
    (dxe,) = torch.autograd.grad(ye, xe, t(z["dy"], dev))
    assert rel_err(n(ye), z["y_eval"]) < TOL and rel_err(n(dxe), z["dx_eval"]) < TOL
    assert rel_err(n(m.running_mean), z["rm2"]) < TOL_STAT      # eval leaves the buffers alone
    d = whitening.WTransform2d(c, gs).to(dev).train()           # default buffers: zeros / all-ones
    with torch.no_grad():
        d(t(z["x1"], dev))
    assert rel_err(n(d.running_mean), z["rm_default1"]) < TOL_STAT
    assert rel_err(n(d.running_variance), z["rv_default1"]) < TOL_STAT
    from dwt_b200 import _native
    assert _native.status(dev) == 0


def _correlated(rng, nimg, c, h, w, offset=2.0):
    z = rng.standard_normal((nimg, c, h, w))
    mix = rng.standard_normal((c, c)) / np.sqrt(c) + np.eye(c)
    return np.einsum("dc,nchw->ndhw", mix, z) + offset


ORACLE_CASES = [   # N, C, H, W, gs
    (8, 64, 56, 56, 4),       # ResNet layer1 site (per-domain slice, reduced N)
    (4, 64, 112, 112, 4),     # ResNet stem site
    (6, 256, 28, 28, 4),
    (5, 32, 28, 28, 4),       # LeNet conv1 site
    (16, 48, 14, 14, 4),      # LeNet conv2 site
    (7, 24, 9, 9, 2),         # HW % 4 != 0 -> scalar path
    (6, 128, 28, 28, 64),     # microbench group size
    (12, 64, 20, 20, 32),
    (9, 48, 10, 10, 16),
    (48, 48, 10, 10, 16),     # tensor-core contraction with a partial 64-channel super-block (TMA zero fill)
    (20, 192, 16, 16, 8),     # tensor-core contraction, 8 groups per super-block
    (5, 24, 7, 7, 8),         # tiled path, HW % 4 != 0
    (6, 36, 8, 8, 12),        # group size not a power of two
]


@pytest.mark.parametrize("case", ORACLE_CASES, ids=lambda c: "n{}c{}h{}w{}g{}".format(*c))
def test_whitening_vs_oracle_fp64(case, dev):
    import whitening
    nimg, c, h, w, gs = case
    rng = np.random.default_rng(hash(case) % (2 ** 31))
    x, dy = _correlated(rng, nimg, c, h, w), rng.standard_normal((nimg, c, h, w))
    rm0 = 0.1 * rng.standard_normal(c)
    a = rng.standard_normal((c // gs, gs, gs))
    rv0 = a @ a.transpose(0, 2, 1) / gs + 0.5 * np.eye(gs)
    y_o, mean_o, w_o, rm1_o, rv1_o, cov_o = O.whiten_forward(x, gs, running_mean=rm0, running_cov=rv0)
    dx_o = O.whiten_backward(x, dy, mean_o, w_o)
    m = whitening.WTransform2d(c, gs, running_m=t(rm0.reshape(1, c, 1, 1), dev), running_var=t(rv0, dev)).train()
    xt = t(x, dev).requires_grad_(True)
    y = m(xt)
    (dx,) = torch.autograd.grad(y, xt, t(dy, dev))
    errs = dict(y=rel_err(n(y), y_o), dx=rel_err(n(dx), dx_o), rm=rel_err(n(m.running_mean).reshape(-1), rm1_o),
                rv=rel_err(n(m.running_variance), rv1_o))
    print(case, errs)
    assert errs["y"] < TOL and errs["dx"] < TOL and errs["rm"] < TOL_STAT and errs["rv"] < TOL_STAT


def test_whitening_large_mean_is_stable(dev):
    """One-pass moments with a pilot shift: |mean| = 50 sigma must not cost accuracy."""
    import whitening
    rng = np.random.default_rng(5)
    x = _correlated(rng, 6, 16, 12, 12, offset=0.0) * 0.2 + 10.0 + 40.0 * np.arange(16).reshape(1, 16, 1, 1) / 16
    y_o, *_ = O.whiten_forward(x, 4)
    m = whitening.WTransform2d(16, 4).to(dev).train()
    assert rel_err(n(m(t(x, dev))), y_o) < TOL


def test_whitening_errors(dev):
    import whitening
    with pytest.raises(ValueError, match="expected 4D input"):
        whitening.WTransform2d(8, 4).to(dev)(torch.zeros(2, 8, 3, device=dev))
    with pytest.raises(ValueError, match="divisible by group_size"):
        whitening.WTransform2d(48, 32).to(dev)(torch.zeros(2, 48, 3, 3, device=dev))
    from dwt_b200 import _native
    with pytest.raises(_native.NativeError, match="no CPU fallback"):
        whitening.WTransform2d(8, 4)(torch.zeros(2, 8, 3, 3))


# --------------------------------------------------------------------------- batch norm
@pytest.mark.parametrize("name", ["bn2d_affine", "bn2d_plain", "bn2d_hw4", "bn2d_cma", "bn1d_2", "bn1d_3", "bn3d"])
def test_bn_vs_reference_golden(name, dev):
    import batch_norm
    z = np.load(os.path.join(HERE, "bn.npz"))
    g = lambda k: z[f"{name}_{k}"]
    cls = {"bn1d": batch_norm.BatchNorm1d, "bn2d": batch_norm.BatchNorm2d, "bn3d": batch_norm.BatchNorm3d}[name[:4]]
    affine = f"{name}_weight" in z
    mom = {"bn2d_cma": None, "bn3d": 0.3}.get(name, 0.1)
    m = cls(g("x1").shape[1], t(g("rm0"), dev), t(g("rv0"), dev), affine=affine, momentum=mom).to(dev).train()
    if affine:
        with torch.no_grad():
            m.weight.copy_(t(g("weight"), dev)); m.bias.copy_(t(g("bias"), dev))
    x = t(g("x1"), dev).requires_grad_(True)
    y = m(x)
    y.backward(t(g("dy"), dev))
    assert rel_err(n(y), g("y1")) < TOL_STAT and rel_err(n(x.grad), g("dx1")) < TOL_STAT
    assert rel_err(n(m.running_mean), g("rm1")) < TOL_STAT and rel_err(n(m.running_var), g("rv1")) < TOL_STAT
    if affine:
        assert rel_err(n(m.weight.grad), g("dweight")) < TOL_STAT and rel_err(n(m.bias.grad), g("dbias")) < TOL_STAT
    with torch.no_grad():
        m(t(g("x2"), dev))
    assert rel_err(n(m.running_mean), g("rm2")) < TOL_STAT and rel_err(n(m.running_var), g("rv2")) < TOL_STAT
    assert int(m.num_batches_tracked) == int(g("nbt2"))
    m.eval()
    xe = t(g("x1"), dev).requires_grad_(True)
    ye = m(xe)
    ye.backward(t(g("dy"), dev))
    assert rel_err(n(ye), g("y_eval")) < TOL_STAT and rel_err(n(xe.grad), g("dx_eval")) < TOL_STAT


@pytest.mark.parametrize("shape", [(8, 512, 7, 7), (6, 128, 28, 28), (4, 2048, 7, 7), (5, 256, 14, 14)],
                         ids=lambda s: "x".join(map(str, s)))
def test_bn_vs_oracle_fp64(shape, dev):
    import batch_norm
    rng = np.random.default_rng(3)
    c = shape[1]
    x = rng.standard_normal(shape) * (0.5 + rng.random((1, c, 1, 1))) + rng.standard_normal((1, c, 1, 1))
    dy = rng.standard_normal(shape)
    rm0, rv0 = 0.1 * rng.standard_normal(c), 0.5 + rng.random(c)
    y_o, mean_o, inv_o, rm1_o, rv1_o = O.bn_forward(x, rm0, rv0)
    dx_o, _, _ = O.bn_backward(x, dy, mean_o, inv_o)
    m = batch_norm.BatchNorm2d(c, t(rm0, dev), t(rv0, dev), affine=False).train()
    xt = t(x, dev).requires_grad_(True)
    y = m(xt)
    y.backward(t(dy, dev))
    assert rel_err(n(y), y_o) < TOL_STAT and rel_err(n(xt.grad), dx_o) < TOL_STAT
    assert rel_err(n(m.running_mean), rm1_o) < TOL_STAT and rel_err(n(m.running_var), rv1_o) < TOL_STAT


# --------------------------------------------------------------------------- MEC
@pytest.mark.parametrize("name", ["plain", "big", "k10", "n1", "ties"])
def test_mec_vs_reference_golden(name, dev):
    import consensus_loss
    z = np.load(os.path.join(HERE, "mec.npz"))
    x, y = t(z[name + "_x"], dev).requires_grad_(True), t(z[name + "_y"], dev).requires_grad_(True)
    crit = consensus_loss.MinEntropyConsensusLoss(num_classes=x.shape[1], device=dev)
    loss = crit(x, y)
    assert loss.dim() == 0
    (0.7 * loss).backward()
    assert abs(loss.item() - float(z[name + "_loss"])) < 1e-5 * max(1.0, abs(loss.item()))
    assert rel_err(n(x.grad), 0.7 * z[name + "_gx"]) < TOL_STAT and rel_err(n(y.grad), 0.7 * z[name + "_gy"]) < TOL_STAT


def test_mec_vs_oracle_batch64(dev):
    import consensus_loss
    rng = np.random.default_rng(9)
    x, y = 3 * rng.standard_normal((64, 65)), 3 * rng.standard_normal((64, 65))
    loss_o, gx_o, gy_o, _ = O.mec_loss(x, y)
    xt, yt = t(x, dev).requires_grad_(True), t(y, dev).requires_grad_(True)
    loss = consensus_loss.MinEntropyConsensusLoss(65, dev)(xt, yt)
    loss.backward()
    assert abs(loss.item() - loss_o) < 1e-5 and rel_err(n(xt.grad), gx_o) < TOL_STAT and rel_err(n(yt.grad), gy_o) < TOL_STAT


# --------------------------------------------------------------------------- fused domain triple
@pytest.mark.parametrize("kind,c,hw,gs", [("whiten", 64, 28, 4), ("whiten", 256, 14, 4), ("bn", 128, 14, 1),
                                           ("bn", 512, 7, 1), ("whiten", 16, 9, 2),
                                           ("whiten", 64, 12, 8),       # large groups, tiled kernels (M < 4096)
                                           ("whiten", 128, 32, 64)])    # large groups, TMA + wgmma kernels, D = 3
@pytest.mark.parametrize("relu", [True, False])
def test_fused_triple_vs_oracle(kind, c, hw, gs, relu, dev):
    """DomainTripleNorm == split/3 -> 3 modules on ALIASED buffers -> cat -> *gamma+beta -> relu
    (resnet50_dwt_mec_officehome.py:220-222), incl. the sequential EMA of SURVEY.md H5."""
    import batch_norm
    import whitening
    from dwt_b200 import DomainTripleNorm
    rng = np.random.default_rng(11)
    nper = 5
    x = np.concatenate([_correlated(rng, nper, c, hw, hw, offset=o) for o in (0.5, -1.0, 2.0)])
    dout = rng.standard_normal(x.shape)
    gamma, beta = 0.5 + rng.random(c), 0.3 * rng.standard_normal(c)
    if kind == "whiten":
        rm = 0.1 * rng.standard_normal(c)
        a = rng.standard_normal((c // gs, gs, gs))
        rv = a @ a.transpose(0, 2, 1) / gs + 0.5 * np.eye(gs)
    else:
        rm, rv = 0.1 * rng.standard_normal(c), 0.5 + rng.random(c)
    rm_t = t(rm.reshape(1, c, 1, 1) if kind == "whiten" else rm, dev)
    rv_t = t(rv, dev)
    if kind == "whiten":
        mods = [whitening.WTransform2d(c, gs, running_m=rm_t, running_var=rv_t).train() for _ in range(3)]
    else:
        mods = [batch_norm.BatchNorm2d(c, rm_t, rv_t, affine=False).train() for _ in range(3)]
    site = DomainTripleNorm(kind, c, gs)
    g_t = t(gamma.reshape(c, 1, 1), dev).requires_grad_(True)
    b_t = t(beta.reshape(c, 1, 1), dev).requires_grad_(True)
    xt = t(x, dev).requires_grad_(True)
    out = site(xt, mods, g_t, b_t, relu=relu)
    out.backward(t(dout, dev))
    # oracle: three sequential domain calls on the same buffers.  The ReLU derivative is taken where the forward under
    # test put it (as autograd does for the fp32 reference): a pre-activation within fp32 rounding of zero may land on
    # either side, and such elements are the only place the two masks may disagree.
    active = n(out) > 0
    flips = 0                                      # elements whose mask differs from the fp64 forward's
    outs, dxs = [], []
    dgamma, dbeta = np.zeros(c), np.zeros(c)
    rm_o, rv_o = rm, rv
    for d in range(3):
        xd, dd = x[d * nper:(d + 1) * nper], dout[d * nper:(d + 1) * nper]
        if kind == "whiten":
            y, mean, w, rm_o, rv_o, _ = O.whiten_forward(xd, gs, running_mean=rm_o, running_cov=rv_o)
        else:
            y, mean, inv, rm_o, rv_o = O.bn_forward(xd, rm_o, rv_o)
        pre = O.scale_shift_relu(y, gamma, beta, False)
        out_o = np.maximum(pre, 0) if relu else pre
        if relu:
            mask = active[d * nper:(d + 1) * nper]
            assert np.all(np.abs(pre[mask != (pre > 0)]) < 1e-5)
            flips += int((mask != (pre > 0)).sum())
        dz = dd * mask if relu else dd
        dgamma += (dz * y).sum(axis=(0, 2, 3)); dbeta += dz.sum(axis=(0, 2, 3))
        dyd = dz * gamma.reshape(1, c, 1, 1)
        dxs.append(O.whiten_backward(xd, dyd, mean, w) if kind == "whiten" else O.bn_backward(xd, dyd, mean, inv)[0])
        outs.append(out_o)
    tol = TOL if kind == "whiten" else TOL_STAT
    assert flips <= 4, flips                       # a systematic forward error would flip many more
    assert rel_err(n(out), np.concatenate(outs)) < tol
    assert rel_err(n(xt.grad), np.concatenate(dxs)) < tol
    assert rel_err(n(g_t.grad).reshape(-1), dgamma) < tol and rel_err(n(b_t.grad).reshape(-1), dbeta) < tol
    assert rel_err(n(rm_t).reshape(-1), rm_o) < TOL_STAT and rel_err(n(rv_t), rv_o) < TOL_STAT
    if kind == "bn":
        assert all(int(m.num_batches_tracked) == 1 for m in mods)


# --------------------------------------------------------------------------- full-size properties
def test_microbench_shape_properties(dev):
    """BASELINE.json config 2 at full size (N=256,C=256,56x56,gs=64): size-independent properties
    instead of a CPU oracle.  With S = (1-eps) Sigma + eps I = L L^T and W = L^-1:
        mean(y) = 0,   (1-eps) cov(y) + eps W W^T = I,   y == fp64 recomputation on the device,
        <dy, J v> == <J^T dy, v> (J v by central differences of the layer itself), sum_m dx = 0."""
    import whitening
    torch.manual_seed(0)
    N, C, H, gs, eps = 256, 256, 56, 64, 1e-3
    mix = torch.randn(C, C, device=dev) / C ** 0.5 + torch.eye(C, device=dev)
    x = torch.einsum("dc,nchw->ndhw", mix, torch.randn(N, C, H, H, device=dev)) + 2.0
    m = whitening.WTransform2d(C, gs).to(dev).train()
    x.requires_grad_(True)
    y = m(x)
    G = C // gs
    yg = y.detach().transpose(0, 1).reshape(G, gs, -1).double()
    mean_y = yg.mean(-1)
    cov_y = yg @ yg.transpose(1, 2) / yg.shape[-1]
    assert mean_y.abs().max() < 1e-4
    xg = x.detach().transpose(0, 1).reshape(G, gs, -1).double()
    xc = xg - xg.mean(-1, keepdim=True)
    sigma = xc @ xc.transpose(1, 2) / xc.shape[-1]
    S = (1 - eps) * sigma + eps * torch.eye(gs, device=dev, dtype=torch.float64)
    W_ref = torch.linalg.inv(torch.linalg.cholesky(S))
    y_ref = (W_ref @ xc).reshape(C, N, H, H).transpose(0, 1)
    assert ((y.detach().double() - y_ref).norm() / y_ref.norm()).item() < TOL
    del y_ref, xc, xg, yg
    ident = (1 - eps) * cov_y + eps * (W_ref @ W_ref.transpose(1, 2))
    assert (ident - torch.eye(gs, device=dev, dtype=torch.float64)).abs().max() < 1e-3
    dy = torch.randn_like(y)
    (dx,) = torch.autograd.grad(y, x, dy)
    # adjoint test: directional derivative by central differences of the layer itself vs <dx, v>
    v = torch.randn_like(x)
    h = 1e-2
    with torch.no_grad():
        jv = (m(x + h * v) - m(x - h * v)) / (2 * h)
    lhs, rhs = (dy.double() * jv.double()).sum().item(), (dx.double() * v.double()).sum().item()
    assert abs(lhs - rhs) < 2e-3 * max(abs(lhs), abs(rhs), 1.0)
    assert dx.sum(dim=(0, 2, 3)).abs().max() < 1e-2 * dx.abs().sum(dim=(0, 2, 3)).max()   # gradient of a centred map


def test_resnet_site_fullsize_idempotence(dev):
    """ResNet stem site at the benchmark size (64 images/domain, 64x112x112, gs=4): whitening an
    already whitened batch is (up to the eps shrink) the identity -- W' ~ I / sqrt((1-eps)/(1-eps) ...)."""
    import whitening
    torch.manual_seed(1)
    x = torch.randn(64, 64, 112, 112, device=dev) * 3 + 1
    m = whitening.WTransform2d(64, 4).to(dev).train()
    with torch.no_grad():
        y = m(x)
        y2 = m(y)
    # cov(y) = (I - eps W W^T)/(1-eps); second pass sees S2 = I - eps W W^T + eps I, whose Cholesky inverse is
    # within O(eps * ||W W^T - I||) of I.  For this well-conditioned input (var 9): W W^T ~ I/9.
    assert ((y2 - y).double().norm() / y.double().norm()).item() < 2e-3
    assert y.mean(dim=(0, 2, 3)).abs().max() < 1e-4


# --------------------------------------------------------------------------- full model
@pytest.mark.parametrize("site_mode", ["modules", "fused"])
def test_resnet_tiny_vs_reference_golden(site_mode, dev):
    """The harness model with the CUDA layers vs the unmodified reference ResNet (CPU, fp32) on the
    same synthetic checkpoint and batch: logits, losses, selected gradients, buffers."""
    import torch.nn.functional as Fn
    import dwt_b200
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    z = np.load(os.path.join(HERE, "resnet_tiny.npz"))
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
    x, labels = synth_batch(seed=2, per_domain=4, size=96)
    model = build_resnet50_dwt(sd, dwt_b200, site_mode=site_mode).to(dev).train()
    logits = model(x.to(dev))
    s, tt, a = torch.split(logits, logits.shape[0] // 3, dim=0)
    cls = Fn.nll_loss(Fn.log_softmax(s, dim=1), labels.to(dev))
    mec = 0.1 * dwt_b200.MinEntropyConsensusLoss(65, dev)(tt, a)
    (cls + mec).backward()
    assert rel_err(n(logits), z["logits"]) < 5e-3          # 53 norm sites deep; per-layer bar is 1e-3
    assert abs(cls.item() - float(z["cls_loss"])) < 5e-3 and abs(mec.item() - float(z["mec_loss"])) < 5e-3
    params = dict(model.named_parameters())
    # Deep-gradient yardstick: the same model built from stock ATen ops (the CPU port of the reference
    # layers, run on this GPU) differs from the CPU fp32 golden by cuDNN-vs-MKLDNN rounding amplified
    # through 53 batch-statistics layers.  Our layers may not be worse than 2x that (floor 2e-2).
    import oracle.torch_port as port
    ref = build_resnet50_dwt({k: v.clone() for k, v in synth_state_dict(seed=1).items()}, port, site_mode="modules").to(dev).train()
    rl = ref(x.to(dev))
    rs, rt, ra = torch.split(rl, rl.shape[0] // 3, dim=0)
    (Fn.nll_loss(Fn.log_softmax(rs, dim=1), labels.to(dev)) + 0.1 * port.MinEntropyConsensusLoss(65, dev)(rt, ra)).backward()
    rparams = dict(ref.named_parameters())
    for k in [k[5:] for k in z.files if k.startswith("grad/")]:
        yard = rel_err(n(rparams[k].grad), z["grad/" + k])
        assert rel_err(n(params[k].grad), z["grad/" + k]) < max(2e-2, 2 * yard), (k, yard)
    bufs = model.state_dict()
    for k in [k[4:] for k in z.files if k.startswith("buf/")]:
        assert rel_err(n(bufs[k]), z["buf/" + k]) < 1e-3, k
    model.eval()
    with torch.no_grad():
        assert rel_err(n(model(x.to(dev))), z["logits_eval"]) < 5e-3


@pytest.mark.parametrize("layout", ["distinct", "mixed"])
def test_fused_triple_buffer_aliasing_classes(layout, dev):
    """The fused site must give each domain's running buffers exactly what three sequential module
    calls give them, whether the three modules share one buffer (tested above), own three buffers,
    or two of them share (source alone, target+aug shared)."""
    import whitening
    from dwt_b200 import DomainTripleNorm
    rng = np.random.default_rng(21)
    c, gs, nper, hw = 32, 4, 4, 12
    x = np.concatenate([_correlated(rng, nper, c, hw, hw, offset=o) for o in (0.5, -1.0, 2.0)])
    rm0 = 0.1 * rng.standard_normal(c)
    a = rng.standard_normal((c // gs, gs, gs))
    rv0 = a @ a.transpose(0, 2, 1) / gs + 0.5 * np.eye(gs)
    owner = {"distinct": [0, 1, 2], "mixed": [0, 1, 1]}[layout]
    bufs = {o: [rm0.copy(), rv0.copy()] for o in set(owner)}
    for d in range(3):                                     # oracle: sequential calls
        _, _, _, nrm, nrv, _ = O.whiten_forward(x[d * nper:(d + 1) * nper], gs, running_mean=bufs[owner[d]][0],
                                                running_cov=bufs[owner[d]][1])
        bufs[owner[d]] = [nrm, nrv]
    tb = {o: (t(rm0.reshape(1, c, 1, 1), dev), t(rv0, dev)) for o in set(owner)}
    mods = [whitening.WTransform2d(c, gs, running_m=tb[o][0], running_var=tb[o][1]).train() for o in owner]
    g_t, b_t = torch.ones(c, 1, 1, device=dev), torch.zeros(c, 1, 1, device=dev)
    with torch.no_grad():
        DomainTripleNorm("whiten", c, gs)(t(x, dev), mods, g_t, b_t, relu=False)
    for o in set(owner):
        assert rel_err(n(tb[o][0]).reshape(-1), bufs[o][0]) < TOL_STAT and rel_err(n(tb[o][1]), bufs[o][1]) < TOL_STAT


# --------------------------------------------------------------------------- channels-last (NHWC) kernels
@pytest.mark.parametrize("kind,c,hw,gs", [("whiten", 64, 28, 4), ("whiten", 256, 14, 4), ("whiten", 16, 10, 4),
                                           ("whiten", 32, 9, 2), ("bn", 128, 14, 1), ("bn", 2048, 7, 1), ("bn", 8, 5, 1),
                                           # launch edges: C = 4, 8 (every float4 column shared by 256 / 128 threads),
                                           # C = 1024 / 2048 / 4096 (one thread per column, grid.y = 1 / 2 / 4)
                                           ("whiten", 4, 3, 4), ("whiten", 8, 4, 2), ("whiten", 1024, 3, 4),
                                           ("whiten", 2048, 2, 2), ("bn", 4096, 2, 1)])
@pytest.mark.parametrize("relu", [True, False])
def test_channels_last_site_matches_oracle(kind, c, hw, gs, relu, dev):
    """The NHWC kernels (torch.channels_last tensors) against the same oracle as the NCHW ones: fused domain
    triple on aliased buffers, forward, backward, dgamma/dbeta, EMA."""
    import batch_norm
    import whitening
    from dwt_b200 import DomainTripleNorm
    rng = np.random.default_rng(31)
    nper = 6
    x = np.concatenate([_correlated(rng, nper, c, hw, hw, offset=o) for o in (0.5, -1.0, 2.0)])
    dout = rng.standard_normal(x.shape)
    gamma, beta = 0.5 + rng.random(c), 0.3 * rng.standard_normal(c)
    if kind == "whiten":
        rm = 0.1 * rng.standard_normal(c)
        a = rng.standard_normal((c // gs, gs, gs))
        rv = a @ a.transpose(0, 2, 1) / gs + 0.5 * np.eye(gs)
    else:
        rm, rv = 0.1 * rng.standard_normal(c), 0.5 + rng.random(c)
    outs, dxs = [], []
    dgamma, dbeta = np.zeros(c), np.zeros(c)
    rm_o, rv_o = rm, rv
    for d in range(3):
        xd, dd = x[d * nper:(d + 1) * nper], dout[d * nper:(d + 1) * nper]
        if kind == "whiten":
            y, mean, w, rm_o, rv_o, _ = O.whiten_forward(xd, gs, running_mean=rm_o, running_cov=rv_o)
        else:
            y, mean, inv, rm_o, rv_o = O.bn_forward(xd, rm_o, rv_o)
        pre = O.scale_shift_relu(y, gamma, beta, False)
        dz = dd * (pre > 0) if relu else dd
        dgamma += (dz * y).sum(axis=(0, 2, 3)); dbeta += dz.sum(axis=(0, 2, 3))
        dyd = dz * gamma.reshape(1, c, 1, 1)
        dxs.append(O.whiten_backward(xd, dyd, mean, w) if kind == "whiten" else O.bn_backward(xd, dyd, mean, inv)[0])
        outs.append(np.maximum(pre, 0) if relu else pre)
    rm_t = t(rm.reshape(1, c, 1, 1) if kind == "whiten" else rm, dev)
    rv_t = t(rv, dev)
    if kind == "whiten":
        mods = [whitening.WTransform2d(c, gs, running_m=rm_t, running_var=rv_t).train() for _ in range(3)]
    else:
        mods = [batch_norm.BatchNorm2d(c, rm_t, rv_t, affine=False).train() for _ in range(3)]
    g_t = t(gamma.reshape(c, 1, 1), dev).requires_grad_(True)
    b_t = t(beta.reshape(c, 1, 1), dev).requires_grad_(True)
    xt = t(x, dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    out = DomainTripleNorm(kind, c, gs)(xt, mods, g_t, b_t, relu=relu)
    assert out.is_contiguous(memory_format=torch.channels_last)
    out.backward(t(dout, dev).contiguous(memory_format=torch.channels_last))
    assert xt.grad.is_contiguous(memory_format=torch.channels_last)
    tol = TOL if kind == "whiten" else TOL_STAT
    assert rel_err(n(out), np.concatenate(outs)) < tol and rel_err(n(xt.grad), np.concatenate(dxs)) < tol
    assert rel_err(n(g_t.grad).reshape(-1), dgamma) < tol and rel_err(n(b_t.grad).reshape(-1), dbeta) < tol
    assert rel_err(n(rm_t).reshape(-1), rm_o) < TOL_STAT and rel_err(n(rv_t), rv_o) < TOL_STAT


def test_channels_last_module_paths(dev):
    """Single-domain modules on channels-last input: train, no-grad train, eval (+ backward), and channel counts
    without a channels-last build (C/4 not a power of two, C/4 > 16384) silently take the NCHW kernels."""
    import whitening
    rng = np.random.default_rng(41)
    for (nimg, c, h, w), gs in [((5, 64, 12, 12), 4), ((5, 48, 12, 12), 4), ((3, 131072, 2, 2), 4)]:
        x = _correlated(rng, nimg, c, h, w) if c <= 64 else rng.standard_normal((nimg, c, h, w)) + 2.0
        dy = rng.standard_normal(x.shape)
        y_o, mean_o, w_o, rm1, rv1, _ = O.whiten_forward(x, gs, running_mean=np.zeros(c), running_cov=np.ones((c // gs, gs, gs)))
        m = whitening.WTransform2d(c, gs).to(dev).train()
        xt = t(x, dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        y = m(xt)
        (dx,) = torch.autograd.grad(y, xt, t(dy, dev))
        assert rel_err(n(y), y_o) < TOL and rel_err(n(dx), O.whiten_backward(x, dy, mean_o, w_o)) < TOL
        assert rel_err(n(m.running_variance), rv1) < TOL_STAT
        m.eval()
        ye, _, we, *_ = O.whiten_forward(x, gs, running_mean=rm1, running_cov=rv1, training=False)
        xe = t(x, dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        yy = m(xe)
        (dxe,) = torch.autograd.grad(yy, xe, t(dy, dev))
        assert rel_err(n(yy), ye) < TOL and rel_err(n(dxe), O.whiten_backward_eval(dy, we)) < TOL


def test_resnet_tiny_channels_last_vs_reference_golden(dev):
    import torch.nn.functional as Fn
    import dwt_b200
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    z = np.load(os.path.join(HERE, "resnet_tiny.npz"))
    sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
    x, labels = synth_batch(seed=2, per_domain=4, size=96)
    model = build_resnet50_dwt(sd, dwt_b200, site_mode="fused", channels_last=True).to(dev).train()
    logits = model(x.to(dev).contiguous(memory_format=torch.channels_last))
    s, tt, a = torch.split(logits, logits.shape[0] // 3, dim=0)
    cls = Fn.nll_loss(Fn.log_softmax(s, dim=1), labels.to(dev))
    mec = 0.1 * dwt_b200.MinEntropyConsensusLoss(65, dev)(tt, a)
    (cls + mec).backward()
    assert rel_err(n(logits), z["logits"]) < 5e-3
    assert abs(cls.item() - float(z["cls_loss"])) < 5e-3 and abs(mec.item() - float(z["mec_loss"])) < 5e-3
    bufs = model.state_dict()
    for k in [k[4:] for k in z.files if k.startswith("buf/")]:
        assert rel_err(n(bufs[k]), z["buf/" + k]) < 1e-3, k


@pytest.mark.parametrize("fmt", ["nchw", "nhwc"])
@pytest.mark.parametrize("kind,c,hw,gs", [("whiten", 64, 14, 4), ("bn", 256, 7, 1)])
def test_fused_residual_tail_equals_unfused(kind, c, hw, gs, fmt, dev):
    """out = relu(site(x)*gamma + beta + identity) folded into the apply pass (Bottleneck tail,
    resnet50_dwt_mec_officehome.py:239-240) vs the same site followed by ATen add + relu: outputs and every
    gradient (x, identity, gamma, beta) must agree to rounding."""
    import batch_norm
    import whitening
    from dwt_b200 import DomainTripleNorm
    torch.manual_seed(3)
    nper = 4
    mk = (lambda a: a.contiguous(memory_format=torch.channels_last)) if fmt == "nhwc" else (lambda a: a.contiguous())
    x0 = mk(torch.randn(3 * nper, c, hw, hw, device=dev) * 1.5 + 0.3)
    r0 = mk(torch.randn(3 * nper, c, hw, hw, device=dev))
    dout = mk(torch.randn(3 * nper, c, hw, hw, device=dev))
    g0, b0 = torch.rand(c, 1, 1, device=dev) + 0.5, 0.2 * torch.randn(c, 1, 1, device=dev)
    res = {}
    for mode in ("fused", "unfused"):
        if kind == "whiten":
            mods = [whitening.WTransform2d(c, gs).to(dev).train() for _ in range(3)]
        else:
            rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
            mods = [batch_norm.BatchNorm2d(c, rm, rv, affine=False).train() for _ in range(3)]
        site = DomainTripleNorm(kind, c, gs)
        x, r = x0.clone().requires_grad_(True), r0.clone().requires_grad_(True)
        g, b = g0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
        if mode == "fused":
            out = site(x, mods, g, b, relu=True, residual=r)
        else:
            out = torch.relu(site(x, mods, g, b, relu=False) + r)
        out.backward(dout)
        res[mode] = [out.detach(), x.grad, r.grad, g.grad, b.grad]
    for a, bb in zip(res["fused"], res["unfused"]):
        assert rel_err(n(a), n(bb)) < 1e-5


def test_head_loss_matches_reference_composition(dev):
    """HeadLoss == nll_loss(log_softmax(source), y) + 0.1 * MinEntropyConsensusLoss(target, target_aug), value
    and gradient of every logit row (oracle in fp64)."""
    import dwt_b200
    rng = np.random.default_rng(77)
    B, K, lam = 64, 65, 0.1
    z = 2.5 * rng.standard_normal((3 * B, K))
    y = rng.integers(0, K, B)
    zs = z[:B] - z[:B].max(1, keepdims=True)
    lsm = zs - np.log(np.exp(zs).sum(1, keepdims=True))
    cls = -lsm[np.arange(B), y].mean()
    g_src = np.exp(lsm); g_src[np.arange(B), y] -= 1.0; g_src /= B
    mec, gx, gy, _ = O.mec_loss(z[B:2 * B], z[2 * B:])
    zt = t(z, dev).requires_grad_(True)
    head = dwt_b200.HeadLoss(K, lam)
    total = head(zt, torch.tensor(y, device=dev))
    (1.7 * total).backward()
    assert abs(total.item() - (cls + lam * mec)) < 1e-5 and abs(head.parts[1].item() - cls) < 1e-5
    assert abs(head.parts[2].item() - lam * mec) < 1e-6
    assert rel_err(n(zt.grad), 1.7 * np.concatenate([g_src, lam * gx, lam * gy])) < TOL_STAT


# --------------------------------------------------------------------------- edge cases
def test_edge_shapes_and_inputs(dev):
    """Single image per domain, a strided (non-dense) input view, a batch that does not split into the
    domains, a half-precision tensor, an empty batch."""
    import whitening
    from dwt_b200 import DomainTripleNorm, _native
    rng = np.random.default_rng(8)
    # one image: statistics over H*W only
    x = _correlated(rng, 1, 8, 9, 9)
    y_o, *_ = O.whiten_forward(x, 4)
    m = whitening.WTransform2d(8, 4).to(dev).train()
    assert rel_err(n(m(t(x, dev))), y_o) < TOL
    # a non-dense view (every second image of a larger batch): made dense internally, values unchanged
    big = t(_correlated(rng, 8, 8, 6, 6), dev)
    view = big[::2]
    assert not view.is_contiguous()
    y_o, *_ = O.whiten_forward(n(view), 4)
    assert rel_err(n(whitening.WTransform2d(8, 4).to(dev).train()(view)), y_o) < TOL
    # domain split must be exact
    site = DomainTripleNorm("whiten", 8, 4)
    mods = [whitening.WTransform2d(8, 4).to(dev).train() for _ in range(3)]
    g, b = torch.ones(8, 1, 1, device=dev), torch.zeros(8, 1, 1, device=dev)
    with pytest.raises(ValueError, match="does not split"):
        site(torch.zeros(4, 8, 3, 3, device=dev), mods, g, b)
    with pytest.raises(_native.NativeError, match="float32"):
        whitening.WTransform2d(8, 4).to(dev)(torch.zeros(2, 8, 3, 3, device=dev, dtype=torch.float16))
    with pytest.raises(_native.NativeError, match="empty tensor"):
        whitening.WTransform2d(8, 4).to(dev)(torch.zeros(0, 8, 3, 3, device=dev))
    with pytest.raises(_native.NativeError, match="group_size"):
        whitening.WTransform2d(256, 128).to(dev)(torch.zeros(2, 256, 4, 4, device=dev))   # groups above 64 are not built


def test_nonpositive_definite_sets_status_instead_of_syncing(dev):
    """The reference raises from torch.cholesky (host sync).  Here a NaN input leaves NaN outputs and a device
    status bit that the caller reads when it wants to."""
    import whitening
    from dwt_b200 import _native
    x = torch.randn(4, 8, 5, 5, device=dev)
    x[0, 0, 0, 0] = float("nan")
    y = whitening.WTransform2d(8, 4).to(dev).train()(x)
    assert torch.isnan(y[:, :4]).any() and not torch.isnan(y[:, 4:]).any()     # only the poisoned group
    assert _native.status(dev) & 1
    ws = _native._workspaces[(dev.index, torch.cuda.current_stream(dev).cuda_stream)]
    ws[:4].zero_()                                                              # caller acknowledges
    assert _native.status(dev) == 0


# --------------------------------------------------------------------------- statistics-collection pass (§8f-3)
@pytest.mark.parametrize("kind,owner", [("whiten", [0, 0, 0]), ("whiten", [0, 1, 1]), ("bn", [0, 0, 0]), ("bn", [0, 1, 2])])
def test_replicated_site_equals_three_identical_domains(kind, owner, dev):
    """resnet50_dwt_mec_officehome.py:380-389 feeds cat((d, d, d)); the replicated site takes d once and must
    leave every branch's buffers where three sequential module calls on d leave them, with the same output."""
    import batch_norm
    import whitening
    from dwt_b200 import DomainTripleNorm
    rng = np.random.default_rng(31)
    c, gs, nper, hw = 32, (4 if kind == "whiten" else 1), 4, 12
    x = _correlated(rng, nper, c, hw, hw, offset=1.5)
    rm0 = 0.1 * rng.standard_normal(c)
    if kind == "whiten":
        a = rng.standard_normal((c // gs, gs, gs))
        rv0 = a @ a.transpose(0, 2, 1) / gs + 0.5 * np.eye(gs)
    else:
        rv0 = 0.5 + rng.random(c)
    bufs = {o: [rm0.copy(), rv0.copy()] for o in set(owner)}
    y_ref = None
    for d in range(3):                                     # oracle: three sequential calls on the same data
        if kind == "whiten":
            y_ref, _, _, nrm, nrv, _ = O.whiten_forward(x, gs, running_mean=bufs[owner[d]][0], running_cov=bufs[owner[d]][1])
        else:
            y_ref, _, _, nrm, nrv = O.bn_forward(x, running_mean=bufs[owner[d]][0], running_var=bufs[owner[d]][1])
        bufs[owner[d]] = [nrm, nrv]
    if kind == "whiten":
        tb = {o: (t(rm0.reshape(1, c, 1, 1), dev), t(rv0, dev)) for o in set(owner)}
        mods = [whitening.WTransform2d(c, gs, running_m=tb[o][0], running_var=tb[o][1]).train() for o in owner]
    else:
        tb = {o: (t(rm0, dev), t(rv0, dev)) for o in set(owner)}
        mods = [batch_norm.BatchNorm2d(c, tb[o][0], tb[o][1], affine=False).train() for o in owner]
    g_t, b_t = torch.ones(c, 1, 1, device=dev), torch.zeros(c, 1, 1, device=dev)
    for fmt in (torch.contiguous_format, torch.channels_last):
        for o in tb:
            tb[o][0].copy_(t(rm0, dev).view_as(tb[o][0])); tb[o][1].copy_(t(rv0, dev))
        with torch.no_grad():
            y = DomainTripleNorm(kind, c, gs)(t(x, dev).contiguous(memory_format=fmt), mods, g_t, b_t, relu=False,
                                              replicated=True)
        assert y.shape[0] == nper and rel_err(n(y), y_ref) < TOL
        for o in set(owner):
            assert rel_err(n(tb[o][0]).reshape(-1), bufs[o][0].reshape(-1)) < TOL_STAT
            assert rel_err(n(tb[o][1]), bufs[o][1]) < TOL_STAT
    if kind == "bn":
        assert all(int(m.num_batches_tracked) == 2 for m in mods)


def test_collect_stats_replicated_matches_reference_form(dev):
    """Whole model: the single-copy pass vs the reference's cat((d,d,d)) pass, the latter run both with the
    CUDA layers and with the stock-ATen port of the reference layers."""
    import dwt_b200
    import oracle.torch_port as port
    from harness.resnet50_dwt import build_resnet50_dwt, collect_stats
    from harness.synth import synth_batch, synth_state_dict
    x, _ = synth_batch(seed=5, per_domain=4, size=96)
    batches = [x[:4].to(dev), x[4:8].to(dev)]

    def fresh(layers, mode, cl=False):
        sd = {k: v.to(dev) for k, v in synth_state_dict(seed=1).items()}
        return build_resnet50_dwt(sd, layers, site_mode=mode, channels_last=cl).to(dev).eval()

    stock = fresh(port, "modules")
    out_stock = collect_stats(stock, batches, passes=2, replicated=False)
    triple = fresh(dwt_b200, "fused")
    out_triple = collect_stats(triple, batches, passes=2, replicated=False)
    single = fresh(dwt_b200, "fused", cl=True)
    out_single = collect_stats(single, [b.contiguous(memory_format=torch.channels_last) for b in batches], passes=2)
    assert out_single.shape[0] == 4 and out_triple.shape[0] == 12
    assert rel_err(n(out_single), n(out_triple[:4])) < 1e-3 and rel_err(n(out_single), n(out_stock[4:8])) < 5e-3
    b_stock, b_triple, b_single = stock.state_dict(), triple.state_dict(), single.state_dict()
    for k, v in b_single.items():
        if "running" in k:
            assert rel_err(n(v), n(b_triple[k])) < 1e-3, k
            assert rel_err(n(v), n(b_stock[k])) < 2e-3, k
        elif k.endswith("num_batches_tracked"):
            assert int(v) == int(b_stock[k]) == int(b_triple[k]), k
    assert not single.training                               # collect_stats restores the caller's mode


def test_tensor_core_path_is_graph_capturable(dev):
    """The TMA/wgmma path (descriptor encode + 6 launches per fwd+bwd) must be capturable into a CUDA graph --
    nothing on it may synchronise, allocate through the driver or touch the context during capture -- and a
    replay must reproduce the eager result bit for bit (fixed-order reductions everywhere)."""
    import dwt_b200
    torch.manual_seed(3)
    nimg, c, hw, gs = 8, 128, 24, 64                       # N*HW = 4608 >= 4096 -> tensor-core kernels
    x = (torch.randn(nimg, c, hw, hw, device=dev) + 2.0).requires_grad_(True)
    dy = torch.randn(nimg, c, hw, hw, device=dev)
    m = dwt_b200.WTransform2d(c, gs).to(dev).train()

    def step():
        y = m(x)
        return y, torch.autograd.grad(y, x, dy)[0]

    for _ in range(2):
        y, dx = step()                                     # eager, default stream
    # keep values, not the autograd graph: a live graph pins x's AccumulateGrad node to the default stream, and the
    # engine's end-of-backward sync with that stream is illegal inside a capture (a PyTorch rule, not the library's)
    y_e, dx_e = y.detach().clone(), dx.detach().clone()
    del y, dx
    torch.cuda.synchronize(dev)
    side = torch.cuda.Stream(dev)                          # the usual pre-capture warm-up on a side stream
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
    assert torch.equal(y_g, y_e) and torch.equal(dx_g, dx_e)


# --------------------------------------------------------------------------- paired augmentation (§8f-4)
def _aug_inputs(g, dev):
    return dict(crop_plain=torch.tensor(g("crop_plain"), device=dev), crop_aug=torch.tensor(g("crop_aug"), device=dev),
                flip=torch.tensor(g("flip"), device=dev), affine=torch.tensor(g("affine"), device=dev))


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("case", ["ref", "strong", "tiny"])
def test_augmentation_is_bit_exact_vs_reference_golden(case, channels_last, dev):
    """One launch must give, bit for bit, what the reference's CPU workers give (torchvision crop/flip/to_tensor/
    normalize around the reference's cv2.warpAffine call) -- integer/fixed-point sampling, so the bar is equality."""
    from dwt_b200 import PairedAugment
    z = np.load(os.path.join(HERE, "augment.npz"))
    g = lambda k: z[f"{case}/{k}"]                                  # noqa: E731
    plain, aug = PairedAugment(crop=int(g("crop")))(torch.tensor(g("images"), device=dev), channels_last=channels_last,
                                                     **_aug_inputs(g, dev))
    assert plain.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    assert np.array_equal(plain.cpu().numpy(), g("plain")) and np.array_equal(aug.cpu().numpy(), g("aug"))


def test_augmentation_full_size_into_model_input(dev):
    """Office-Home geometry (256 -> 224), the views written straight into the target | target-aug thirds of the
    model's [3B, 3, 224, 224] input; checked against the numpy oracle (itself pinned bit-exact to the reference)."""
    from dwt_b200 import PairedAugment, draw_params
    from oracle import augment_oracle as A
    rng = np.random.default_rng(8)
    B = 6
    images = rng.integers(0, 256, (B, 256, 256, 3), dtype=np.uint8)
    images[0, :8] = 255; images[1, :, -8:] = 0                        # saturated borders
    p = draw_params(B, 256, 224, rng, affine_sigma=0.1)
    p["affine"][0] = torch.tensor([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])  # identity warp = plain crop of the aug corner
    p["affine"][1] = torch.tensor([[0.5, 0.4, 0.0], [-0.4, 0.6, 0.0]])  # far outside the reference's range
    batch = torch.zeros(3 * B, 3, 224, 224, device=dev)
    pa = PairedAugment(crop=224)
    gp = {k: v.to(dev) for k, v in p.items()}
    pa(torch.tensor(images, device=dev), out_plain=batch[B:2 * B], out_aug=batch[2 * B:], **gp)
    src = rng.integers(0, 256, (B, 256, 256, 3), dtype=np.uint8)
    pa(torch.tensor(src, device=dev), crop_plain=gp["crop_plain"], out_plain=batch[:B], want_aug=False)   # source domain
    o_plain, o_aug = A.paired(images, p["crop_plain"].numpy(), p["crop_aug"].numpy(), p["flip"].numpy(),
                              p["affine"].numpy(), 224)
    o_src, _ = A.paired(src, p["crop_plain"].numpy(), p["crop_aug"].numpy(), np.zeros(B, np.uint8), p["affine"].numpy(), 224)
    out = batch.cpu().numpy()
    assert np.array_equal(out[B:2 * B], o_plain) and np.array_equal(out[2 * B:], o_aug) and np.array_equal(out[:B], o_src)


def test_augmentation_errors(dev):
    from dwt_b200 import PairedAugment, _native
    pa = PairedAugment(crop=8)
    img = torch.zeros(2, 6, 6, 3, dtype=torch.uint8, device=dev)
    cp = torch.zeros(2, 2, dtype=torch.int32, device=dev)
    with pytest.raises(_native.NativeError):
        pa(img, crop_plain=cp, want_aug=False)                        # crop larger than the image
    with pytest.raises(ValueError):
        pa(img.float(), crop_plain=cp, want_aug=False)                # not uint8
    with pytest.raises(ValueError):
        PairedAugment(crop=4)(img, crop_plain=cp)                     # augmented view without its parameters
    with pytest.raises(_native.NativeError):
        PairedAugment(crop=4)(img.cpu(), crop_plain=cp, want_aug=False)
