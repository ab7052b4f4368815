"""The measurement harness (harness/resnet50_dwt.py) against the UNMODIFIED reference model
(resnet50_dwt_mec_officehome.py ResNet of the reference project) on CPU, both built on stock ATen layers:
same synthetic checkpoint, same batch -> same logits, loss, gradients, buffers, eval logits.
Guards the topology restatement (incl. the Bottleneck tail that the fused site folds in).  What the reference computed
is stored in tests/golden/ref_resnet.npz and ref_modules.npz (tests/golden/make_golden_models.py); gradients and
buffers are compared through their norms and a fixed sample of their elements."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLDEN, "ref_resnet.npz"))


@pytest.fixture(scope="module")
def gold():
    spec = importlib.util.spec_from_file_location("make_golden_models", os.path.join(GOLDEN, "make_golden_models.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def t(a):
    return torch.from_numpy(np.asarray(a))


def test_harness_equals_reference_model(ref, gold):
    import oracle.torch_port as port
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    torch.set_num_threads(8)
    sd = synth_state_dict(1)
    x, y = synth_batch(2, 2, size=64)
    clone = lambda: {k: v.clone() for k, v in sd.items()}       # noqa: E731
    mine = build_resnet50_dwt(clone(), port)
    assert {k[len("buf_sample/"):] for k in ref.files if k.startswith("buf_sample/")} == set(mine.state_dict())

    mine.train()
    out = mine(x)
    s, tg, a = out.split(out.shape[0] // 3)
    loss = F.nll_loss(F.log_softmax(s, 1), y) + 0.1 * port.MinEntropyConsensusLoss(65, "cpu")(tg, a)
    loss.backward()
    assert torch.allclose(t(ref["logits"]), out.detach(), atol=1e-5) and abs(float(ref["loss"]) - loss.item()) < 1e-5
    for k, p in mine.named_parameters():
        g = p.grad.reshape(-1)
        g1 = t(ref["grad_sample/" + k]).double()
        g2 = g[t(gold.sample_index(g.numel()))].double()
        assert (g1 - g2).norm() <= 1e-4 * g1.norm() + 1e-9, k
        assert abs(g.double().norm().item() - float(ref["grad_norm/" + k])) <= 1e-4 * float(ref["grad_norm/" + k]) + 1e-9, k
    for k, b in mine.state_dict().items():
        v = b.float().reshape(-1)
        assert torch.allclose(t(ref["buf_sample/" + k]), v[t(gold.sample_index(v.numel()))], atol=1e-5), k
    mine.eval()
    with torch.no_grad():
        assert torch.allclose(t(ref["eval_logits"]), mine(x), atol=1e-4)


def test_module_surface_is_the_references_own(gold):
    """Against the UNMODIFIED reference modules: attributes, buffer identity, state-dict keys and initial values (same
    RNG stream), repr, checkpoint-version shim and every error text, string for string."""
    import warnings
    warnings.filterwarnings("ignore")
    from dwt_b200 import batch_norm as B, whitening as W
    want = json.loads(str(np.load(os.path.join(GOLDEN, "ref_modules.npz"))["json"]))

    def err(fn, *a):
        try:
            fn(*a)
        except ValueError as e:
            return str(e)
        return None

    def same_state(m, w):
        return list(m.state_dict()) == w["keys"] and all(
            torch.equal(m.state_dict()[k].cpu(), torch.tensor(w["state"][k], dtype=m.state_dict()[k].dtype)) for k in w["keys"])

    assert len(want["whitening"]) == len(gold.WHITEN_CASES) and len(want["batch_norm"]) == len(gold.BN_CASES)
    for case, w in zip(gold.WHITEN_CASES, want["whitening"]):
        args = gold.whiten_args(case)
        a = W.WTransform2d(**args)
        for k in gold.WHITEN_ATTRS:
            assert getattr(a, k) == w["attrs"][k], (k, case)
        assert a.running_m is args.get("running_m") and a.running_var is args.get("running_var")
        assert same_state(a, w), case
        for bad, e in zip(gold.whiten_bad_inputs(case), w["errors"]):
            check = lambda m: (m._check_input_dim(bad), m._check_group_size())      # noqa: E731
            assert err(check, a) == e, case
    for (cls, kw), w in zip(gold.BN_CASES, want["batch_norm"]):
        torch.manual_seed(0)
        a = getattr(B, cls)(6, torch.zeros(6), torch.ones(6), **kw)
        assert repr(a) == w["repr"] and a._version == w["version"]
        assert same_state(a, w), (cls, kw)
        assert [n for n, _ in a.named_parameters()] == w["params"]
        assert [n for n, _ in a.named_buffers()] == w["buffers"]
        for nd, e in zip(range(2, 7), w["errors"]):
            x = torch.zeros(*([2, 6] + [3] * (nd - 2)))
            assert err(a._check_input_dim, x) == e, (cls, nd)
        if kw.get("track_running_stats", True):
            v1 = {k: v for k, v in a.state_dict().items() if "num_batches" not in k}
            a.load_state_dict(v1)                             # pre-version-2 checkpoint: no counter


def test_space_to_depth_stem_equals_the_reference_stem(ref):
    """The harness option stem_s2d (7x7/2 convolution evaluated as the 4x4/1 convolution of the 2x2 space-to-depth image)
    against the UNMODIFIED reference model's conv1: same output and the same gradient of the [64, 3, 7, 7] weight (fp32
    summation order is the only difference), in both memory formats; and the whole model's logits on top of it.  (The
    GPU golden test at 224x224 runs the same option on the CUDA layers.)"""
    import oracle.torch_port as port
    from harness.resnet50_dwt import build_resnet50_dwt
    from harness.synth import synth_batch, synth_state_dict
    torch.set_num_threads(8)
    sd = synth_state_dict(1)
    x, _ = synth_batch(3, 2, size=64)
    clone = lambda: {k: v.clone() for k, v in sd.items()}       # noqa: E731
    probe = torch.randn(6, 64, 32, 32, generator=torch.Generator().manual_seed(0))
    idx = t(ref["stem_index"])
    r_stem, gr, r_logits = t(ref["stem_sample"]), t(ref["stem_weight_grad"]), t(ref["stem_logits"])
    for cl in (False, True):
        mine = build_resnet50_dwt(clone(), port, channels_last=cl, stem_s2d=True).train()
        xi = x.contiguous(memory_format=torch.channels_last) if cl else x
        assert mine.conv1.weight.shape == gr.shape == (64, 3, 7, 7)
        m_stem = mine._stem(xi)
        assert m_stem.shape == probe.shape
        m_s = m_stem.detach().contiguous().reshape(-1)[idx]
        assert torch.allclose(r_stem, m_s, atol=1e-5), (r_stem - m_s).abs().max()
        (gm,) = torch.autograd.grad((m_stem * probe).sum(), mine.conv1.weight)
        assert (gr - gm).norm() <= 1e-5 * gr.norm(), ((gr - gm).norm() / gr.norm()).item()
        # 2 x 2 pixels per image reach layer4 at this size: the batch statistics amplify the rounding differences
        assert (r_logits - mine(xi)).abs().max() <= 1e-3 * r_logits.abs().max()
