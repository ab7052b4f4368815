"""Model-level golden fixtures from the UNMODIFIED reference project on CPU, for the tests that compare with it:

    python tests/golden/make_golden_models.py /path/to/reference    # writes tests/golden/ref_*.npz

ref_lenet.npz: usps_mnist.py LeNet outputs (parameters from seeded_params).  ref_resnet.npz: the ResNet's logits, loss,
gradient norms and a fixed sample of every gradient and buffer, and its stem.  ref_modules.npz: the module surface.
"""
from __future__ import annotations

import importlib
import importlib.util
import json
import os
import sys
import warnings

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SUPPORT = os.path.join(ROOT, "tests", "support")
SAMPLE = 128
# tests/test_harness_vs_reference.py and tests/test_config1_plumbing.py import sample_index, seeded_params and the case
# lists below: change them only together with regenerating the fixtures


def sample_index(numel: int, k: int = SAMPLE) -> np.ndarray:
    """Fixed element sample of a tensor with `numel` elements (all of them when it is small)."""
    if numel <= k:
        return np.arange(numel)
    return np.sort(np.random.default_rng(numel).choice(numel, k, replace=False))


def seeded_params(model: torch.nn.Module) -> None:
    """Overwrite every parameter with a fixed seeded draw scaled by 1/sqrt(fan-in), in named_parameters() order."""
    rng = np.random.default_rng(0)
    with torch.no_grad():
        for _, p in model.named_parameters():
            fan_in = max(1, p.numel() // p.shape[0])
            p.copy_(torch.from_numpy((rng.standard_normal(tuple(p.shape)) / np.sqrt(fan_in)).astype(np.float32)))


def lenet(ref: str) -> dict:
    sys.path[:0] = [os.path.join(SUPPORT, "port_utils"), os.path.join(SUPPORT, "stubs"), ref]
    cwd = os.getcwd()
    os.chdir(ref)
    try:
        script = importlib.import_module("usps_mnist")
    finally:
        os.chdir(cwd)
    torch.manual_seed(0)
    net = script.LeNet(group_size=4)
    seeded_params(net)
    x = torch.randn(16, 1, 28, 28)
    out = {"buf/" + k: v.clone().numpy() for k, v in net.named_buffers()}
    out["param_names"] = np.array([k for k, _ in net.named_parameters()])
    net.train()
    out["x"], out["train_out"] = x.numpy(), net(x).detach().numpy()
    net.eval()
    with torch.no_grad():
        out["eval_out"] = net(x).numpy()
    for p in (os.path.join(SUPPORT, "port_utils"), os.path.join(SUPPORT, "stubs"), ref):
        sys.path.remove(p)
    sys.modules.pop("whitening", None)
    return out


def resnet(ref: str) -> dict:
    from harness.synth import synth_batch, synth_state_dict
    sys.path[:0] = [os.path.join(ref, "utils"), ref]
    cwd = os.getcwd()
    os.chdir(ref)
    try:
        script = importlib.import_module("resnet50_dwt_mec_officehome")
        mec = importlib.import_module("consensus_loss")
    finally:
        os.chdir(cwd)
    torch.set_num_threads(8)
    sd = synth_state_dict(1)
    clone = lambda: {k: v.clone() for k, v in sd.items()}       # noqa: E731
    out = {}
    # the whole model: one training step, then eval logits
    x, y = synth_batch(2, 2, size=64)
    net = script.ResNet(script.Bottleneck, [3, 4, 6, 3], clone())
    net.load_state_dict(clone(), strict=False)
    net.train()
    logits = net(x)
    s, t, a = logits.split(logits.shape[0] // 3)
    loss = F.nll_loss(F.log_softmax(s, 1), y) + 0.1 * mec.MinEntropyConsensusLoss(65, "cpu")(t, a)
    loss.backward()
    out["logits"], out["loss"] = logits.detach().numpy(), np.float64(loss.item())
    for k, p in net.named_parameters():
        g = p.grad.reshape(-1)
        out["grad_norm/" + k] = np.float64(g.double().norm().item())
        out["grad_sample/" + k] = g[torch.from_numpy(sample_index(g.numel()))].numpy()
    for k, b in net.state_dict().items():
        v = b.float().reshape(-1)
        out["buf_sample/" + k] = v[torch.from_numpy(sample_index(v.numel()))].numpy()
    net.eval()
    with torch.no_grad():
        out["eval_logits"] = net(x).numpy()
    # the stem: conv1 output and weight gradient against a fixed probe, and the logits of a second batch
    x3, _ = synth_batch(3, 2, size=64)
    net = script.ResNet(script.Bottleneck, [3, 4, 6, 3], clone())
    net.load_state_dict(clone(), strict=False)
    net.train()
    probe = torch.randn(6, 64, 32, 32, generator=torch.Generator().manual_seed(0))
    stem = net.conv1(x3)
    (gw,) = torch.autograd.grad((stem * probe).sum(), net.conv1.weight)
    idx = sample_index(stem.numel(), 16384)
    out["stem_index"], out["stem_sample"] = idx, stem.detach().reshape(-1)[torch.from_numpy(idx)].numpy()
    out["stem_weight_grad"] = gw.numpy()
    out["stem_logits"] = net(x3).detach().numpy()
    return out


def modules(ref: str) -> dict:
    def load(name):
        spec = importlib.util.spec_from_file_location("ref_" + name, os.path.join(ref, "utils", name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod

    def err(fn, *a):
        try:
            fn(*a)
        except ValueError as e:
            return str(e)
        return None

    def sd(m):
        return {k: v.tolist() for k, v in m.state_dict().items()}

    RW, RB = load("whitening"), load("batch_norm")
    res = {"whitening": [], "batch_norm": []}
    for case in WHITEN_CASES:
        r = RW.WTransform2d(**whiten_args(case))
        errs = []
        for bad in whiten_bad_inputs(case):
            errs.append(err(lambda m: (m._check_input_dim(bad), m._check_group_size()), r))
        res["whitening"].append({"attrs": {k: getattr(r, k) for k in WHITEN_ATTRS}, "keys": list(r.state_dict()),
                                 "state": sd(r), "errors": errs})
    for cls, kw in BN_CASES:
        torch.manual_seed(0)
        r = getattr(RB, cls)(6, torch.zeros(6), torch.ones(6), **kw)
        res["batch_norm"].append({"repr": repr(r), "version": r._version, "keys": list(r.state_dict()), "state": sd(r),
                                  "params": [n for n, _ in r.named_parameters()],
                                  "buffers": [n for n, _ in r.named_buffers()],
                                  "errors": [err(r._check_input_dim, torch.zeros(*([2, 6] + [3] * (nd - 2))))
                                             for nd in range(2, 7)]})
    return res


# module-surface cases, shared with tests/test_harness_vs_reference.py
WHITEN_ATTRS = ["num_features", "momentum", "track_running_stats", "eps", "alpha", "group_size", "num_groups"]
WHITEN_CASES = [dict(num_features=8, group_size=4), dict(num_features=8, group_size=16), dict(num_features=48, group_size=32),
                dict(num_features=8, group_size=4, external=True),
                dict(num_features=8, group_size=4, external=True, track_running_stats=False, momentum=0.3, eps=1e-2, alpha=2)]
BN_CASES = [(cls, kw) for cls in ("BatchNorm1d", "BatchNorm2d", "BatchNorm3d")
            for kw in [dict(affine=True), dict(affine=False), dict(affine=True, track_running_stats=False),
                       dict(momentum=None, eps=1e-3)]]


def whiten_args(case: dict) -> dict:
    args = {k: v for k, v in case.items() if k != "external"}
    if case.get("external"):
        args.update(running_m=torch.zeros(1, 8, 1, 1), running_var=torch.ones(2, 4, 4))
    return args


def whiten_bad_inputs(case: dict) -> list:
    return [torch.zeros(2, 8, 3), torch.zeros(2, case["num_features"], 3, 3)]


if __name__ == "__main__":
    ref = os.path.abspath(sys.argv[1])
    sys.path.insert(0, ROOT)
    warnings.filterwarnings("ignore")
    np.savez_compressed(os.path.join(HERE, "ref_lenet.npz"), **lenet(ref))
    np.savez_compressed(os.path.join(HERE, "ref_resnet.npz"), **resnet(ref))
    np.savez_compressed(os.path.join(HERE, "ref_modules.npz"), json=np.array(json.dumps(modules(ref))))
    print("torch", torch.__version__)
