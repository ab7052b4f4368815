"""BASELINE.json configs[0]: usps_mnist.py USPS->MNIST, group_size=4, 1 epoch -- plumbing.

CPU side: the LeNet restatement used on the GPU (harness/lenet_dwt.py) against the reference script's own LeNet,
through the outputs that model gave on the same weights and batch (tests/golden/ref_lenet.npz, written by
tests/golden/make_golden_models.py from the unmodified reference).  GPU side: one epoch of the restated LeNet on the
CUDA layers.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_models", os.path.join(GOLDEN, "make_golden_models.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_lenet_restatement_matches_reference_lenet():
    import oracle.torch_port as port
    from harness.lenet_dwt import LeNetDWT
    ref = np.load(os.path.join(GOLDEN, "ref_lenet.npz"))
    mine = LeNetDWT(port, group_size=4)
    assert [k for k, _ in mine.named_parameters()] == list(ref["param_names"])
    golden_module().seeded_params(mine)
    bufs = {k[len("buf/"):]: torch.from_numpy(ref[k]) for k in ref.files if k.startswith("buf/")}
    assert set(bufs) == {k for k, _ in mine.named_buffers()}
    mine.load_state_dict({**dict(mine.named_parameters()), **bufs}, strict=True)
    x = torch.from_numpy(ref["x"])
    mine.train()
    assert torch.allclose(mine(x), torch.from_numpy(ref["train_out"]), atol=1e-5)
    mine.eval()
    with torch.no_grad():
        assert torch.allclose(mine(x), torch.from_numpy(ref["eval_out"]), atol=1e-5)


@pytest.mark.gpu
def test_config1_lenet_epoch_on_cuda_layers():
    import dwt_b200
    import oracle.torch_port as port
    from dwt_b200 import _native
    from harness.lenet_dwt import LeNetDWT, train_epoch
    from harness.synth_digits import digit_batches
    dev = torch.device("cuda", 0)
    torch.manual_seed(1)
    model = LeNetDWT(dwt_b200, group_size=4).to(dev)
    twin = LeNetDWT(port, group_size=4).to(dev)           # same topology on stock ATen ops, same weights
    twin.load_state_dict(model.state_dict())
    batches = digit_batches(seed=3, steps=16)
    log = train_epoch(model, torch.optim.SGD(model.parameters(), lr=1e-2, momentum=0.5), batches, dev)
    log_twin = train_epoch(twin, torch.optim.SGD(twin.parameters(), lr=1e-2, momentum=0.5), batches, dev)   # (Adam's sign-like steps amplify 1e-7 differences)
    assert _native.status(dev) == 0
    assert all(abs(a[0] - b[0]) < 2e-2 * max(1.0, abs(b[0])) for a, b in zip(log, log_twin)), (log[-3:], log_twin[-3:])
    assert log[-1][0] < log[0][0]                          # the plumbing run learns
    model.eval(); twin.eval()
    x = batches[0][2].to(dev)
    with torch.no_grad():
        assert (model(x) - twin(x)).abs().max() < 5e-2 * twin(x).abs().max()
