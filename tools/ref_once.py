"""Scratch: the reference's operator sequence (oracle/torch_port.py, stock ATen ops) on the GPU -- the command profiled
for a "where the time goes today" launch list.
    python tools/ref_once.py micro     one WTransform2d fwd+bwd at BASELINE configs[1] after 2 warm-ups
    python tools/ref_once.py resnet    one ResNet-50-DWT training step (3x64 images) after 2 warm-ups"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "dwt-domain-adaptation_b200"), ROOT]
import torch
import bench
import oracle.torch_port as port
from harness.synth import synth_batch

dev = torch.device("cuda", 0)
what = sys.argv[1] if len(sys.argv) > 1 else "micro"
if what == "micro":
    N, C, H, gs = 256, 256, 56, 64
    torch.manual_seed(0)
    x = (torch.randn(N, C, H, H, device=dev) + 2.0).requires_grad_(True)
    dy = torch.randn(N, C, H, H, device=dev)
    m = port.WTransform2d(C, gs).to(dev).train()
    for _ in range(3):
        torch.autograd.grad(m(x), x, dy)
else:
    torch.backends.cudnn.benchmark = True
    model = bench.build_model(port, dev, "modules")
    opt = bench.make_optimizer(model)
    mec = port.MinEntropyConsensusLoss(65, dev)
    im, lb = synth_batch(3, 64)
    im, lb = im.to(dev), lb.to(dev)
    for _ in range(3):
        bench.train_step(model, mec, opt, im, lb)
torch.cuda.synchronize()
print("done")
