"""Scratch: build the bench model (NHWC, fused sites), run 2 warm-up steps and ONE training step eagerly --
the command to profile for a launch list.  python tools/one_step.py [--stem direct|s2d]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "dwt-domain-adaptation_b200"), ROOT]
import torch, bench, dwt_b200
from harness.synth import synth_batch
dev = torch.device("cuda", 0)
torch.backends.cudnn.benchmark = True
stem = sys.argv[sys.argv.index("--stem") + 1] if "--stem" in sys.argv else bench.DEFAULT_STEM
model = bench.build_model(dwt_b200, dev, "fused", channels_last=True, stem_s2d=stem == "s2d")
sync = None
opt = bench.make_optimizer(model)
head = dwt_b200.HeadLoss(65, 0.1)
im, lb = synth_batch(3, 64)
im, lb = im.to(dev).contiguous(memory_format=torch.channels_last), lb.to(dev)
for _ in range(3):
    bench.train_step(model, None, opt, im, lb, sync, head)
torch.cuda.synchronize()
print("done")
