"""Channels-last max-pool on the library's own kernels (extension; SURVEY.md §8f "callers either side of the path").

``MaxPool2d(kernel_size, stride, padding)`` stands where the reference model has ``nn.MaxPool2d(kernel_size=3,
stride=2, padding=1)`` (resnet50_dwt_mec_officehome.py:295, applied right behind the stem whitening site at :337-338).
Same results as the stock op bit for bit (ties, NaN, gradient routing); one byte of argmax per output element instead of
an int64.  It takes dense ``torch.channels_last`` CUDA tensors with C % 4 == 0 only -- the layout the benchmark step runs
in; anything else raises (build the model with ``nn.MaxPool2d`` for NCHW).  float32 or bfloat16 (autocast); the output
and the gradient keep the input's dtype.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _native as nv


class _MaxPoolFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, s, p):
        lib = nv.lib()
        dev = nv.require_cuda(x, bf16=True)
        if x.dim() != 4 or not x.is_contiguous(memory_format=torch.channels_last) or x.shape[1] % 4:
            raise nv.NativeError("dwt_b200.MaxPool2d takes dense channels_last [N, C, H, W] tensors with C % 4 == 0; "
                                 f"got shape {tuple(x.shape)}, strides {tuple(x.stride())}")
        n, c, h, w = x.shape
        oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        flags = nv.DTYPE_BF16 if x.dtype == torch.bfloat16 else 0
        y = torch.empty((n, c, oh, ow), dtype=x.dtype, device=dev, memory_format=torch.channels_last)
        idx = torch.empty(n * oh * ow * c, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            nv.check(lib.dwt_maxpool_fwd(nv.ptr(x), nv.ptr(y), nv.ptr(idx), n, h, w, c, k, s, p, flags, nv.stream_ptr(dev)))
        ctx.save_for_backward(idx)
        ctx.cfg = (n, c, h, w, k, s, p, x.dtype, flags)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = nv.lib()
        (idx,) = ctx.saved_tensors
        n, c, h, w, k, s, p, dtype, flags = ctx.cfg
        dy = dy.to(dtype).contiguous(memory_format=torch.channels_last)
        dev = nv.require_cuda(dy, bf16=True)
        dx = torch.empty((n, c, h, w), dtype=dtype, device=dev, memory_format=torch.channels_last)
        with torch.cuda.device(dev):
            nv.check(lib.dwt_maxpool_bwd(nv.ptr(dy), nv.ptr(idx), nv.ptr(dx), n, h, w, c, k, s, p, flags, nv.stream_ptr(dev)))
        return dx, None, None, None


class MaxPool2d(nn.Module):
    def __init__(self, kernel_size, stride=None, padding=0):
        super().__init__()
        self.kernel_size, self.stride, self.padding = int(kernel_size), int(stride or kernel_size), int(padding)

    def forward(self, x):
        return _MaxPoolFunction.apply(x, self.kernel_size, self.stride, self.padding)

    def extra_repr(self):
        return f"kernel_size={self.kernel_size}, stride={self.stride}, padding={self.padding}"
