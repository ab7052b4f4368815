"""Instance whitening: each image whitened by its own statistics, on the tensor-core whitening kernels.

``InstanceWTransform2d`` is to ``WTransform2d`` what ``nn.InstanceNorm2d`` is to ``nn.BatchNorm2d``.  Per image and group of
``group_size`` channels, with the image's own mean and (biased) covariance over its H*W pixels:

    S = (1 - eps) cov + eps I = L L^T,   W = L^-1,   y = W (x - mean)

This removes an image's feature correlations ("style") rather than its domain's: the per-sample statistic of Switchable
Whitening (Pan et al., ICCV 2019), of instance-selective whitening (RobustNet, Choi et al., CVPR 2021) and the whitening
step of WCT style transfer (Li et al., NeurIPS 2017).  There are no running statistics, no buffers and no parameters:
training and evaluation compute the same thing, and the gradient always flows through the per-image statistics.

Group sizes 8, 16, 32, 64 (after ``min(C, group_size)`` clamping, as ``WTransform2d``) with H*W >= 256, float32 or bfloat16,
NCHW or channels-last (dwt_whiten_instance_*, include/dwt_b200.h); anything else raises ``NativeError``.  It lives outside
whitening.py because the reference-facing ``whitening`` shim star-imports that file.
"""
from __future__ import annotations

import torch.nn as nn

from . import functional as F
from .whitening import _MSG_GROUPS, _MSG_RANK


class InstanceWTransform2d(nn.Module):
    def __init__(self, num_features, group_size, eps=1e-3):
        super().__init__()
        self.num_features = num_features
        self.group_size = min(num_features, group_size)          # WTransform2d's clamping
        self.num_groups = num_features // self.group_size
        self.eps = eps

    def extra_repr(self):
        return f"{self.num_features}, group_size={self.group_size}, eps={self.eps}"

    def forward(self, x):
        rank = x.dim()
        if rank != 4:
            raise ValueError(_MSG_RANK.format(rank))
        if self.num_features % self.group_size:
            raise ValueError(_MSG_GROUPS.format(self.group_size, self.num_features))
        if x.shape[1] != self.num_features:
            raise ValueError(f"expected {self.num_features} channels (got {x.shape[1]})")
        return F.instance_whiten(x, group_size=self.group_size, eps=self.eps)
