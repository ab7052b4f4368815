"""Whitening followed by a learnable colouring: the whitening-and-colouring transform (Siarohin, Sangineto, Sebe,
"Whitening and Coloring Batch Transform", ICLR 2019) on the tensor-core whitening kernels.

``WCTransform2d`` is ``WTransform2d`` (same constructor arguments, buffers, attributes, error texts and running-statistic
updates, bit for bit) with two parameters: per group of ``group_size`` channels a learnable matrix ``weight[g]``
(gs x gs, initialised to the identity) and a per-channel ``bias`` (zeros).  With W = L^-1 from S = (1 - eps) cov + eps I:

    y = weight[g] W (x - mean) + bias

A per-channel scale cannot reshape the decorrelation of a group; the colouring matrix can.  It runs in the whitening
kernels themselves (dwt_whiten_color_*): the matrix product weight W is formed per group, the bias starts the apply's
accumulator, and no tensor pass is added over ``WTransform2d``.  Group sizes 8, 16, 32, 64 on the tensor-core kernels
only (H*W >= 32 and a multiple of 4, at least 4096 samples per domain); anything else raises ``NativeError``.  At the
initial parameters the output equals ``WTransform2d``'s bit for bit.  It lives outside whitening.py because the
reference-facing ``whitening`` shim star-imports that file.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import functional as F
from .whitening import WTransform2d, _Whitening


class WCTransform2d(_Whitening):
    def __init__(self, num_features, group_size, running_m=None, running_var=None, momentum=0.1,
                 track_running_stats=True, eps=1e-3, alpha=1):
        super().__init__(num_features, group_size, running_m, running_var, momentum, track_running_stats, eps, alpha)
        self.weight = nn.Parameter(torch.empty(self.num_groups, self.group_size, self.group_size))
        self.bias = nn.Parameter(torch.empty(num_features))
        self.reset_parameters()

    _check_input_dim = WTransform2d._check_input_dim
    _check_group_size = WTransform2d._check_group_size

    def reset_parameters(self):
        """Identity colouring: weight[g] = I, bias = 0 (the output is ``WTransform2d``'s)."""
        with torch.no_grad():
            self.weight.copy_(torch.eye(self.group_size).expand_as(self.weight))
            self.bias.zero_()

    def forward(self, x):
        self._check_input_dim(x)
        self._check_group_size()
        tracking = self.track_running_stats
        return F.color(x, self.weight, self.bias, group_size=self.group_size, n_domains=1,
                       training_stats=self.training or not tracking, eps=self.eps, momentum=self.momentum,
                       update_running=self.training and tracking, running=[(self.running_mean, self.running_variance)])
