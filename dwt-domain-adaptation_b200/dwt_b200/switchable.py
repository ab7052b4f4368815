"""Switchable whitening: a learned mix of batch and per-image statistics, on the tensor-core whitening kernels.

``SwitchableWTransform2d`` is the whitening layer of Switchable Whitening (Pan et al., ICCV 2019) in the Cholesky basis of
``WTransform2d`` / ``InstanceWTransform2d``.  Per image and group of ``group_size`` channels, with the batch's mean and
covariance (bw, bn; the running buffers in eval) and the image's own (iw, in):

    m = a_b mu_b + a_i mu_n
    cov_hat = w_bw cov_b + w_iw cov_n + w_bn diag(cov_b) + w_in diag(cov_n)
    S = (1 - eps) cov_hat + eps I = L L^T,   W = L^-1,   y = W (x - m)

``components`` picks the statistics to mix: a non-empty subset of ("bw", "iw", "bn", "in"); ("bw", "iw") is the paper's
SW^a and all four its SW^b without layer norm.  ``mean_weight`` and ``var_weight`` hold one logit per component (initialised
to ones): the variance weights are softmax(var_weight), and the mean weights softmax(mean_weight) summed into a_b and a_i,
because "bn" uses the batch mean as "bw" does and "in" the image's as "iw" does.

Buffers, state-dict keys, ``group_size`` clamping, modes and error texts are ``WTransform2d``'s: a ``WTransform2d``'s state
dict loads (the two logits aside), and the running buffers hold the same batch statistics.  There is no affine; the
caller adds it.  Group sizes 8, 16, 32, 64 with H*W >= 256, float32 or bfloat16, NCHW or channels-last
(dwt_whiten_switch_*, include/dwt_b200.h); anything else raises ``NativeError``.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import functional as F
from .whitening import WTransform2d, _Whitening

COMPONENTS = ("bw", "iw", "bn", "in")
_MEAN_SLOT = {"bw": 0, "bn": 0, "iw": 1, "in": 1}        # mix = (a_b, a_i, w_bw, w_iw, w_bn, w_in)
_VAR_SLOT = {"bw": 2, "iw": 3, "bn": 4, "in": 5}


class SwitchableWTransform2d(_Whitening):
    def __init__(self, num_features, group_size, components=("bw", "iw"), running_m=None, running_var=None, momentum=0.1,
                 track_running_stats=True, eps=1e-3):
        comps = tuple(components) if not isinstance(components, str) else (components,)
        if not comps or len(set(comps)) != len(comps) or any(k not in COMPONENTS for k in comps):
            raise ValueError(f"components must be a non-empty subset of {COMPONENTS} without repeats (got {components!r})")
        super().__init__(num_features, group_size, running_m, running_var, momentum, track_running_stats, eps)
        self.components = comps
        self.mean_weight = nn.Parameter(torch.ones(len(comps)))
        self.var_weight = nn.Parameter(torch.ones(len(comps)))
        # scatter of the softmaxes into the six mix slots (not state: a WTransform2d's state dict stays loadable)
        mean_map, var_map = torch.zeros(len(comps), 6), torch.zeros(len(comps), 6)
        for k, name in enumerate(comps):
            mean_map[k, _MEAN_SLOT[name]] = 1.0
            var_map[k, _VAR_SLOT[name]] = 1.0
        self.register_buffer("_mean_map", mean_map, persistent=False)
        self.register_buffer("_var_map", var_map, persistent=False)

    _check_input_dim = WTransform2d._check_input_dim
    _check_group_size = WTransform2d._check_group_size

    def extra_repr(self):
        return f"{self.num_features}, group_size={self.group_size}, components={self.components}, eps={self.eps}"

    def mix(self):
        """The six kernel weights (a_b, a_i, w_bw, w_iw, w_bn, w_in) as a differentiable float32 tensor (no host sync)."""
        pm = torch.softmax(self.mean_weight.float(), 0).unsqueeze(-1)
        pv = torch.softmax(self.var_weight.float(), 0).unsqueeze(-1)
        return (pm * self._mean_map).sum(0) + (pv * self._var_map).sum(0)

    def forward(self, x):
        self._check_input_dim(x)
        self._check_group_size()
        if x.shape[1] != self.num_features:
            raise ValueError(f"expected {self.num_features} channels (got {x.shape[1]})")
        tracking = self.track_running_stats
        # WTransform2d's modes: train updates the buffers even under no_grad; eval whitens with them
        return F.switchable_whiten(x, self.mix(), group_size=self.group_size, training_stats=self.training or not tracking,
                                   eps=self.eps, momentum=self.momentum, update_running=self.training and tracking,
                                   running=(self.running_mean, self.running_variance))
