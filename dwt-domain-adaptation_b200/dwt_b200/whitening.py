"""Drop-in for the reference's ``utils/whitening.py`` (same class names, constructor and
forward signatures, attributes, buffers and error texts), computing on hand-written sm_90a
kernels through libdwt_b200.so.

Reference: /root/reference/utils/whitening.py:5-71.
Differences that are deliberate:
  * buffers default to the input's device lazily instead of "CUDA if available"
    (whitening.py:23-24) -- they are created on CPU like any nn.Module buffer and move with
    ``.to(device)``; externally owned buffers are registered as-is, never copied (aliasing
    across the three domain modules survives, SURVEY.md H5);
  * CUDA only: a CPU tensor raises (there is no CPU fallback by design).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import functional as F

# whitening.py:66 and :70-71 -- the second text carries the source file's line continuation (four tabs) verbatim
_MSG_RANK = "expected 4D input (got {}D input)"
_MSG_GROUPS = "expected number of channels divisible by group_size (got {} group_size" + "\t" * 4 + "for {} number of features"


class _Whitening(nn.Module):
    """Hyper-parameters and the two statistics buffers; the arithmetic is one call into the C ABI."""

    def __init__(self, num_features, group_size, running_m=None, running_var=None, momentum=0.1,
                 track_running_stats=True, eps=1e-3, alpha=1):
        super().__init__()
        gs = min(num_features, group_size)                         # whitening.py:14 clamps, :15 floors
        for name, value in (("num_features", num_features), ("momentum", momentum), ("eps", eps), ("alpha", alpha),
                            ("track_running_stats", track_running_stats), ("group_size", gs),
                            ("num_groups", num_features // gs), ("running_m", running_m), ("running_var", running_var)):
            setattr(self, name, value)
        borrowed = track_running_stats and running_m is not None   # whitening.py:19: the caller's tensors, not copies
        mean = running_m if borrowed else torch.zeros(1, num_features, 1, 1)
        # default second moment: an all-ones matrix per group, not the identity (whitening.py:24)
        second = running_var if borrowed else torch.ones(self.num_groups, gs, gs)
        self.register_buffer("running_mean", mean)
        self.register_buffer("running_variance", second)

    def _check_input_dim(self, input):
        raise NotImplementedError

    def _check_group_size(self):
        raise NotImplementedError

    def _iterations(self):
        """The whitening basis as functional.norm's `iterations`: 0 is the inverse Cholesky factor (the ZCA layers,
        zca.py, return their Newton-Schulz iterations or "eigh")."""
        return 0

    def forward(self, x):
        self._check_input_dim(x)
        self._check_group_size()
        tracking = self.track_running_stats
        # train mode updates the buffers even under no_grad and even when they were default-constructed
        # (whitening.py:57-59); eval mode normalises with them (:42-43,50-51)
        return F.norm(x, None, None, kind="whiten", group_size=self.group_size, n_domains=1,
                      training_stats=self.training or not tracking, eps=self.eps, momentum=self.momentum,
                      update_running=self.training and tracking,
                      running=[(self.running_mean, self.running_variance)], iterations=self._iterations())


class WTransform2d(_Whitening):
    def _check_input_dim(self, input):
        rank = input.dim()
        if rank != 4:
            raise ValueError(_MSG_RANK.format(rank))

    def _check_group_size(self):
        if self.num_features % self.group_size:
            raise ValueError(_MSG_GROUPS.format(self.group_size, self.num_features))
