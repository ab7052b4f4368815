"""Latent-domain batch norm: batch norm by the statistics of latent domains under per-image soft domain weights.

``LatentDomainBatchNorm1d`` / ``LatentDomainBatchNorm2d`` are the mDA layer of Mancini et al., "Boosting Domain
Adaptation by Discovering Latent Domains" (CVPR 2018).  ``BatchNorm2d`` and ``DomainTripleNorm`` need every domain as a
contiguous, equal slice of the batch with a hard label; here each image n carries a weight w_nd per domain d -- a softmax
the network infers, or one-hot labels of uneven, interleaved domains -- and per channel:

    s_d = sum_n w_nd,   mu_d = sum_n w_nd m_n / s_d,   sigma2_d = the w-weighted variance of the images' pixels
    y_n = weight * sum_d w_nd (x_n - mu_d) / sqrt(sigma2_d + eps) + bias

``forward(x, weights)`` takes weights [N, num_domains] as given (cast to float32; no softmax, no value checks) and returns
their gradient.  A domain whose weights sum to exactly 0 is skipped: it adds to no output and its buffers stay untouched.

Buffers hold one row per domain: ``running_mean`` [D, C] (zeros) and ``running_var`` [D, C] (ones), updated by
``F.batch_norm``'s convention (unbiased variance; ``momentum=None`` is the cumulative average), so one-hot weights keep
the buffers a ``BatchNorm2d`` per domain would.  ``weight`` / ``bias`` start as ``torch.nn.BatchNorm2d``'s (ones,
zeros).  Modes (train, eval, ``track_running_stats=False``) and error texts are the package ``BatchNorm2d``'s.  Any C and
spatial size, 1 <= D <= 8, float32 or bfloat16, NCHW or channels-last (dwt_bn_latent_*, include/dwt_b200.h).
"""
from __future__ import annotations

import torch
from torch import nn

from . import functional as F


class _LatentDomainBatchNorm(nn.Module):
    _ranks: tuple = ()
    _rank_text = ""

    def __init__(self, num_features, num_domains, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        self.num_features, self.num_domains = num_features, num_domains
        self.eps, self.momentum = eps, momentum
        self.affine, self.track_running_stats = affine, track_running_stats
        if affine:
            self.weight = nn.Parameter(torch.ones(num_features))
            self.bias = nn.Parameter(torch.zeros(num_features))
        else:
            self.register_parameter("weight", None)
            self.register_parameter("bias", None)
        if track_running_stats:
            self.register_buffer("running_mean", torch.zeros(num_domains, num_features))
            self.register_buffer("running_var", torch.ones(num_domains, num_features))
            self.register_buffer("num_batches_tracked", torch.zeros((), dtype=torch.long))
        else:
            for name in ("running_mean", "running_var", "num_batches_tracked"):
                self.register_buffer(name, None)

    def extra_repr(self):
        return (f"{self.num_features}, num_domains={self.num_domains}, eps={self.eps}, momentum={self.momentum}, "
                f"affine={self.affine}, track_running_stats={self.track_running_stats}")

    def forward(self, x, weights, *, relu=False, residual=None):
        """relu / residual: the site relu(self(x) [+ residual]) in the same kernels (needs affine=True)."""
        if (relu or residual is not None) and self.weight is None:
            raise ValueError("a fused ReLU or residual needs the layer's affine parameters (affine=True)")
        if x.dim() not in self._ranks:
            raise ValueError("expected {} input (got {}D input)".format(self._rank_text, x.dim()))
        if x.shape[1] != self.num_features:
            raise ValueError(f"expected {self.num_features} channels (got {x.shape[1]})")
        if weights.dim() != 2 or tuple(weights.shape) != (x.shape[0], self.num_domains):
            raise ValueError(f"expected weights of shape [{x.shape[0]}, {self.num_domains}] (got {list(weights.shape)})")
        tracking, factor = self.track_running_stats, 0.0
        if self.training and tracking:
            self.num_batches_tracked += 1
            # momentum None = cumulative moving average over the batches seen so far (the package's _BatchNorm)
            factor = self.momentum if self.momentum is not None else 1.0 / self.num_batches_tracked.item()
        batch_stats = self.training or not tracking
        if batch_stats and x.numel() // x.shape[1] <= 1:                   # F.batch_norm's own guard
            raise ValueError("Expected more than 1 value per channel when training, got input size {}".format(
                tuple(x.shape)))
        return F.latent_domain_batch_norm(x, weights, self.weight, self.bias, training_stats=batch_stats, eps=self.eps,
                                          momentum=factor, update_running=self.training and tracking,
                                          running=(self.running_mean, self.running_var) if tracking else (None, None),
                                          relu=relu, residual=residual)


class LatentDomainBatchNorm1d(_LatentDomainBatchNorm):
    _ranks, _rank_text = (2, 3), "2D or 3D"


class LatentDomainBatchNorm2d(_LatentDomainBatchNorm):
    _ranks, _rank_text = (4,), "4D"
