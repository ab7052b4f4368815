"""Latent-domain whitening: whitening by the statistics of latent domains under per-image soft domain weights, on the
register-resident kernels at group sizes 1, 2, 4 and the tensor-core whitening kernels at 8 to 64.

``LatentDomainWTransform2d`` is the whitening form of the mDA layer of Mancini et al., "Boosting Domain Adaptation by
Discovering Latent Domains" (CVPR 2018).  ``WTransform2d`` and ``DomainTripleNorm`` need every domain as a contiguous,
equal slice of the batch with a hard label; here each image n carries a weight w_nd per domain d -- a softmax the network
infers, or one-hot labels of uneven, interleaved domains -- and per group of ``group_size`` channels:

    s_d = sum_n w_nd,   mu_d = sum_n w_nd m_n / s_d,   Sigma_d = the w-weighted covariance of the images' pixels
    S_d = (1 - eps) Sigma_d + eps I = L_d L_d^T,   W_d = L_d^-1,   y_n = sum_d w_nd W_d (x_n - mu_d)

``forward(x, weights)`` takes weights [N, num_domains] as given (cast to float32; no softmax, no value checks) and returns
their gradient.  A domain whose weights sum to exactly 0 is skipped: it adds to no output and its buffers stay untouched.

Buffers hold one row per domain: ``running_mean`` [D, C] and ``running_variance`` [D, C/gs, gs, gs], initialised as
``WTransform2d``'s (zero mean, an all-ones matrix per group) and updated by its convention, so one-hot weights keep the
buffers a ``WTransform2d`` per domain would.  ``group_size`` clamping, modes (train, eval, ``track_running_stats=False``)
and error texts are ``WTransform2d``'s.  There is no affine; the caller adds it.  1 <= D <= 8, float32 or bfloat16,
NCHW or channels-last.  Group sizes 1, 2, 4 take any H*W (dwt_whiten_latent_small_*: ResNet-50-DWT's stem and layer1
sites and the digits LeNet's sites at group size 4; the clamping gives 1 or 2 on narrow layers); group sizes 8, 16, 32,
64 need H*W >= 256 (dwt_whiten_latent_*, include/dwt_b200.h).  Anything else raises ``NativeError``.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import functional as F
from .whitening import _MSG_GROUPS, _MSG_RANK


class LatentDomainWTransform2d(nn.Module):
    def __init__(self, num_features, group_size, num_domains, momentum=0.1, track_running_stats=True, eps=1e-3):
        super().__init__()
        self.num_features = num_features
        self.group_size = min(num_features, group_size)          # WTransform2d's clamping
        self.num_groups = num_features // self.group_size
        self.num_domains = num_domains
        self.momentum = momentum
        self.track_running_stats = track_running_stats
        self.eps = eps
        gs = self.group_size
        self.register_buffer("running_mean", torch.zeros(num_domains, num_features))
        self.register_buffer("running_variance", torch.ones(num_domains, self.num_groups, gs, gs))

    def extra_repr(self):
        return f"{self.num_features}, group_size={self.group_size}, num_domains={self.num_domains}, eps={self.eps}"

    def forward(self, x, weights, *, gamma=None, beta=None, relu=False, residual=None):
        """gamma / beta ([C] each, together), relu, residual: the site relu(gamma * self(x) + beta [+ residual]); at group
        sizes up to 4 in the same kernels (functional.latent_domain_whiten)."""
        rank = x.dim()
        if rank != 4:
            raise ValueError(_MSG_RANK.format(rank))
        if self.num_features % self.group_size:
            raise ValueError(_MSG_GROUPS.format(self.group_size, self.num_features))
        if x.shape[1] != self.num_features:
            raise ValueError(f"expected {self.num_features} channels (got {x.shape[1]})")
        if weights.dim() != 2 or tuple(weights.shape) != (x.shape[0], self.num_domains):
            raise ValueError(f"expected weights of shape [{x.shape[0]}, {self.num_domains}] (got {list(weights.shape)})")
        tracking = self.track_running_stats
        # WTransform2d's modes: train updates the buffers even under no_grad; eval whitens with them
        return F.latent_domain_whiten(x, weights, group_size=self.group_size, training_stats=self.training or not tracking,
                                      eps=self.eps, momentum=self.momentum, update_running=self.training and tracking,
                                      running=(self.running_mean, self.running_variance), weight=gamma, bias=beta,
                                      relu=relu, residual=residual)
