"""float64 reference of whitening in the exact ZCA basis (dwt_whiten_eigh_*, ExactZCAWTransform2d), written from its
definition:

    S = (1 - eps) cov + eps I = U diag(lambda) U^T,  W = S^-1/2 = U diag(lambda^-1/2) U^T,  y = W (x - mean)

``exact_torch`` is the function as an ATen op sequence that autograd differentiates.  S^-1/2 is either
``inv_sqrt`` -- torch.linalg.eigh forward, the closed-form Daleckii-Krein backward the bwd_eigh kernel evaluates,

    dL/dS = U [(U^T R U) o F] U^T,  F_ij = -1 / (sqrt(l_i) sqrt(l_j) (sqrt(l_i) + sqrt(l_j))),  R = dL/dW,

finite for repeated eigenvalues -- or (``autograd_eigh=True``) autograd through torch.linalg.eigh itself, whose
backward divides by l_i - l_j and is only usable on well-separated spectra.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


class _InvSqrt(torch.autograd.Function):
    @staticmethod
    def forward(ctx, S):
        lam, U = torch.linalg.eigh(S)
        ctx.save_for_backward(lam, U)
        return (U * lam.rsqrt()[..., None, :]) @ U.transpose(-1, -2)

    @staticmethod
    def backward(ctx, R):
        lam, U = ctx.saved_tensors
        r = lam.sqrt()
        Fm = -1.0 / (r[..., :, None] * r[..., None, :] * (r[..., :, None] + r[..., None, :]))
        Ut = U.transpose(-1, -2)
        return U @ ((Ut @ R @ U) * Fm) @ Ut


def inv_sqrt(S, autograd_eigh=False):
    """S^-1/2 of a batch of symmetric positive definite matrices."""
    if not autograd_eigh:
        return _InvSqrt.apply(S)
    lam, U = torch.linalg.eigh(S)
    return (U * lam.rsqrt()[..., None, :]) @ U.transpose(-1, -2)


def exact_torch(x, gs, eps=1e-3, running_mean=None, running_cov=None, train=True, autograd_eigh=False):
    """x [N, C, H, W] (any device and float dtype; differentiable) -> y, mean [C], un-shrunk covariance [G, gs, gs]
    (train: the batch's), W [G, gs, gs].  Eval (train=False) normalises with running_mean and running_cov."""
    n, c = x.shape[:2]
    g = c // gs
    xg = x.transpose(0, 1).reshape(g, gs, -1)
    if train:
        mean = xg.mean(-1)
        xc = xg - mean[..., None]
        cov = torch.bmm(xc, xc.transpose(1, 2)) / xg.shape[-1]
    else:
        mean = running_mean.reshape(g, gs).to(x.dtype)
        cov = running_cov.reshape(g, gs, gs).to(x.dtype)
    eye = torch.eye(gs, dtype=x.dtype, device=x.device)
    W = inv_sqrt((1 - eps) * cov + eps * eye, autograd_eigh)
    y = F.conv2d(x - mean.reshape(1, c, 1, 1), W.reshape(c, gs, 1, 1), groups=g)
    return y, mean.reshape(-1), cov, W
