"""float64 references of whitening in the ZCA basis (dwt_whiten_zca_*, ZCAWTransform2d), written from its definition:

    S = (1 - eps) cov + eps I,  t = tr S,  N = S / t,  P_0 = I,  P_k = (3 P_{k-1} - P_{k-1}^3 N) / 2,  W = P_T / sqrt(t)
    y = W (x - mean)

* ``zca_forward`` / ``zca_backward``: numpy, the forward and the closed-form backward (the reverse recursion the
  bwd_zca kernel runs), one domain.
* ``zca_torch``: the same function as an ATen op sequence (mean, bmm, the iterations, a grouped 1x1 convolution), which
  autograd differentiates.  In float64 it is the reference of the GPU tests and of the closed form; in float32 on the
  GPU it is the operator-sequence baseline of tools/zca_micro.py.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def _groups(x, gs):
    """[N, C, H, W] -> [G, gs, N*H*W]"""
    n, c = x.shape[:2]
    return np.ascontiguousarray(np.moveaxis(np.asarray(x, np.float64).reshape(n, c, -1), 1, 0)).reshape(c // gs, gs, -1)


def _ungroup(v, shape):
    n, c = shape[:2]
    return np.moveaxis(v.reshape(c, n, -1), 0, 1).reshape(shape)


def zca_forward(x, gs, iterations, eps=1e-3, running_mean=None, running_cov=None, train=True):
    """-> y, mean [C], W [G, gs, gs], state (the backward's inputs: S, the iterates P_0..P_T, t, a).  Eval (train=False)
    normalises with running_mean [C] and running_cov [G, gs, gs]."""
    xg = _groups(x, gs)
    g = xg.shape[0]
    if train:
        mean = xg.mean(-1)
        xc = xg - mean[..., None]
        cov = xc @ np.swapaxes(xc, 1, 2) / xg.shape[-1]
    else:
        mean = np.asarray(running_mean, np.float64).reshape(g, gs)
        cov = np.asarray(running_cov, np.float64).reshape(g, gs, gs)
        xc = xg - mean[..., None]
    eye = np.eye(gs)
    S = (1 - eps) * cov + eps * eye
    t = np.trace(S, axis1=1, axis2=2)[:, None, None]
    N = S / t
    Ps = [np.broadcast_to(eye, S.shape).copy()]
    for _ in range(iterations):
        P = Ps[-1]
        Ps.append(0.5 * (3 * P - P @ P @ P @ N))
    W = Ps[-1] / np.sqrt(t)
    y = _ungroup(W @ xc, np.shape(x))
    return y, mean.reshape(-1), W, dict(S=S, N=N, Ps=Ps, t=t, a=1 - eps, cov=cov)


def zca_grad_S(R, state):
    """dL/dS of L(W(S)) given R = dL/dW [G, gs, gs]: the reverse of the Newton-Schulz recursion."""
    N, Ps, t = state["N"], state["Ps"], state["t"]
    T = len(Ps) - 1
    Q = R / np.sqrt(t)
    tbar = -0.5 * t ** -1.5 * np.sum(R * Ps[T], axis=(1, 2))[:, None, None]
    Nbar = np.zeros_like(N)
    for k in range(T, 0, -1):
        P = Ps[k - 1]
        P2 = P @ P
        Nbar -= 0.5 * P2 @ P @ Q
        QN = Q @ N
        Q = 1.5 * Q - 0.5 * (QN @ P2 + P @ QN @ P + P2 @ QN)
    eye = np.eye(N.shape[-1])
    return Nbar / t + (tbar - np.sum(Nbar * N, axis=(1, 2))[:, None, None] / t) * eye


def zca_backward(x, dy, mean, W, state, train=True):
    """dx of y = W (x - mean): W^T (dy - mean dy) + (a/M)(G + G^T) xc in training, W^T dy in eval."""
    gs = W.shape[-1]
    xg, dg = _groups(x, gs), _groups(dy, gs)
    xc = xg - np.asarray(mean).reshape(xg.shape[0], gs)[..., None]
    Wt = np.swapaxes(W, 1, 2)
    if not train:
        return _ungroup(Wt @ dg, np.shape(x))
    M = xg.shape[-1]
    G = zca_grad_S(dg @ np.swapaxes(xc, 1, 2), state)
    dx = Wt @ (dg - dg.mean(-1, keepdims=True)) + state["a"] / M * (G + np.swapaxes(G, 1, 2)) @ xc
    return _ungroup(dx, np.shape(x))


def zca_torch(x, gs, iterations, eps=1e-3, running_mean=None, running_cov=None, train=True, state=None):
    """The same function in ATen ops on x [N, C, H, W] (any device and float dtype; differentiable).  -> y, mean [C],
    un-shrunk covariance [G, gs, gs] (train: the batch's), W [G, gs, gs].  state: a dict that receives zca_forward's
    state of this computation (numpy float64), for zca_backward on exactly these iterates."""
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
    S = (1 - eps) * cov + eps * eye
    t = S.diagonal(dim1=1, dim2=2).sum(-1)[:, None, None]
    N = S / t
    P = eye.expand(g, gs, gs)
    Ps = [P]
    for _ in range(iterations):
        P = 0.5 * (3 * P - torch.bmm(torch.bmm(torch.bmm(P, P), P), N))
        Ps.append(P)
    W = P / t.sqrt()
    if state is not None:
        def f64(v):
            return v.detach().cpu().double().numpy()
        state.update(S=f64(S), N=f64(N), Ps=[f64(v) for v in Ps], t=f64(t), a=1 - eps, cov=f64(cov))
    y = F.conv2d(x - mean.reshape(1, c, 1, 1), W.reshape(c, gs, 1, 1), groups=g)
    return y, mean.reshape(-1), cov, W


def conditioned_input(rng, n, c, hw, gs, cond, shift=0.0):
    """[n, c, hw[0], hw[1]] whose per-group batch covariance has condition number `cond` exactly (n*h*w >= gs): the
    samples are whitened, then given a log-spaced spectrum from 1 down to 1/cond under a random rotation per group."""
    h, w = hw
    z = rng.standard_normal((n, c, h, w))
    out = np.empty_like(z)
    for g in range(c // gs):
        zg = np.moveaxis(z[:, g * gs:(g + 1) * gs], 1, 0).reshape(gs, -1)
        zg = zg - zg.mean(-1, keepdims=True)
        lam, v = np.linalg.eigh(zg @ zg.T / zg.shape[-1])
        zg = v @ np.diag(lam ** -0.5) @ v.T @ zg
        q, _ = np.linalg.qr(rng.standard_normal((gs, gs)))
        a = q @ np.diag(np.sqrt(np.logspace(0, -np.log10(cond), gs))) @ q.T
        out[:, g * gs:(g + 1) * gs] = np.moveaxis((a @ zg).reshape(gs, n, h, w), 0, 1)
    return out + shift
