"""Float64 reference of instance whitening (dwt_whiten_instance_*, InstanceWTransform2d).

Per image n and group of gs channels, over the image's M pixels, with S = (1 - eps) cov + eps I = L L^T and W = L^-1:

    y = W (x - mu),   mu and cov (biased) the image's own

iw_torch is built from differentiable torch operations (autograd through torch.linalg.cholesky and inverse gives the exact
backward) and runs on whatever device x is on; closed_form_backward is the hand-derived backward the kernels implement.
"""
import torch


def iw_torch(x, gs, eps=1e-3):
    """x [N, C, *] -> (y, mu [N, G, gs], cov [N, G, gs, gs], W [N, G, gs, gs])."""
    n, c = x.shape[:2]
    xg = x.reshape(n, c // gs, gs, -1)
    mu = xg.mean(-1, keepdim=True)
    xc = xg - mu
    cov = xc @ xc.transpose(-1, -2) / xg.shape[-1]
    s = (1 - eps) * cov + eps * torch.eye(gs, dtype=x.dtype, device=x.device)
    w = torch.linalg.inv(torch.linalg.cholesky(s))
    return (w @ xc).reshape(x.shape), mu.squeeze(-1), cov, w


def closed_form_backward(x, gs, dout, eps=1e-3):
    """dx of <dout, y> by the formulas the kernels implement, per image and group:
        R = sum_m dout xc^T,  Bm = (2 (1 - eps) / M) sym(W^T Phi(-R W^T) W),  dx = W^T (dout - mean_M dout) + Bm xc
    Phi keeps the strict lower triangle and half the diagonal."""
    n, c = x.shape[:2]
    _, mu, _, w = iw_torch(x, gs, eps)
    xc = x.reshape(n, c // gs, gs, -1) - mu.unsqueeze(-1)
    dy = dout.reshape(xc.shape)
    m = xc.shape[-1]
    wt = w.transpose(-1, -2)
    p = -(dy @ xc.transpose(-1, -2) @ wt)
    p = torch.tril(p, -1) + 0.5 * torch.diag_embed(torch.diagonal(p, dim1=-2, dim2=-1))
    sp = wt @ p @ w
    bm = (1 - eps) / m * (sp + sp.transpose(-1, -2))
    return (wt @ (dy - dy.mean(-1, keepdim=True)) + bm @ xc).reshape(x.shape)
