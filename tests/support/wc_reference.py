"""Float64 reference of the whitening-and-colouring transform (dwt_whiten_color_*, WCTransform2d).

Per group of gs channels, with S = (1 - eps) cov + eps I = L L^T and W = L^-1 (the Cholesky basis of WTransform2d):

    y = color_g W (x - mu) + bias

Training uses the batch mean and biased covariance; eval passes mean / cov (the running buffers).  wc_torch is built from
differentiable torch operations (autograd through torch.linalg.cholesky and inverse gives the exact backward);
closed_form_backward is the hand-derived backward the kernels implement.
"""
import torch


def wc_torch(x, gs, color, bias, eps=1e-3, mean=None, cov=None):
    """x [N, C, *] float64 -> (y, mu [G, gs], cov [G, gs, gs], W [G, gs, gs]); mean [C] / cov [G, gs, gs] given: eval."""
    n, c = x.shape[:2]
    g = c // gs
    xg = x.reshape(n, g, gs, -1).permute(1, 2, 0, 3).reshape(g, gs, -1)
    m = xg.shape[-1]
    if mean is None:
        mu = xg.mean(-1, keepdim=True)
        xc = xg - mu
        cov = xc @ xc.transpose(1, 2) / m
    else:
        mu = mean.reshape(g, gs, 1).to(x.dtype)
        xc = xg - mu
        cov = cov.to(x.dtype)
    s = (1 - eps) * cov + eps * torch.eye(gs, dtype=x.dtype)
    w = torch.linalg.inv(torch.linalg.cholesky(s))
    yg = color.to(x.dtype) @ (w @ xc) + bias.to(x.dtype).reshape(g, gs, 1)
    y = yg.reshape(g, gs, n, -1).permute(2, 0, 1, 3).reshape(x.shape)
    return y, mu.squeeze(-1), cov, w


def closed_form_backward(x, gs, color, dout, eps=1e-3, mean=None, cov=None):
    """-> (dx, dcolor, dbias) of <dout, y> by the formulas the kernels implement:
        R = sum_m dout xc^T,  dcolor = R W^T,  dbias = sum_m dout
        train: R_hat = color^T R,  Bm = (2 (1 - eps) / M) sym(W^T Phi(-R_hat W^T) W),  dx = W^T color^T (dout - mean_M dout) + Bm xc
        eval:  dx = W^T color^T dout
    Phi keeps the strict lower triangle and half the diagonal."""
    n, c = x.shape[:2]
    g = c // gs
    train = mean is None
    _, mu, _, w = wc_torch(x, gs, color, torch.zeros(c, dtype=x.dtype), eps, mean, cov)
    grp = lambda t: t.reshape(n, g, gs, -1).permute(1, 2, 0, 3).reshape(g, gs, -1)
    xc, dy = grp(x) - mu.unsqueeze(-1), grp(dout)
    m = xc.shape[-1]
    color = color.to(x.dtype)
    r = dy @ xc.transpose(1, 2)
    dcolor = r @ w.transpose(1, 2)
    dbias = dy.sum(-1).reshape(-1)
    a1 = w.transpose(1, 2) @ color.transpose(1, 2)
    if train:
        rh = color.transpose(1, 2) @ r
        p = -(rh @ w.transpose(1, 2))
        p = torch.tril(p, -1) + 0.5 * torch.diag_embed(torch.diagonal(p, dim1=1, dim2=2))
        sp = w.transpose(1, 2) @ p @ w
        bm = (1 - eps) / m * (sp + sp.transpose(1, 2))
        dxg = a1 @ (dy - dy.mean(-1, keepdim=True)) + bm @ xc
    else:
        dxg = a1 @ dy
    dx = dxg.reshape(g, gs, n, -1).permute(2, 0, 1, 3).reshape(x.shape)
    return dx, dcolor, dbias
