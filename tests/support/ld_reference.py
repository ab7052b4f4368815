"""Float64 reference of latent-domain whitening (dwt_whiten_latent_*, LatentDomainWTransform2d).

Per group of gs channels, with each image's own mean and (biased) covariance m_n, C_n over its M pixels, weights w [N, D]
and s_d = sum_n w_nd:

    mu_d = sum_n w_nd m_n / s_d,   Sigma_d = sum_n w_nd [C_n + (m_n - mu_d)(m_n - mu_d)^T] / s_d   (or the running buffers)
    S_d = (1 - eps) Sigma_d + eps I = L_d L_d^T,   W_d = L_d^-1,   y_n = sum_d w_nd W_d (x_n - mu_d)

A domain with s_d == 0 is left out of the computation (so autograd gives its weights a zero gradient).  ld_torch is built
from differentiable torch operations (autograd through torch.linalg.cholesky and inverse gives the exact backward, weights
included) and runs on whatever device x is on; closed_form_backward is the hand-derived backward the kernels implement.
"""
import torch


def _phi(a):
    return torch.tril(a, -1) + 0.5 * torch.diag_embed(torch.diagonal(a, dim1=-2, dim2=-1))


def ld_torch(x, gs, w, eps=1e-3, running=None):
    """x [N, C, *], w [N, D] -> dict of y (x's shape), m [N, G, gs], cov [N, G, gs, gs], s [D], live (the domains with
    s_d != 0) and per domain d (None when skipped): mu[d] [G, gs], sigma[d] [G, gs, gs], w_mat[d] [G, gs, gs].
    running: (mean [D, C], cov [D, G, gs, gs]) to whiten with (eval) instead of the weighted statistics."""
    n, c = x.shape[:2]
    g = c // gs
    xg = x.reshape(n, g, gs, -1)
    m_px = xg.shape[-1]
    m = xg.mean(-1)
    xc = xg - m.unsqueeze(-1)
    cov = xc @ xc.transpose(-1, -2) / m_px
    s = w.sum(0)
    d_count = w.shape[1]
    mu, sigma, w_mat, live = [None] * d_count, [None] * d_count, [None] * d_count, []
    y = torch.zeros_like(xg)
    eye = torch.eye(gs, dtype=x.dtype, device=x.device)
    for d in range(d_count):
        if float(s[d].detach()) == 0.0:
            continue
        live.append(d)
        wd = w[:, d]
        if running is None:
            mu[d] = torch.einsum("n,ngi->gi", wd, m) / s[d]
            u = m - mu[d]
            sigma[d] = (torch.einsum("n,ngij->gij", wd, cov) + torch.einsum("n,ngi,ngj->gij", wd, u, u)) / s[d]
        else:
            mu[d] = running[0][d].reshape(g, gs).to(x)
            sigma[d] = running[1][d].reshape(g, gs, gs).to(x)
        w_mat[d] = torch.linalg.inv(torch.linalg.cholesky((1 - eps) * sigma[d] + eps * eye))
        y = y + wd.reshape(n, 1, 1, 1) * (w_mat[d] @ (xg - mu[d].unsqueeze(-1)))
    return dict(y=y.reshape(x.shape), m=m, cov=cov, s=s, live=live, mu=mu, sigma=sigma, w_mat=w_mat)


def closed_form_backward(x, gs, dout, w, eps=1e-3, running=None):
    """(dx, dweights [N, D]) of <dout, y> by the formulas the kernels implement, per group, over the domains with
    s_d != 0 (dweights[:, d] = 0 for the others), with g_n = sum_px dout, R_n = sum_px dout (x - m_n)^T, u_nd = m_n - mu_d:
        Wbar_d = sum_n w_nd [R_n + g_n u_nd^T],  mubar_d = -W_d^T sum_n w_nd g_n,
        P_d = (1 - eps) sym(W_d^T Phi(-Wbar_d W_d^T) W_d)       (Phi: strict lower triangle and half the diagonal)
        dx = sum_d w_nd W_d^T dout + [train] (1/M) sum_d (w_nd / s_d) [mubar_d + 2 P_d (x - mu_d)]
        dweights_nd = sum_g <W_d, R_n + g_n u_nd^T> + [train] (1/s_d) [<mubar_d, u_nd> + <P_d, C_n + u_nd u_nd^T - Sigma_d>]"""
    f = ld_torch(x, gs, w, eps, running)
    n, c = x.shape[:2]
    xg = x.reshape(n, c // gs, gs, -1)
    m_px = xg.shape[-1]
    dy = dout.reshape(xg.shape)
    g = dy.sum(-1)
    r = dy @ (xg - f["m"].unsqueeze(-1)).transpose(-1, -2)
    dx = torch.zeros_like(xg)
    dw = torch.zeros_like(w)
    for d in f["live"]:
        wm, wt, mu, s = f["w_mat"][d], f["w_mat"][d].transpose(-1, -2), f["mu"][d], f["s"][d]
        wd = w[:, d]
        u = f["m"] - mu
        rd = r + g.unsqueeze(-1) * u.unsqueeze(-2)               # sum_px dout (x - mu_d)^T
        dx = dx + wd.reshape(n, 1, 1, 1) * (wt @ dy)
        dw[:, d] = (wm * rd).sum((1, 2, 3))
        if running is None:
            wbar = torch.einsum("n,ngij->gij", wd, rd)
            mubar = -(wt @ torch.einsum("n,ngi->gi", wd, g).unsqueeze(-1)).squeeze(-1)
            t = wt @ _phi(-(wbar @ wt)) @ wm
            p = (1 - eps) * 0.5 * (t + t.transpose(-1, -2))
            dx = dx + (wd / (s * m_px)).reshape(n, 1, 1, 1) * (mubar.unsqueeze(-1) + 2.0 * p @ (xg - mu.unsqueeze(-1)))
            corr = (mubar * u).sum((1, 2)) + (p * (f["cov"] + u.unsqueeze(-1) * u.unsqueeze(-2) - f["sigma"][d])).sum((1, 2, 3))
            dw[:, d] = dw[:, d] + corr / s
    return dx.reshape(x.shape), dw
