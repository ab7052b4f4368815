"""Float64 reference of switchable whitening (dwt_whiten_switch_*, SwitchableWTransform2d).

Per image n and group of gs channels, over the image's M pixels, with the image's own mean and (biased) covariance
mu_n, cov_n and the batch's mu_b, cov_b over all N*M pixels (or the running buffers in eval), and
mix = (a_b, a_i, w_bw, w_iw, w_bn, w_in):

    m_n = a_b mu_b + a_i mu_n
    cov_hat = w_bw cov_b + w_iw cov_n + w_bn diag(cov_b) + w_in diag(cov_n)
    S = (1 - eps) cov_hat + eps I = L L^T,   W = L^-1,   y = W (x - m_n)

sw_torch is built from differentiable torch operations (autograd through torch.linalg.cholesky and inverse gives the exact
backward, mix included) and runs on whatever device x is on; closed_form_backward is the hand-derived backward the
kernels implement.
"""
import torch


def _diag(a):
    return torch.diag_embed(torch.diagonal(a, dim1=-2, dim2=-1))


def sw_torch(x, gs, mix, eps=1e-3, running=None):
    """x [N, C, *], mix [6] -> dict of y (x's shape), m [N, G, gs], w [N, G, gs, gs], mu_n, cov_n, mu_b [G, gs],
    cov_b [G, gs, gs].  running: (mean [C], cov [G, gs, gs]) to whiten with (eval) instead of the batch statistics."""
    n, c = x.shape[:2]
    xg = x.reshape(n, c // gs, gs, -1)
    m_px = xg.shape[-1]
    mu_n = xg.mean(-1)
    xc = xg - mu_n.unsqueeze(-1)
    cov_n = xc @ xc.transpose(-1, -2) / m_px
    if running is None:
        mu_b = xg.mean((0, 3))
        xb = xg - mu_b.unsqueeze(-1)
        cov_b = torch.einsum("ngim,ngjm->gij", xb, xb) / (n * m_px)
    else:
        mu_b = running[0].reshape(c // gs, gs).to(x)
        cov_b = running[1].reshape(c // gs, gs, gs).to(x)
    a_b, a_i, w_bw, w_iw, w_bn, w_in = mix
    m = a_b * mu_b + a_i * mu_n
    chat = w_bw * cov_b + w_iw * cov_n + w_bn * _diag(cov_b) + w_in * _diag(cov_n)
    s = (1 - eps) * chat + eps * torch.eye(gs, dtype=x.dtype, device=x.device)
    w = torch.linalg.inv(torch.linalg.cholesky(s))
    y = (w @ (xg - m.unsqueeze(-1))).reshape(x.shape)
    return dict(y=y, m=m, w=w, mu_n=mu_n, cov_n=cov_n, mu_b=mu_b, cov_b=cov_b)


def closed_form_backward(x, gs, dout, mix, eps=1e-3, running=None):
    """(dx, dmix [6]) of <dout, y> by the formulas the kernels implement, per image and group:
        R = sum_m dout (x - m_n)^T,  P_n = (1 - eps) sym(W^T Phi(-R W^T) W),  dm_n = -W^T sum_m dout
        Q_n = w_iw P_n + w_in diag(P_n),  Q_b = sum_n (w_bw P_n + w_bn diag(P_n))
        dx = W^T dout + (a_i / M) dm_n + (2 / M) Q_n (x - mu_n)
             [train: + (a_b / NM) sum_k dm_k + (2 / NM) Q_b (x - mu_b)]
        dmix = sum over images and groups of (<dm_n, mu_b>, <dm_n, mu_n>, <P_n, cov_b>, <P_n, cov_n>,
                                              <diag P_n, cov_b>, <diag P_n, cov_n>)
    Phi keeps the strict lower triangle and half the diagonal."""
    f = sw_torch(x, gs, mix, eps, running)
    n, c = x.shape[:2]
    a_b, a_i, w_bw, w_iw, w_bn, w_in = mix
    xg = x.reshape(n, c // gs, gs, -1)
    m_px = xg.shape[-1]
    dy = dout.reshape(xg.shape)
    w, wt = f["w"], f["w"].transpose(-1, -2)
    r = dy @ (xg - f["m"].unsqueeze(-1)).transpose(-1, -2)
    p = -(r @ wt)
    p = torch.tril(p, -1) + 0.5 * _diag(p)
    t = wt @ p @ w
    pn = (1 - eps) * 0.5 * (t + t.transpose(-1, -2))
    dm = -(wt @ dy.sum(-1, keepdim=True)).squeeze(-1)
    q = w_iw * pn + w_in * _diag(pn)
    dx = wt @ dy + (a_i / m_px) * dm.unsqueeze(-1) + (2.0 / m_px) * q @ (xg - f["mu_n"].unsqueeze(-1))
    if running is None:
        qb = (w_bw * pn + w_bn * _diag(pn)).sum(0)
        dx = dx + (a_b / (n * m_px)) * dm.sum(0).unsqueeze(-1) + (2.0 / (n * m_px)) * qb @ (xg - f["mu_b"].unsqueeze(-1))
    dmix = torch.stack([(dm * f["mu_b"]).sum(), (dm * f["mu_n"]).sum(), (pn * f["cov_b"]).sum(), (pn * f["cov_n"]).sum(),
                        (pn * _diag(f["cov_b"])).sum(), (pn * _diag(f["cov_n"])).sum()])
    return dx.reshape(x.shape), dmix
