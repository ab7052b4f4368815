"""Float64 reference of latent-domain batch norm (dwt_bn_latent_*, LatentDomainBatchNorm1d / 2d).

Per channel, with each image's own mean and (biased) variance m_n, v_n over its M pixels, weights w [N, D] and
s_d = sum_n w_nd:

    mu_d = sum_n w_nd m_n / s_d,   sigma2_d = sum_n w_nd [v_n + (m_n - mu_d)^2] / s_d   (or the running buffers)
    r_d = (sigma2_d + eps)^-1/2,   y_n = gamma sum_d w_nd r_d (x_n - mu_d) + beta

A domain with s_d == 0 is left out (so autograd gives its weights a zero gradient).  ldbn_torch is built from
differentiable torch operations and runs on whatever device x is on; closed_form_backward is the hand-derived backward the
kernels implement.
"""
import torch


def ldbn_torch(x, w, gamma=None, beta=None, eps=1e-5, running=None):
    """x [N, C, *], w [N, D] -> dict of y (x's shape), m, v [N, C], s [D], and per domain d (None when skipped): mu[d],
    var[d] [C] (the biased sigma2_d).  running: (mean [D, C], var [D, C]) to normalise with (eval)."""
    n, c = x.shape[:2]
    xr = x.reshape(n, c, -1)
    m = xr.mean(-1)
    v = ((xr - m.unsqueeze(-1)) ** 2).mean(-1)
    s = w.sum(0)
    z = torch.zeros_like(xr)
    mus, vars_ = [], []
    for d in range(w.shape[1]):
        if float(s[d].detach()) == 0.0:
            mus.append(None)
            vars_.append(None)
            continue
        wd = w[:, d].unsqueeze(-1)
        if running is None:
            mu = (wd * m).sum(0) / s[d]
            var = (wd * (v + (m - mu) ** 2)).sum(0) / s[d]
        else:
            mu, var = running[0][d], running[1][d]
        mus.append(mu)
        vars_.append(var)
        z = z + wd.unsqueeze(-1) * ((var + eps).rsqrt().unsqueeze(-1) * (xr - mu.unsqueeze(-1)))
    y = z if gamma is None else z * gamma.reshape(1, c, 1) + beta.reshape(1, c, 1)
    return dict(y=y.reshape(x.shape), m=m, v=v, s=s, mu=mus, var=vars_)


def closed_form_backward(x, dout, w, gamma=None, eps=1e-5, running=None):
    """-> dx, dweights [N, D], dgamma, dbeta [C] (the last two None without gamma), by the formulas of dwt_b200.h."""
    n, c = x.shape[:2]
    xr, dyr = x.reshape(n, c, -1), dout.reshape(n, c, -1)
    M = xr.shape[-1]
    f = ldbn_torch(x, w, eps=eps, running=running)
    m, v, s = f["m"], f["v"], f["s"]
    g = dyr if gamma is None else dyr * gamma.reshape(1, c, 1)
    G = g.sum(-1)
    H = (g * (xr - m.unsqueeze(-1))).sum(-1)
    a = torch.zeros_like(m)
    dx = torch.zeros_like(xr)
    dw = torch.zeros_like(w)
    for d in range(w.shape[1]):
        if f["mu"][d] is None:
            continue
        mu, var = f["mu"][d], f["var"][d]
        r = (var + eps).rsqrt()
        wd = w[:, d].unsqueeze(-1)
        a = a + wd * r
        e = m - mu
        first = r * (H + G * e)
        if running is None:
            A = (wd * G).sum(0)
            B = (wd * (H + G * e)).sum(0)
            dx = dx - (wd / (M * s[d])).unsqueeze(-1) * ((r * A).unsqueeze(-1) + (r ** 3 * B).unsqueeze(-1) * (xr - mu.unsqueeze(-1)))
            first = first - (r * A * e + 0.5 * r ** 3 * B * (v + e ** 2 - var)) / s[d]
        dw[:, d] = first.sum(1)
    dx = dx + a.unsqueeze(-1) * g
    if gamma is None:
        return dx.reshape(x.shape), dw, None, None
    zhat = ldbn_torch(x, w, eps=eps, running=running)["y"].reshape(n, c, -1)
    return dx.reshape(x.shape), dw, (dyr * zhat).sum((0, 2)), dyr.sum((0, 2))


def running_update(f, running, momentum, M):
    """The EMA of dwt_bn_latent_fwd on (mean [D, C], var [D, C]) from ldbn_torch's statistics f (copies)."""
    rm, rv = running[0].clone(), running[1].clone()
    for d in range(rm.shape[0]):
        sd = float(f["s"][d].detach())
        if f["mu"][d] is None or M * sd <= 1.0:
            continue
        rm[d] = (1 - momentum) * rm[d] + momentum * f["mu"][d]
        rv[d] = (1 - momentum) * rv[d] + momentum * f["var"][d] * (M * sd / (M * sd - 1))
    return rm, rv
