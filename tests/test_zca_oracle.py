"""CPU checks of the ZCA basis: the float64 references against each other and against eigh, the module surface, and the
refusals of the C ABI (argument checks run before any device call, so fake pointers do)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "support"))
import zca_reference as Z  # noqa: E402


# The iteration as defined is not self-correcting: once P_k has converged, a rounding error E in the eigenbasis of N
# (eigenvalues l_i) is multiplied by (2 - r - r^2) / 2 per step, r = sqrt(l_j / l_i) -- by more than 1 in magnitude as
# soon as the condition number exceeds about 2.4.  Past convergence, ill-conditioned groups therefore lose every digit
# even in float64 (test_iteration_is_unstable_past_convergence).  The closed form matches autograd to 1e-10 where the
# function itself is that well determined: T <= 5 up to condition number 1e3, T = 8 up to 1e2, and T = 16 on
# well-conditioned groups.
@pytest.mark.parametrize("gs", [8, 16, 32, 64])
@pytest.mark.parametrize("T, cond", [(1, 1.0), (1, 1e3), (2, 1.0), (2, 1e3), (5, 1.0), (5, 10.0), (5, 1e3), (8, 100.0),
                                     (16, 1.0), (16, 2.0)])
def test_closed_form_backward_matches_autograd(gs, T, cond):
    rng = np.random.default_rng(gs * 100 + T)
    x = Z.conditioned_input(rng, 8, 2 * gs, (4, 5), gs, cond, shift=0.5)
    dy = rng.standard_normal(x.shape)
    xt = torch.tensor(x, requires_grad=True)
    st = {}
    yt, mt, _, Wt = Z.zca_torch(xt, gs, T, state=st)
    (dxt,) = torch.autograd.grad(yt, xt, torch.tensor(dy))
    dx = Z.zca_backward(x, dy, mt.detach().numpy(), Wt.detach().numpy(), st)          # on the same iterates
    err = np.abs(dx - dxt.numpy()).max() / np.abs(dxt.numpy()).max()
    assert err < 1e-10, err
    y, _, W, _ = Z.zca_forward(x, gs, T)                                              # the numpy forward, independently
    assert np.abs(y - yt.detach().numpy()).max() < 1e-10 * np.abs(y).max()
    assert np.abs(W - Wt.detach().numpy()).max() < 1e-10 * np.abs(W).max()


@pytest.mark.parametrize("gs", [8, 64])
def test_iteration_is_unstable_past_convergence(gs):
    """Two float64 evaluations in different summation orders: equal at T = 5, unrelated at T = 16 on a group of
    condition number 1e3 (the function, not an implementation, is ill-determined there)."""
    rng = np.random.default_rng(gs)
    x = Z.conditioned_input(rng, 8, gs, (4, 5), gs, 1e3)
    for T, lo, hi in ((5, 0.0, 1e-12), (16, 1e-2, np.inf)):
        with np.errstate(all="ignore"):
            _, _, W, _ = Z.zca_forward(x, gs, T)
        _, _, _, Wt = Z.zca_torch(torch.tensor(x), gs, T)
        Wt = Wt.numpy()
        err = np.abs(W - Wt).max() / np.abs(Wt).max() if np.isfinite(Wt).all() and np.isfinite(W).all() else np.inf
        assert lo <= err <= hi, (T, err)


@pytest.mark.parametrize("gs", [8, 16, 64])
def test_eval_backward_and_running_statistics(gs):
    rng = np.random.default_rng(gs)
    x = Z.conditioned_input(rng, 4, gs, (5, 5), gs, 30.0)
    rm = rng.standard_normal(gs)
    a = rng.standard_normal((gs, 2 * gs))
    rc = (a @ a.T / (2 * gs))[None]
    y, mean, W, st = Z.zca_forward(x, gs, 5, running_mean=rm, running_cov=rc, train=False)
    dy = rng.standard_normal(x.shape)
    xt = torch.tensor(x, requires_grad=True)
    yt, *_ = Z.zca_torch(xt, gs, 5, running_mean=torch.tensor(rm), running_cov=torch.tensor(rc), train=False)
    (dxt,) = torch.autograd.grad(yt, xt, torch.tensor(dy))
    assert np.abs(y - yt.detach().numpy()).max() < 1e-10 * np.abs(y).max()
    dx = Z.zca_backward(x, dy, mean, W, st, train=False)
    assert np.abs(dx - dxt.numpy()).max() < 1e-10 * np.abs(dx).max()


@pytest.mark.parametrize("gs", [8, 32, 64])
def test_many_iterations_reach_the_inverse_square_root(gs):
    # condition number 2: below the ~2.4 where converged iterates stop being stable (see above)
    rng = np.random.default_rng(7)
    x = Z.conditioned_input(rng, 8, gs, (8, 8), gs, 2.0)
    _, _, W, st = Z.zca_forward(x, gs, 60)
    lam, v = np.linalg.eigh(st["S"][0])
    ref = v @ np.diag(lam ** -0.5) @ v.T
    assert np.abs(W[0] - ref).max() < 1e-10 * np.abs(ref).max()
    y, *_ = Z.zca_forward(x, gs, 60, eps=0.0)
    yg = Z._groups(y, gs)[0]
    assert np.abs(yg @ yg.T / yg.shape[-1] - np.eye(gs)).max() < 1e-8       # eps = 0: the output is white


def test_state_dicts_load_across_bases():
    import dwt_b200
    z, w = dwt_b200.ZCAWTransform2d(64, 16, iterations=3), dwt_b200.WTransform2d(64, 16)
    assert set(z.state_dict()) == set(w.state_dict()) == {"running_mean", "running_variance"}
    with torch.no_grad():
        w.running_mean.normal_()
        w.running_variance.normal_()
    z.load_state_dict(w.state_dict())
    assert all(torch.equal(z.state_dict()[k], w.state_dict()[k]) for k in w.state_dict())
    w2 = dwt_b200.WTransform2d(64, 16)
    w2.load_state_dict(z.state_dict())
    assert torch.equal(w2.running_variance, w.running_variance)
    assert (z.group_size, z.num_groups, z.eps, z.momentum, z.iterations) == (16, 4, 1e-3, 0.1, 3)
    assert dwt_b200.ZCAWTransform2d(8, 16).group_size == 8                    # clamps like WTransform2d


@pytest.mark.parametrize("bad", [0, 17, -1, 2.0, True, None])
def test_bad_iterations_are_refused(bad):
    import dwt_b200
    with pytest.raises(ValueError, match="iterations"):
        dwt_b200.ZCAWTransform2d(64, 16, iterations=bad)


def test_cpu_tensors_and_bad_inputs_are_refused():
    import dwt_b200
    m = dwt_b200.ZCAWTransform2d(64, 16)
    with pytest.raises(dwt_b200._native.NativeError, match="no CPU fallback"):
        m(torch.zeros(2, 64, 8, 8))
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(2, 64, 8))
    with pytest.raises(ValueError, match="expected number of channels divisible by group_size"):
        dwt_b200.ZCAWTransform2d(48, 32)(torch.zeros(2, 48, 3, 3))


def test_domain_site_refuses_mixed_bases():
    import dwt_b200
    site = dwt_b200.DomainTripleNorm("whiten", 64, 16)
    mods = [dwt_b200.ZCAWTransform2d(64, 16), dwt_b200.ZCAWTransform2d(64, 16, iterations=4), dwt_b200.WTransform2d(64, 16)]
    with pytest.raises(ValueError, match="share one basis"):
        site(torch.zeros(6, 64, 8, 8), mods, None, None)
    with pytest.raises(dwt_b200._native.NativeError, match="tensor-core"):
        dwt_b200.DomainTripleNorm("whiten", 64, 4)(torch.zeros(6, 64, 8, 8), [dwt_b200.ZCAWTransform2d(64, 4)] * 3, None, None)


# ---- C ABI refusals, no device call ----------------------------------------------------------------------------------
_FAKE = 1 << 20          # 1 MiB: every fake pointer is 256-byte aligned


def _zca_fwd(lib, N=8, C=128, HW=3136, gs=64, D=1, mode=0, iterations=5, save_p=_FAKE):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_zca_fwd(p, p, N, C, HW, gs, D, mode, 1e-3, 0.1, 0, None, None, iterations, p, p,
                                  None if save_p is None else ctypes.c_void_p(save_p), p, 1 << 40, None)


def _zca_bwd(lib, N=8, C=128, HW=3136, gs=64, D=1, mode=0, iterations=5, save_p=_FAKE):
    p = ctypes.c_void_p(_FAKE)
    return lib.dwt_whiten_zca_bwd(p, p, p, N, C, HW, gs, D, mode, 1e-3, iterations, p, p,
                                  None if save_p is None else ctypes.c_void_p(save_p), p, 1 << 40, None)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native.lib()


@pytest.mark.parametrize("call", [_zca_fwd, _zca_bwd])
@pytest.mark.parametrize("kw, code, text", [
    (dict(gs=1), -4, b"ZCA basis"), (dict(gs=2), -4, b"ZCA basis"), (dict(gs=4), -4, b"ZCA basis"),
    (dict(gs=128), -4, b"ZCA basis"), (dict(C=128, gs=256), -4, b"group_size"),
    (dict(HW=16, N=512), -4, b"ZCA basis"),                                 # HW < 32: the tiled family
    (dict(HW=36, N=64), -4, b"ZCA basis"),                                  # N*HW < 4096 per domain
    (dict(HW=34, N=512), -4, b"ZCA basis"),                                 # HW % 4 != 0
    (dict(HW=36, N=512, mode=0x200), -4, b"HW >= 32 and a multiple of 8"),   # NCHW bf16: HW % 8 != 0
    (dict(C=64, gs=4, mode=0x100), -4, b"ZCA basis"),                       # channels-last group size 4
    (dict(iterations=0), -1, b"iterations 0 outside [1,16]"),
    (dict(iterations=17), -1, b"iterations 17 outside [1,16]"),
    (dict(save_p=None), -1, b"save_p"),
    (dict(save_p=_FAKE + 4), -1, b"save_p must be 16-byte aligned"),
])
def test_c_abi_refusals(lib, call, kw, code, text):
    assert call(lib, **kw) == code
    assert text in lib.dwt_last_error(), lib.dwt_last_error()
