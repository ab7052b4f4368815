"""Whitening in the ZCA basis: W = S^-1/2 by Newton-Schulz iteration (decorrelated batch norm; IterNorm's iteration).

``ZCAWTransform2d`` is ``WTransform2d`` with the other standard whitening basis: the same constructor arguments, buffers,
attributes, error texts and running-statistic updates, plus ``iterations``.  Per group of ``group_size`` channels, with
S = (1 - eps) cov + eps I as in ``WTransform2d``:

    t = tr S,  N = S / t,  P_0 = I,  P_k = (3 P_{k-1} - P_{k-1}^3 N) / 2  (k = 1..iterations),  W = P_T / sqrt(t)

and y = W (x - mean).  At a finite T this is IterNorm's partial whitening (W -> S^-1/2 as T grows); the backward is
the exact gradient of that function.  The running buffers receive the same EMA of the un-shrunk covariance as
``WTransform2d``'s, bit for bit, so state dicts load into either class.

``ExactZCAWTransform2d`` computes the same basis exactly, W = S^-1/2 by an eigendecomposition of S.

Both layers run on the tensor-core kernels only (dwt_whiten_zca_* / dwt_whiten_eigh_*): group sizes 8, 16, 32, 64, H*W >= 32 and a
multiple of 4, at least 4096 samples per domain.  Anything else raises ``NativeError``; nothing falls back to another
basis or family.  They live outside whitening.py because the reference-facing ``whitening`` shim star-imports that file.
"""
from __future__ import annotations

from . import _native as nv
from .whitening import WTransform2d, _Whitening


class ZCAWTransform2d(_Whitening):
    def __init__(self, num_features, group_size, running_m=None, running_var=None, momentum=0.1,
                 track_running_stats=True, eps=1e-3, alpha=1, iterations=5):
        if isinstance(iterations, bool) or not isinstance(iterations, int) or not 1 <= iterations <= nv.ZCA_MAX_ITERATIONS:
            raise ValueError(f"iterations must be an int in [1, {nv.ZCA_MAX_ITERATIONS}] (got {iterations!r})")
        super().__init__(num_features, group_size, running_m, running_var, momentum, track_running_stats, eps, alpha)
        self.iterations = iterations

    _check_input_dim = WTransform2d._check_input_dim
    _check_group_size = WTransform2d._check_group_size

    def _iterations(self):
        return self.iterations

    def extra_repr(self):
        return f"{self.num_features}, group_size={self.group_size}, iterations={self.iterations}"


class ExactZCAWTransform2d(_Whitening):
    """Whitening in the exact ZCA basis: W = S^-1/2 = U diag(lambda^-1/2) U^T from the eigendecomposition
    S = U diag(lambda) U^T of S = (1 - eps) cov + eps I, and y = W (x - mean) (decorrelated batch norm's whitening).

    ``WTransform2d``'s constructor, buffers, attributes, error texts and running-statistic updates (bit for bit, so state
    dicts load into any of the three classes).  Unlike ``ZCAWTransform2d``'s finite Newton-Schulz iteration, the output
    is white at every condition number; the price is an iterative eigensolver per group (dwt_whiten_eigh_fwd, a cyclic
    Jacobi method) in place of a fixed number of matrix products.  The backward is the exact gradient of S^-1/2
    (Daleckii-Krein), finite for repeated eigenvalues.  A group whose S is not positive definite -- in eval mode, an
    indefinite running buffer -- sets the not-positive-definite status, as in ``WTransform2d``.  Same tensor-core-only
    geometry as ``ZCAWTransform2d``.
    """

    _check_input_dim = WTransform2d._check_input_dim
    _check_group_size = WTransform2d._check_group_size

    def _iterations(self):
        return nv.EIGH
