"""Fused domain-triple norm site (extension beyond the reference's module API; SURVEY.md §8f-1).

The reference runs every norm site as
    split/3 -> bns(x_s) | bnt(x_t) | bnt_aug(x_t') -> cat -> cat -> * gamma + beta -> relu
(resnet50_dwt_mec_officehome.py:220-222,335-337): three module calls, two full-tensor
concatenations, an affine pass and a ReLU pass.  ``DomainTripleNorm`` does the whole site in two
tensor-sized kernel launches (statistics, apply; a small finalize launch between them) over the
un-split tensor, the three domains batched on grid.z, gamma/beta/ReLU (and the Bottleneck's residual
tail) folded into the apply pass, and the running-statistic EMA applied source -> target ->
target-aug in order so aliased buffers end exactly as after three sequential module calls
(SURVEY.md H5).  Backward is likewise two tensor-sized launches and also yields dgamma/dbeta and,
for the residual tail, the gradient of the identity branch.

It owns no state: it borrows the running buffers of the three domain modules at call time, and with them their
hyper-parameters -- eps, momentum and, for whitening, the basis: three ``ZCAWTransform2d`` modules make a ZCA site,
three ``ExactZCAWTransform2d`` modules an exact-ZCA site (both on the tensor-core kernels, no fused epilogue), and
modules that disagree on the basis are refused.  A matrix ``gamma`` [C/gs, gs, gs] with ``WTransform2d`` modules at group
sizes 8..64 colours the site instead (the whitening-and-colouring transform, functional.color: y = gamma_g W (x - mean) +
beta, one call for all domains).

``replicated=True`` is the statistics-collection pass (SURVEY.md §8f-3;
resnet50_dwt_mec_officehome.py:380-389): the reference feeds ``cat((data, data, data))`` through
the network in train mode under ``no_grad`` so that every domain branch folds the target batch
into its running buffers.  The three thirds are identical, so are their statistics and their
outputs: here x is the single copy [N, C, H, W], the statistics are computed once, the output is
written once, and a buffer shared by k branches receives the k-fold EMA in one update,
r <- (1-m)^k r + (1 - (1-m)^k) s -- a third of the traffic at every site and a third of the
convolution work between them.  The output is the first third of the reference's: with the first
domain module in eval mode (tracking running statistics) it is x normalised with that module's
running buffers, as ``cat((data, data, data))`` through eval-mode modules gives, and no buffer moves.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _native as nv
from . import functional as F
from .whitening import _Whitening


class DomainTripleNorm(nn.Module):
    def __init__(self, kind, num_features, group_size=4, n_domains=3):
        super().__init__()
        if kind not in ("whiten", "bn"):
            raise ValueError("kind must be 'whiten' or 'bn'")
        self.kind, self.num_features, self.n_domains = kind, num_features, n_domains
        self.group_size = min(num_features, group_size) if kind == "whiten" else 1
        # group sizes 1, 2, 4: gamma / beta / ReLU / residual are folded into the apply kernels.  Larger groups (the
        # tensor-core kernels; e.g. ResNet(..., group_size=64), resnet50_dwt_mec_officehome.py:266): the three domains
        # still share ONE statistics + ONE apply launch with the ordered EMA, the shared affine / ReLU / residual
        # follow as plain tensor ops (two extra elementwise passes; autograd differentiates them).
        self.kernel_epilogue = self.group_size in (1, 2, 4)

    def forward(self, x, domain_modules, gamma, beta, relu=False, residual=None, replicated=False, count_batches=True):
        """x: [n_domains*N, C, H, W]; domain_modules: the per-domain WTransform2d / BatchNorm2d
        modules, whose buffers receive the EMA updates in training mode and normalise the batch in eval mode (as the
        modules themselves would); gamma/beta: [C,1,1];
        residual (needs relu=True): out = relu(norm(x)*gamma + beta + residual), the Bottleneck tail
        (resnet50_dwt_mec_officehome.py:239-240) folded into the apply pass.
        count_batches=False: the caller has already done the `num_batches_tracked += 1` of the three BatchNorm
        modules (batch_norm.py:58) -- a model bumps all its counters with ONE multi-tensor launch per step instead of
        126 one-element kernels."""
        mods = list(domain_modules)
        if len(mods) != self.n_domains:
            raise ValueError(f"expected {self.n_domains} domain modules")
        if x.dim() != 4:
            raise ValueError('expected 4D input (got {}D input)'.format(x.dim()))
        if gamma is not None and gamma.dim() == 3 and tuple(gamma.shape[1:]) != (1, 1):    # [C,1,1]: per channel
            return self._forward_color(x, mods, gamma, beta, relu, residual, replicated, count_batches)
        if not self.kernel_epilogue and torch.bfloat16 in (x.dtype, getattr(residual, "dtype", None)):
            # the tensor epilogue would promote to float32 and round twice: the whole site in float32, rounded once
            out = self.forward(x.float(), mods, gamma, beta, relu, None if residual is None else residual.float(), replicated,
                               count_batches)
            return out.to(x.dtype)
        if replicated:
            return self._forward_replicated(x, mods, gamma, beta, relu, residual, count_batches)
        iterations = self._iterations(mods)
        running, eps, momentum, update = self._running_args(mods, count_batches)
        # modules in eval mode normalise with their running statistics, as each module called on its domain would
        batch_stats = mods[0].training or not mods[0].track_running_stats
        if not self.kernel_epilogue:
            y = F.norm(x, None, None, kind=self.kind, group_size=self.group_size, n_domains=self.n_domains,
                       training_stats=batch_stats, eps=eps, momentum=momentum, update_running=update, running=running,
                       iterations=iterations)
            return self._tensor_epilogue(y, gamma, beta, relu, residual)
        return F.norm(x, gamma, beta, kind=self.kind, group_size=self.group_size, n_domains=self.n_domains,
                      training_stats=batch_stats, eps=eps, momentum=momentum, update_running=update,
                      running=running, relu=relu, residual=residual)

    def _forward_color(self, x, mods, gamma, beta, relu, residual, replicated, count_batches):
        """gamma [C/gs, gs, gs], beta [C] or [C,1,1]: the colouring transform in the whitening kernels (one call for all
        domains, or the replicated pass); ReLU and the residual follow as tensor ops."""
        gs = self.group_size
        if self.kind != "whiten" or self.kernel_epilogue:
            raise nv.NativeError("a matrix gamma (colouring) is built for whitening at group_size 8, 16, 32, 64 on the "
                                 f"tensor-core kernels (got {self.kind}, group_size {gs})")
        if self._iterations(mods):
            raise nv.NativeError("a matrix gamma (colouring) whitens in the Cholesky basis: the domain modules must be "
                                 "WTransform2d")
        if tuple(gamma.shape) != (self.num_features // gs, gs, gs):
            raise ValueError(f"a matrix gamma has shape [C/gs, gs, gs] = {[self.num_features // gs, gs, gs]}, "
                             f"got {list(gamma.shape)}")
        if residual is not None and not relu:
            raise ValueError("a fused residual needs relu=True")
        bias = beta.reshape(-1)
        if replicated:
            y = self._forward_replicated(x, mods, gamma, bias, False, None, count_batches, color=True)
        else:
            running, eps, momentum, update = self._running_args(mods, count_batches)
            y = F.color(x, gamma, bias, group_size=gs, n_domains=self.n_domains,
                        training_stats=mods[0].training or not mods[0].track_running_stats, eps=eps, momentum=momentum,
                        update_running=update, running=running)
        return self._tensor_epilogue(y, None, None, relu, residual)

    def _iterations(self, mods):
        """The whitening basis the domain modules share (functional.norm's iterations: 0 = Cholesky, "eigh" = exact ZCA)."""
        if self.kind != "whiten":
            return 0
        basis = {m._iterations() if isinstance(m, _Whitening) else 0 for m in mods}
        if len(basis) != 1:
            raise ValueError("the domain modules of a whitening site must share one basis (WTransform2d, "
                             "ExactZCAWTransform2d, or ZCAWTransform2d with one number of iterations); got iterations "
                             f"{sorted(basis, key=str)}")
        iterations = basis.pop()
        if iterations and self.kernel_epilogue:
            raise nv.NativeError("the ZCA basis runs on the tensor-core kernels: group_size 8, 16, 32, 64 "
                                 f"(got {self.group_size})")
        return iterations

    def _running_args(self, mods, count_batches):
        """-> (running buffer pairs, eps, momentum, update_running) of a call on mods (statistics of the batch when
        they train, of the running buffers in eval)."""
        m0 = mods[0]
        update = m0.training and m0.track_running_stats
        if self.kind == "whiten":
            running = [(m.running_mean, m.running_variance) for m in mods]
            eps, momentum = m0.eps, m0.momentum
        else:
            if count_batches:
                counters = [m.num_batches_tracked for m in mods if m.training and m.track_running_stats]
                if counters:
                    torch._foreach_add_(counters, 1)
            running = [(m.running_mean, m.running_var) for m in mods]
            eps = m0.eps
            momentum = m0.momentum if m0.momentum is not None or not update else 1.0 / m0.num_batches_tracked.item()
        return running, eps, momentum or 0.0, update

    def forward_with_downsample(self, x, domain_modules, gamma, beta, xd, down, down_modules, down_gamma, down_beta,
                                count_batches=True):
        """relu(self(x) + down(xd)): the residual tail of a downsampling Bottleneck (resnet50_dwt_mec_officehome.py:
        236-240), `down` being the downsample branch's DomainTripleNorm.  Channels-last tensors of one shape with
        both sites on the fused-epilogue kernels run as ONE two-site call (functional.tail_pair: the identity tensor is
        never written); anything else runs the two-call composition down(xd) -> self(x, residual=identity).  Results,
        gradients and running buffers are the same either way -- in bfloat16 too: the two-site kernels round the
        identity to bf16 before they add it, as the composition stores it."""
        mods, down_mods = list(domain_modules), list(down_modules)
        self._iterations(mods)              # a ZCA basis the fused-epilogue kernels lack is refused, never run as Cholesky
        down._iterations(down_mods)
        pair =(self.kernel_epilogue and down.kernel_epilogue and self.kind == down.kind
                and self.group_size == down.group_size and self.n_domains == down.n_domains
                and len(mods) == len(down_mods) == self.n_domains and x.dim() == 4 and x.shape == xd.shape
                and mods[0].training and down_mods[0].training
                and x.dtype == xd.dtype
                and all(F._channels_last_family(t, self.group_size) for t in (x, xd)))
        if not pair:
            identity = down(xd, down_mods, down_gamma, down_beta, relu=False, count_batches=count_batches)
            return self(x, mods, gamma, beta, True, residual=identity, count_batches=count_batches)
        down_args = down._running_args(down_mods, count_batches)
        site_args = self._running_args(mods, count_batches)
        return F.tail_pair(x, xd, gamma, beta, down_gamma, down_beta, kind=self.kind, group_size=self.group_size,
                           n_domains=self.n_domains, sites=(site_args, down_args))

    @staticmethod
    def _tensor_epilogue(y, gamma, beta, relu, residual):
        if residual is not None and not relu:
            raise ValueError("a fused residual needs relu=True")
        if gamma is not None:
            y = y * gamma + beta
        if residual is not None:
            y = y + residual
        return torch.relu(y) if relu else y

    def _forward_replicated(self, x, mods, gamma, beta, relu, residual, count_batches=True, color=False):
        """One copy of the batch stands for all n_domains branches (see the module docstring).  The output is what
        mods[0] gives on x: batch statistics when it trains (or tracks no running statistics), its running buffers in
        eval -- normalised before any training branch that shares those buffers updates them, as in the reference's
        order of calls.  color: gamma is a colouring matrix (_forward_color); the output is returned without epilogue."""
        second = "running_variance" if self.kind == "whiten" else "running_var"
        keep = {}                                  # distinct buffer pair -> product of (1 - factor) over its branches
        for m in mods:
            if not (m.training and m.track_running_stats):
                continue
            if self.kind == "bn":
                if count_batches:
                    m.num_batches_tracked += 1
                f = m.momentum if m.momentum is not None else 1.0 / m.num_batches_tracked.item()
            else:
                f = m.momentum
            rm, rv = m.running_mean, getattr(m, second)
            key = (rm.data_ptr(), rv.data_ptr())
            prod, _ = keep.get(key, (1.0, None))
            keep[key] = (prod * (1.0 - f), (rm, rv))
        means = {k[0] for k in keep}
        seconds = {k[1] for k in keep}
        if len(means) != len(keep) or len(seconds) != len(keep):
            raise ValueError("replicated statistics need each running_mean paired with one second-moment buffer")
        m0 = mods[0]
        iterations = self._iterations(mods)
        common = dict(kind=self.kind, group_size=self.group_size, n_domains=1, training_stats=True, eps=m0.eps,
                      iterations=iterations)
        if self.kernel_epilogue:
            common.update(relu=relu, residual=residual)
            g_arg, b_arg = gamma, beta
        else:
            g_arg = b_arg = None

        def site(training_stats, momentum, update_running, running):
            if color:
                return F.color(x, gamma, beta, group_size=self.group_size, n_domains=1, training_stats=training_stats,
                               eps=m0.eps, momentum=momentum, update_running=update_running, running=running)
            return F.norm(x, g_arg, b_arg, momentum=momentum, update_running=update_running, running=running,
                          **dict(common, training_stats=training_stats))
        out = None
        if not m0.training and m0.track_running_stats:
            out = site(False, 0.0, False, [(m0.running_mean, getattr(m0, second))])
        for prod, pair in keep.values():           # one launch per distinct buffer set (one, in a loaded model)
            y = site(True, 1.0 - prod, True, [pair])
            out = y if out is None else out
        if out is None:
            out = site(True, 0.0, False, [(m0.running_mean, getattr(m0, second))])
        return out if self.kernel_epilogue or color else self._tensor_epilogue(out, gamma, beta, relu, residual)
