"""autograd Functions over the C ABI: one forward call + one hand-derived backward call each.

Saved for backward: the layer input x plus the tiny per-group statistics (mean, W) -- never a
centred copy, a transposed copy or the covariance graph the reference's autograd keeps
(utils/whitening.py:44-55).

Activations are float32 or bfloat16 (what torch.autocast(dtype=torch.bfloat16) hands over from a convolution): route()
decides whether the bf16 kernels (DWT_DTYPE_BF16) take a bf16 call or the float32 kernels run on upcast copies.
Statistics, parameters, their gradients and the running buffers are float32 either way, like nn.BatchNorm2d under autocast.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import torch

from . import _native as nv


def _channels_last(x):
    """x is a 4-D tensor dense in torch.channels_last order (and not also NCHW-contiguous)."""
    return x.dim() == 4 and not x.is_contiguous() and x.is_contiguous(memory_format=torch.channels_last)


def _channels_last_family(x, group_size):
    """x runs on the channels-last kernels of group sizes 1, 2, 4 (nv.channels_last_supported) as it is."""
    return _channels_last(x) and nv.channels_last_supported(x.shape[1], group_size)


def _nhwc_tensor_core(x, group_size, n_domains):
    """The channels-last tensor-core rule for x (nv.tensor_core_nhwc_supported on its per-domain geometry) with a
    16-byte-aligned data_ptr(); a misaligned view is not taken (the forward copies it to NCHW)."""
    return (x.dim() == 4 and x.shape[0] % n_domains == 0 and x.data_ptr() % 16 == 0
            and nv.tensor_core_nhwc_supported(x.shape[0] // n_domains, x.shape[1], x.shape[2] * x.shape[3], group_size))


class Route(NamedTuple):
    """How a norm call reaches the kernels (the Python side of route() in csrc/api.cu)."""
    nhwc: bool        # x goes as it is, channels-last (DWT_LAYOUT_NHWC); else NCHW-contiguous
    bf16: bool        # the kernels take the bf16 activations (DWT_DTYPE_BF16)
    cl: bool          # the channels-last kernels of group sizes 1, 2, 4: they also take a second gradient addend
    align: int        # bytes of alignment the kernels need of dout (a misaligned one is copied); 0: any, or refused


def route(x, residual, kind, group_size, n_domains):
    """The Route of a norm call on x (and the residual), or None when the call runs the float32 kernels on upcast copies:
    bf16 activations the bf16 kernels lack (a geometry or alignment they are not built for, mixed dtypes).  Ask again
    for the float32 copies: their rules differ (a channels-last call at group size 128 stays channels-last)."""
    gs = group_size if kind == "whiten" else 1
    dtypes = {x.dtype} | ({residual.dtype} if residual is not None else set())
    cl = _channels_last_family(x, gs)
    if torch.bfloat16 in dtypes and dtypes <= set(_ACT_DTYPES):
        if dtypes != {torch.bfloat16}:
            return None
        if _channels_last(x):   # the bf16 tensor-core kernels stop at group size 64
            tc = kind == "whiten" and residual is None and gs <= nv.MAX_GROUP_SIZE and _nhwc_tensor_core(x, gs, n_domains)
            return Route(True, True, cl, 0 if cl else 16) if cl or tc else None
        if _bf16_small(x, gs, residual) or _bf16_tensor_core(x, kind, gs, n_domains, residual):
            return Route(False, True, False, 8 if gs in (1, 2, 4) else 16)     # register-resident or tensor-core kernels
        return None
    nhwc = cl or (_channels_last(x) and _nhwc_tensor_core(x, gs, n_domains))
    # tensor-core kernels: 16 bytes for their TMA loads (group size 128 in NCHW fp32 as well: it has no other kernel)
    return Route(nhwc, False, cl, 16 if not cl and (nhwc or gs > nv.MAX_GROUP_SIZE) else 0)


def _bf16_tensor_core(x, kind, group_size, n_domains, residual):
    """A bf16 NCHW whitening call the tensor-core kernels take in bf16 (nv.tensor_core_bf16_supported, 16-byte-aligned
    x; a non-contiguous x is copied into a fresh, aligned tensor by the forward)."""
    if kind != "whiten" or residual is not None or x.dim() < 3 or x.shape[0] % n_domains:
        return False
    n, c, hw = x.shape[0] // n_domains, x.shape[1], math.prod(x.shape[2:])
    return nv.tensor_core_bf16_supported(n, c, hw, group_size) and (not x.is_contiguous() or x.data_ptr() % 16 == 0)


def _bf16_small(x, group_size, residual):
    """A bf16 NCHW call the register-resident kernels take in bf16 (nv.small_bf16_supported: whitening at group sizes
    1, 2, 4 or batch norm, HW % 4 == 0): x and the residual bf16 and 8-byte aligned, or non-contiguous (then copied
    into a fresh, aligned tensor by _NormFunction.forward)."""
    return nv.small_bf16_supported(math.prod(x.shape[2:]), group_size) and all(
        t.dtype == torch.bfloat16 and (not t.is_contiguous() or t.data_ptr() % 8 == 0) for t in (x, residual) if t is not None)


def _check_param(name, t, numel):
    """The C ABI takes raw pointers: a strided or mis-sized statistics / affine tensor would be read or written out
    of bounds on the device, where the reference raises a shape error.  Validate before taking data_ptr()."""
    if t is None:
        return
    if t.numel() != numel:
        raise ValueError(f"{name} has {t.numel()} elements, expected {numel}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous (it is written / read through a raw pointer)")


def _check_running(running, c, gs, domains=True):
    """_check_param of (mean, second-moment) running buffer pairs: C and C*gs elements.  domains: name the domain."""
    for d, (rm_t, rv_t) in enumerate(running):
        at = f" of domain {d}" if domains else ""
        _check_param(f"running mean{at}", rm_t, c)
        _check_param(f"running second moment{at}", rv_t, c * gs)


def _bump_versions(running):
    """The kernels wrote the running buffers in place behind autograd's back: bump their version counters (each buffer
    once) so a graph that saved one of them notices (the reference's in-place EMA, whitening.py:58-59, does the same)."""
    seen = set()
    for buf in (t for pair in running for t in pair):
        if buf is not None and id(buf) not in seen:
            seen.add(id(buf))
            torch.autograd.graph.increment_version(buf)


def _prepare_dout(ctx, dout, x, fmt, align=0, cl=False):
    """The incoming gradient as the kernels read it -> (dout, dout2): dout in x's dtype, dense in memory format fmt, its
    data_ptr() a multiple of align (0: any; a misaligned one is copied).  dout2 is the second addend fork_for_sum parked
    on ctx's node (see there): the channels-last kernels of group sizes 1, 2, 4 (cl) add it where they read dout when it
    matches dout; any other path adds it now."""
    dout2 = ctx.__dict__.pop("_dwt_extra_grad", None)
    if dout.dtype != x.dtype:
        dout = dout.to(x.dtype)
    if dout2 is not None and not (cl and dout2.shape == dout.shape and dout2.dtype == dout.dtype
                                  and dout2.is_contiguous(memory_format=torch.channels_last)):
        dout, dout2 = dout + dout2, None
    dout = dout.contiguous(memory_format=fmt)
    if align and dout.data_ptr() % align:        # a fresh tensor keeps the layout
        dout = dout.clone(memory_format=fmt)
    return dout, dout2


def _fwd_entry(lib, kind, basis, head, epilogue, stats, save_p, tail):
    """Call the forward entry point of a norm call in `basis`.  head: (x, y, N, C, HW, gs, n_domains, mode, eps, momentum,
    update_running, running means, running second moments); epilogue: (gamma, beta, residual, ReLU byte map, epilogue
    bits), the colouring matrix and bias in the colour basis; stats: (save_mean, save_w); tail: (workspace, bytes, stream)."""
    if basis == nv.EIGH:
        return lib.dwt_whiten_eigh_fwd(*head, *stats, save_p, *tail)
    if basis == nv.COLOR:
        return lib.dwt_whiten_color_fwd(*head, *epilogue[:2], *stats, *tail)
    if basis:
        return lib.dwt_whiten_zca_fwd(*head, int(basis), *stats, save_p, *tail)
    if kind == "whiten":
        return lib.dwt_whiten_fwd(*head, *epilogue, *stats, *tail)
    return lib.dwt_bn_fwd(*head[:5], *head[6:], *epilogue, *stats, *tail)         # batch norm: no group_size argument


def _bwd_entry(lib, kind, basis, io, dout2, geom, stats, epilogue, grads, save_p, tail):
    """Call the backward entry point of a norm call in `basis`.  io: (x, dout, dx); dout2: the second gradient addend;
    geom: (N, C, HW, gs, n_domains, mode, eps); stats: (save_mean, save_w); epilogue: (gamma, beta, ReLU byte map,
    dresidual, epilogue bits), the colouring matrix in the colour basis; grads: (dgamma, dbeta), (dcolor, dbias) in the
    colour basis; tail: (workspace, bytes, stream)."""
    if basis == nv.EIGH:
        return lib.dwt_whiten_eigh_bwd(*io, *geom, *stats, save_p, *tail)
    if basis == nv.COLOR:
        return lib.dwt_whiten_color_bwd(*io, *geom, *stats, epilogue[0], *grads, *tail)
    if basis:
        return lib.dwt_whiten_zca_bwd(*io, *geom, int(basis), *stats, save_p, *tail)
    x, dout, dx = io
    if kind == "whiten":
        return lib.dwt_whiten_bwd(x, dout, dout2, dx, *geom, *stats, *epilogue, *grads, *tail)
    n, c, hw, _, n_domains, mode, _ = geom                                        # batch norm: no group_size or eps
    return lib.dwt_bn_bwd(x, dout, dout2, dx, n, c, hw, n_domains, mode, *stats, *epilogue, *grads, *tail)


class _NormFunction(torch.autograd.Function):
    """Shared by whitening (kind='whiten') and domain batch norm (kind='bn').

    x is [n_domains*N, C, *]; `running` is a list of n_domains (mean, second-moment) buffer pairs
    (entries may alias); gamma/beta are [C]-sized or None; relu fuses max(.,0) behind the affine; r: route() of the call;
    basis: 0 for the Cholesky basis; 1..16, the Newton-Schulz iterations of the ZCA basis (dwt_whiten_zca_*, whitening
    without gamma/beta or residual; the per-group matrices of the iteration are saved for backward); nv.EIGH for the exact
    ZCA basis (dwt_whiten_eigh_*; the per-group eigenvectors and eigenvalues are saved for backward); or nv.COLOR for the
    Cholesky basis coloured, y = gamma_g W (x - mean) + beta (dwt_whiten_color_*: gamma is the colouring matrix
    [C/gs, gs, gs] and beta the bias with C elements, both float32 and shared by the n_domains domains of x).
    """

    @staticmethod
    def forward(ctx, x, gamma, beta, residual, kind, group_size, n_domains, mode, eps, momentum, update_running,
                running, relu, r, basis):
        lib = nv.lib()
        gs = group_size if kind == "whiten" else 1
        if not r.nhwc and not x.is_contiguous():
            x = x.contiguous()
        n_all, c, hw = x.shape[0], x.shape[1], math.prod(x.shape[2:])
        layout = (nv.LAYOUT_NHWC if r.nhwc else 0) | (nv.DTYPE_BF16 if r.bf16 else 0)
        if n_all % n_domains != 0:
            raise ValueError(f"batch of {n_all} does not split into {n_domains} domains")
        n = n_all // n_domains
        stats = [gamma, beta, *[t for pair in running for t in pair]]
        dev = nv.require_cuda(x, residual, *stats, bf16=True)
        nv.require_cuda(*stats)                      # parameters and running buffers are float32 whatever x is
        _check_running(running, c, gs)
        epi = nv.EPI_NONE
        if basis == nv.COLOR:
            gamma_c, beta_c = _aligned(gamma), _aligned(beta)
            _check_param("color / weight", gamma_c, c * gs)
            _check_param("bias", beta_c, c)
        else:
            _check_param("gamma / weight", gamma, c)
            _check_param("beta / bias", beta, c)
            if basis and (kind != "whiten" or gamma is not None or residual is not None):
                raise nv.NativeError("the ZCA basis whitens without a fused gamma/beta/ReLU epilogue or residual")
            if residual is not None:
                if gamma is None or not relu or residual.shape != x.shape:
                    raise ValueError("a fused residual needs gamma/beta, relu=True and a tensor shaped like x")
                residual = residual.contiguous(memory_format=torch.channels_last) if r.nhwc else residual.contiguous()
            if gamma is not None:
                epi = nv.EPI_AFFINE | (nv.EPI_RELU if relu else 0) | (nv.EPI_RESIDUAL if residual is not None else 0)
                gamma_c, beta_c = gamma.detach().reshape(-1).contiguous(), beta.detach().reshape(-1).contiguous()
            else:
                gamma_c = beta_c = None
        y = torch.empty_like(x)                      # keeps x's memory format
        # residual tail on the channels-last kernels: the apply pass leaves one byte per float4 with the four
        # (out > 0) bits, which is all the backward needs of the output
        mask = torch.empty(x.numel() // 4, dtype=torch.uint8, device=dev) if (residual is not None and r.nhwc) else None
        save_mean = torch.empty(n_domains, c, dtype=torch.float32, device=dev)
        save_w = torch.empty(n_domains, c // gs, gs, gs, dtype=torch.float32, device=dev)
        if basis == nv.EIGH:                         # save_e: U, then the eigenvalues
            save_p = torch.empty(n_domains, c // gs, gs + 1, gs, dtype=torch.float32, device=dev)
        elif basis and basis != nv.COLOR:
            save_p = torch.empty(n_domains, c // gs, basis, gs, gs, dtype=torch.float32, device=dev)
        else:
            save_p = None
        ws = nv.workspace(dev, n, c, hw, gs, n_domains)
        need_running = (mode == nv.MODE_EVAL) or update_running
        rm = nv.ptr_array([p[0] for p in running]) if need_running else None
        rv = nv.ptr_array([p[1] for p in running]) if need_running else None
        head = (nv.ptr(x), nv.ptr(y), n, c, hw, gs, n_domains, mode | layout, eps, momentum, int(update_running), rm, rv)
        with torch.cuda.device(dev):
            rc = _fwd_entry(lib, kind, basis, head, (nv.ptr(gamma_c), nv.ptr(beta_c), nv.ptr(residual), nv.ptr(mask), epi),
                            (nv.ptr(save_mean), nv.ptr(save_w)), nv.ptr(save_p), (nv.ptr(ws), ws.numel(), nv.stream_ptr(dev)))
        nv.check(rc)
        nv.poll_status(dev)
        if update_running and mode == nv.MODE_TRAIN:
            _bump_versions(running)
        # backward of relu(z + residual): dz = dout * (out > 0) is also the residual's gradient
        ctx.residual_mode = None
        if mask is not None:
            # channels-last: the backward reduction masks dout with the saved bits and writes dz, bwd_apply reads it
            ctx.save_for_backward(x, save_mean, save_w, gamma_c, beta_c, mask)
            ctx.residual_mode = "mask"
        elif residual is not None:
            # NCHW: dz is formed by one ATen pass from the saved output; the kernels then run the plain affine epilogue
            ctx.save_for_backward(x, save_mean, save_w, gamma_c, beta_c, y)
            epi = nv.EPI_AFFINE
            ctx.residual_mode = "aten"
        elif save_p is not None:
            ctx.save_for_backward(x, save_mean, save_w, gamma_c, beta_c, save_p)
        else:
            ctx.save_for_backward(x, save_mean, save_w, gamma_c, beta_c)
        ctx.basis = basis
        ctx.cfg = (kind, gs, n_domains, mode | layout, eps, epi, n, c, hw,
                   None if gamma is None else (gamma.shape, beta.shape))
        ctx.route = r
        return y

    @staticmethod
    def backward(ctx, dout):
        lib = nv.lib()
        x, save_mean, save_w, gamma_c, beta_c, *extra = ctx.saved_tensors
        mask = save_p = None
        if ctx.residual_mode == "mask":
            mask = extra[0]
        elif ctx.residual_mode == "aten":
            dout2 = ctx.__dict__.pop("_dwt_extra_grad", None)
            if dout2 is not None:
                dout = dout + dout2
            dout = torch.ops.aten.threshold_backward(dout, extra[0], 0)
        elif extra:
            save_p = extra[0]
        kind, gs, n_domains, mode, eps, epi, n, c, hw, shapes = ctx.cfg
        r = ctx.route
        dout, dout2 = _prepare_dout(ctx, dout, x, torch.channels_last if r.nhwc else torch.contiguous_format, r.align, r.cl)
        dev = nv.require_cuda(dout, bf16=True)
        dx = torch.empty_like(x)                     # x's layout: channels-last when the forward ran NHWC
        want_affine = gamma_c is not None and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2])
        d_res = None
        if ctx.residual_mode == "mask":
            d_res = torch.empty_like(x)              # dz, written even when the residual needs no gradient
        elif ctx.residual_mode == "aten" and ctx.needs_input_grad[3]:
            d_res = dout
        dgamma = torch.empty_like(gamma_c) if want_affine else None
        dbeta = torch.empty_like(beta_c) if want_affine else None
        ws = nv.workspace(dev, n, c, hw, gs, n_domains)
        with torch.cuda.device(dev):
            rc = _bwd_entry(lib, kind, ctx.basis, (nv.ptr(x), nv.ptr(dout), nv.ptr(dx)), nv.ptr(dout2),
                            (n, c, hw, gs, n_domains, mode, eps), (nv.ptr(save_mean), nv.ptr(save_w)),
                            (nv.ptr(gamma_c), nv.ptr(beta_c), nv.ptr(mask), nv.ptr(d_res) if mask is not None else None, epi),
                            (nv.ptr(dgamma), nv.ptr(dbeta)), nv.ptr(save_p), (nv.ptr(ws), ws.numel(), nv.stream_ptr(dev)))
        nv.check(rc)
        if want_affine:
            dgamma, dbeta = dgamma.view(shapes[0]), dbeta.view(shapes[1])
        return (dx, dgamma, dbeta, d_res if ctx.needs_input_grad[3] else None) + (None,) * 11


class _TailPairFunction(torch.autograd.Function):
    """out = relu(site(x) + site_d(xd)): the residual tail of a downsampling Bottleneck, both norm sites (domain-triple,
    gamma/beta each) and the ReLU in the kernels of dwt_tail2_fwd / dwt_tail2_bwd.  Channels-last, training statistics.
    `sites` holds per site (running pairs, eps, momentum, update_running); the running buffers get the same EMA updates
    as from the two-call composition."""

    @staticmethod
    def forward(ctx, x, xd, gamma, beta, gamma_d, beta_d, kind, group_size, n_domains, sites):
        lib = nv.lib()
        gs = group_size if kind == "whiten" else 1
        if not (x.shape == xd.shape and _channels_last_family(x, gs) and _channels_last_family(xd, gs)):
            raise ValueError("the two-site tail takes two channels-last tensors of one shape with a channels-last build")
        if x.shape[0] % n_domains != 0:
            raise ValueError(f"batch of {x.shape[0]} does not split into {n_domains} domains")
        n_all, c = x.shape[0], x.shape[1]
        hw = x.shape[2] * x.shape[3]
        n = n_all // n_domains
        if xd.dtype != x.dtype:
            raise ValueError("the two-site tail takes two tensors of one dtype")
        bf16 = x.dtype == torch.bfloat16
        stats = [gamma, beta, gamma_d, beta_d, *[t for run, *_ in sites for pair in run for t in pair]]
        dev = nv.require_cuda(x, xd, *stats, bf16=True)
        nv.require_cuda(*stats)
        params = [(gamma, beta), (gamma_d, beta_d)]
        c_sites = (nv.TailSite * 2)()
        keep = []                                    # save tensors and pointer arrays alive across the call
        saved = []
        for k, (inp, (g, b), (running, eps, momentum, update)) in enumerate(zip((x, xd), params, sites)):
            _check_running(running, c, gs)
            _check_param("gamma / weight", g, c)
            _check_param("beta / bias", b, c)
            g_c, b_c = g.detach().reshape(-1).contiguous(), b.detach().reshape(-1).contiguous()
            save_mean = torch.empty(n_domains, c, dtype=torch.float32, device=dev)
            save_w = torch.empty(n_domains, c // gs, gs, gs, dtype=torch.float32, device=dev)
            rm = nv.ptr_array([pr[0] for pr in running]) if update else None
            rv = nv.ptr_array([pr[1] for pr in running]) if update else None
            c_sites[k] = nv.TailSite(inp.data_ptr(), eps, momentum, int(update), rm, rv, g_c.data_ptr(), b_c.data_ptr(),
                                     save_mean.data_ptr(), save_w.data_ptr(), None, None, None)
            keep += [g_c, b_c, rm, rv]
            saved += [save_mean, save_w, g_c]
        y = torch.empty_like(x)
        mask = torch.empty(x.numel() // 4, dtype=torch.uint8, device=dev)
        ws = nv.workspace(dev, n, c, hw, gs, n_domains)
        nv_kind = (nv.KIND_WHITEN if kind == "whiten" else nv.KIND_BN) | (nv.DTYPE_BF16 if bf16 else 0)
        with torch.cuda.device(dev):
            rc = lib.dwt_tail2_fwd(nv_kind, c_sites, nv.ptr(y), nv.ptr(mask), n, c, hw, gs, n_domains, nv.ptr(ws), ws.numel(),
                                   nv.stream_ptr(dev))
        nv.check(rc)
        nv.poll_status(dev)
        _bump_versions([pair for running, _, _, update in sites if update for pair in running])
        ctx.save_for_backward(x, xd, mask, *saved)
        ctx.cfg = (nv_kind, gs, n_domains, n, c, hw, [s[1] for s in sites], gamma.shape, gamma_d.shape)
        return y

    @staticmethod
    def backward(ctx, dout):
        lib = nv.lib()
        x, xd, mask, mean0, w0, g0, mean1, w1, g1 = ctx.saved_tensors
        nv_kind, gs, n_domains, n, c, hw, eps, gshape, gshape_d = ctx.cfg
        dout, dout2 = _prepare_dout(ctx, dout, x, torch.channels_last, cl=True)
        dev = nv.require_cuda(dout, bf16=True)
        dz = torch.empty_like(x)
        dx, dxd = torch.empty_like(x), torch.empty_like(xd)
        grads = [torch.empty(2, c, dtype=torch.float32, device=dev) for _ in range(2)]   # (dgamma, dbeta) per site
        c_sites = (nv.TailSite * 2)()
        for k, (inp, mean, w, g, d_in, gr) in enumerate(zip((x, xd), (mean0, mean1), (w0, w1), (g0, g1), (dx, dxd), grads)):
            c_sites[k] = nv.TailSite(inp.data_ptr(), eps[k], 0.0, 0, None, None, g.data_ptr(), g.data_ptr(), mean.data_ptr(),
                                     w.data_ptr(), d_in.data_ptr(), gr[0].data_ptr(), gr[1].data_ptr())
        ws = nv.workspace(dev, n, c, hw, gs, n_domains)
        with torch.cuda.device(dev):
            rc = lib.dwt_tail2_bwd(nv_kind, c_sites, nv.ptr(dout), nv.ptr(dout2), nv.ptr(mask), nv.ptr(dz), n, c, hw, gs, n_domains,
                                   nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        return (dx, dxd, grads[0][0].view(gshape), grads[0][1].view(gshape), grads[1][0].view(gshape_d),
                grads[1][1].view(gshape_d)) + (None,) * 4


def tail_pair(x, xd, gamma, beta, gamma_d, beta_d, *, kind, group_size, n_domains, sites):
    """relu(site(x) + site_d(xd)) in training mode on channels-last tensors of one shape (see _TailPairFunction);
    sites = ((running, eps, momentum, update_running) of site, the same of site_d)."""
    return _TailPairFunction.apply(x, xd, gamma, beta, gamma_d, beta_d, kind, group_size, n_domains,
                                   [(r, float(e), float(m), bool(u)) for r, e, m, u in sites])


class _ForkForSum(torch.autograd.Function):
    """a, b = fork(y): two aliases of y whose gradients are NOT summed by autograd.  y must be the output of a
    _NormFunction, _TailPairFunction or _LatentBandwidthFunction node (the producer): backward hands the first gradient on as y's gradient and parks the second on the
    producer's node, whose backward passes it to the kernels as the second addend (dwt_whiten_bwd's dout2).  If y gets
    other gradients as well, autograd adds them to the first one as usual -- the parked addend is independent of that."""

    @staticmethod
    def forward(ctx, y):
        ctx.producer = y.grad_fn
        return y.view_as(y), y.view_as(y)

    @staticmethod
    def backward(ctx, ga, gb):
        producer, ctx.producer = ctx.producer, None
        if ga is None or gb is None:
            return ga if gb is None else gb
        if producer is None or "_dwt_extra_grad" in producer.__dict__:
            return ga + gb
        producer.__dict__["_dwt_extra_grad"] = gb
        return ga


def fork_for_sum(y):
    """Use the output of a fused site twice -- e.g. as the next Bottleneck's input AND its identity branch
    (resnet50_dwt_mec_officehome.py:217-240) -- without autograd's elementwise addition of the two gradients: returns
    (a, b), two aliases of y.  Falls back to (y, y) when y was not produced by one of this package's norm sites or no
    gradient is being recorded; results are identical either way."""
    fn = getattr(y, "grad_fn", None)
    if not torch.is_grad_enabled() or fn is None or not isinstance(fn, (_NormFunction._backward_cls, _TailPairFunction._backward_cls,
                                                                        _LatentBandwidthFunction._backward_cls)):
        return y, y
    return _ForkForSum.apply(y)


_ACT_DTYPES = (torch.float32, torch.bfloat16)


def norm(x, gamma, beta, *, kind, group_size, n_domains, training_stats, eps, momentum, update_running,
         running, relu=False, residual=None, iterations=0):
    """iterations: 0 whitens in the Cholesky basis; 1..16 in the ZCA basis by that many Newton-Schulz iterations;
    nv.EIGH ("eigh") in the exact ZCA basis by eigendecomposition (both ZCA bases: the tensor-core kernels only, a call
    they cannot take raises NativeError, it is never sent to another family or basis)."""
    if iterations != nv.EIGH and iterations and not 1 <= iterations <= nv.ZCA_MAX_ITERATIONS:
        raise ValueError(f"iterations must be in [1, {nv.ZCA_MAX_ITERATIONS}] (got {iterations})")
    return _norm(x, gamma, beta, residual, kind, group_size, n_domains, training_stats, eps, momentum, update_running,
                 running, relu, iterations)


def _norm(x, gamma, beta, residual, kind, group_size, n_domains, training_stats, eps, momentum, update_running, running,
          relu, basis):
    """A _NormFunction call in `basis` on x as route() takes it."""
    mode = nv.MODE_TRAIN if training_stats else nv.MODE_EVAL
    args = (kind, group_size, n_domains, mode, float(eps), float(momentum), bool(update_running), running, bool(relu))
    r = route(x, residual, kind, group_size, n_domains)
    if r is None:
        # geometries and alignments the bf16 kernels lack (NCHW HW % 4 != 0, BatchNorm1d on [N, C], a misaligned
        # view, ...) or mixed dtypes: the float32 kernels on upcast copies (x.float() keeps channels-last strides), the
        # result (and through autograd every gradient of x and the residual) back in x's dtype
        xf, rf = x.float(), None if residual is None else residual.float()
        y = _NormFunction.apply(xf, gamma, beta, rf, *args, route(xf, rf, kind, group_size, n_domains), basis)
        return y.to(x.dtype)
    return _NormFunction.apply(x, gamma, beta, residual, *args, r, basis)


def _aligned(t):
    """t as a contiguous float32 tensor whose data_ptr() is 16-byte aligned (the colouring entry points' rule)."""
    t = t.detach().contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def color(x, weight, bias, *, group_size, n_domains, training_stats, eps, momentum, update_running, running):
    """y = weight_g W (x - mean) + bias: whitening in the Cholesky basis, then the learnable colouring of each group of
    group_size channels (weight [C/gs, gs, gs], bias with C elements, float32; _NormFunction's colour basis).  The
    tensor-core kernels only: a call they cannot take raises NativeError.  bf16 activations run the bf16 kernels where
    they are built, else the float32 kernels on upcast copies (functional.norm's rule)."""
    return _norm(x, weight, bias, None, "whiten", group_size, n_domains, training_stats, eps, momentum, update_running,
                 running, False, nv.COLOR)


def _tma_ready(x):
    """-> (x dense in its own layout, channels-last or NCHW, with a 16-byte-aligned data_ptr() for the kernels' TMA reads;
    that memory format)."""
    fmt = torch.channels_last if _channels_last(x) else torch.contiguous_format
    x = x.contiguous(memory_format=fmt)
    return (x.clone(memory_format=fmt) if x.data_ptr() % 16 else x), fmt


def _apply_per_image(fn, x, *args):
    """fn.apply(x, *args) for the per-image kernels: a bfloat16 NCHW x whose H*W is not a multiple of 8 (the bf16 kernels'
    TMA rows) runs the same kernels in float32 on an upcast copy, the result in bfloat16."""
    if x.dtype == torch.bfloat16 and not _channels_last(x) and math.prod(x.shape[2:]) % 8:
        return fn.apply(x.float(), *args).to(x.dtype)
    return fn.apply(x, *args)


class _InstanceFunction(torch.autograd.Function):
    """Instance whitening (dwt_whiten_instance_fwd / _bwd): every image of x [N, C, *] whitened by the mean and covariance
    of its own pixels, per group of group_size channels, in the Cholesky basis.  No running statistics; the gradient
    always flows through the per-image mean and covariance.  x is float32 or bfloat16, NCHW-contiguous or (4-D)
    channels-last; it goes to the kernels in its own layout and dtype."""

    @staticmethod
    def forward(ctx, x, group_size, eps):
        dev = nv.require_cuda(x, bf16=True)
        lib = nv.lib()
        gs = group_size
        x, fmt = _tma_ready(x)
        n, c, hw = x.shape[0], x.shape[1], math.prod(x.shape[2:])
        flags = (nv.LAYOUT_NHWC if fmt == torch.channels_last else 0) | (nv.DTYPE_BF16 if x.dtype == torch.bfloat16 else 0)
        y = torch.empty_like(x)
        save_mean = torch.empty(n, c, dtype=torch.float32, device=dev)
        save_w = torch.empty(n, max(c // gs, 1), gs, gs, dtype=torch.float32, device=dev)
        ws = nv.grow_workspace(dev, lib.dwt_instance_workspace_bytes(n, c, hw, gs))
        with torch.cuda.device(dev):
            rc = lib.dwt_whiten_instance_fwd(nv.ptr(x), nv.ptr(y), n, c, hw, gs, flags, eps, nv.ptr(save_mean),
                                             nv.ptr(save_w), nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        nv.poll_status(dev)
        ctx.save_for_backward(x, save_mean, save_w)
        ctx.cfg = (gs, flags, eps, n, c, hw, fmt)
        return y

    @staticmethod
    def backward(ctx, dout):
        lib = nv.lib()
        x, save_mean, save_w = ctx.saved_tensors
        gs, flags, eps, n, c, hw, fmt = ctx.cfg
        dout, _ = _prepare_dout(ctx, dout, x, fmt, 16)
        dev = nv.require_cuda(dout, bf16=True)
        dx = torch.empty_like(x)
        ws = nv.grow_workspace(dev, lib.dwt_instance_workspace_bytes(n, c, hw, gs))
        with torch.cuda.device(dev):
            rc = lib.dwt_whiten_instance_bwd(nv.ptr(x), nv.ptr(dout), nv.ptr(dx), n, c, hw, gs, flags, eps, nv.ptr(save_mean),
                                             nv.ptr(save_w), nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        return dx, None, None


def instance_whiten(x, *, group_size, eps):
    """Instance whitening of x [N, C, *]: per image n and group g of group_size channels, with M pixels,
    S = (1 - eps) cov + eps I of the image's own (biased) covariance, W = inverse(cholesky(S)), y = W (x - mean).
    The tensor-core kernels only (group sizes 8, 16, 32, 64, H*W >= 256; dwt_b200.h): a call they cannot take raises
    NativeError with the library's reason and is never sent to another kernel family.  A bfloat16 NCHW x whose H*W is not
    a multiple of 8 (the bf16 kernels' TMA rows) runs the same kernels in float32 on an upcast copy, the result in
    bfloat16."""
    if x.dim() < 3:
        raise ValueError(f"instance whitening expects [N, C, *] input (got {x.dim()}D input)")
    nv.require_cuda(x, bf16=True)
    return _apply_per_image(_InstanceFunction, x, int(group_size), float(eps))


class _SwitchFunction(torch.autograd.Function):
    """Switchable whitening (dwt_whiten_switch_fwd / _bwd): every image of x [N, C, *] whitened by a mixture, with the six
    weights of mix (a_b, a_i, w_bw, w_iw, w_bn, w_in; float32, on the device), of the batch's and its own mean and
    covariance, per group of group_size channels, in the Cholesky basis.  The gradient of mix is returned.  Running buffers
    as _NormFunction's (one domain).  x is float32 or bfloat16, NCHW-contiguous or (4-D) channels-last; it goes to the
    kernels in its own layout and dtype."""

    @staticmethod
    def forward(ctx, x, mix, group_size, mode, eps, momentum, update_running, running):
        dev = nv.require_cuda(x, bf16=True)
        rm_t, rv_t = running
        nv.require_cuda(mix, rm_t, rv_t)
        lib = nv.lib()
        gs = group_size
        x, fmt = _tma_ready(x)
        n, c, hw = x.shape[0], x.shape[1], math.prod(x.shape[2:])
        mix_c = _aligned(mix)
        _check_param("mix", mix_c, 6)
        need_running = (mode == nv.MODE_EVAL) or update_running
        if need_running:
            _check_running([running], c, gs, domains=False)
        flags = mode | (nv.LAYOUT_NHWC if fmt == torch.channels_last else 0) | (nv.DTYPE_BF16 if x.dtype == torch.bfloat16 else 0)
        y = torch.empty_like(x)
        g = max(c // gs, 1)
        save_mean = torch.empty(n, c, dtype=torch.float32, device=dev)
        save_w = torch.empty(n, g, gs, gs, dtype=torch.float32, device=dev)
        save_stats = torch.empty(n + 1, g, gs * gs + gs, dtype=torch.float32, device=dev)
        ws = nv.grow_workspace(dev, lib.dwt_switch_workspace_bytes(n, c, hw, gs))
        rm, rv = (nv.ptr(rm_t), nv.ptr(rv_t)) if need_running else (None, None)
        with torch.cuda.device(dev):
            rc = lib.dwt_whiten_switch_fwd(nv.ptr(x), nv.ptr(y), n, c, hw, gs, flags, eps, momentum, int(update_running), rm,
                                           rv, nv.ptr(mix_c), nv.ptr(save_mean), nv.ptr(save_w), nv.ptr(save_stats),
                                           nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        nv.poll_status(dev)
        if update_running and mode == nv.MODE_TRAIN:
            _bump_versions([running])
        ctx.save_for_backward(x, mix_c, save_mean, save_w, save_stats)
        ctx.cfg = (gs, flags, eps, n, c, hw, fmt)
        return y

    @staticmethod
    def backward(ctx, dout):
        lib = nv.lib()
        x, mix_c, save_mean, save_w, save_stats = ctx.saved_tensors
        gs, flags, eps, n, c, hw, fmt = ctx.cfg
        dout, _ = _prepare_dout(ctx, dout, x, fmt, 16)
        dev = nv.require_cuda(dout, bf16=True)
        dx = torch.empty_like(x)
        dmix = torch.empty(6, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        ws = nv.grow_workspace(dev, lib.dwt_switch_workspace_bytes(n, c, hw, gs))
        with torch.cuda.device(dev):
            rc = lib.dwt_whiten_switch_bwd(nv.ptr(x), nv.ptr(dout), nv.ptr(dx), n, c, hw, gs, flags, eps, nv.ptr(mix_c),
                                           nv.ptr(save_mean), nv.ptr(save_w), nv.ptr(save_stats), nv.ptr(dmix), nv.ptr(ws),
                                           ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        return dx, dmix, None, None, None, None, None, None


def switchable_whiten(x, mix, *, group_size, training_stats, eps, momentum, update_running, running):
    """Switchable whitening of x [N, C, *]: per image n and group g of group_size channels, with the image's own mean and
    (biased) covariance mu_n, cov_n and the batch's mu_b, cov_b (training_stats=False: the running buffers), and
    mix = (a_b, a_i, w_bw, w_iw, w_bn, w_in), a float32 tensor of 6 used as given (no softmax):
        m = a_b mu_b + a_i mu_n,  cov_hat = w_bw cov_b + w_iw cov_n + w_bn diag(cov_b) + w_in diag(cov_n),
        S = (1 - eps) cov_hat + eps I,  W = inverse(cholesky(S)),  y = W (x - m).
    running = (mean with C elements, second moment [C/gs, gs, gs]): read when training_stats is False; updated with
    (mu_b, cov_b) by momentum when training_stats and update_running.  mix gets its gradient.
    The tensor-core kernels only (group sizes 8, 16, 32, 64, H*W >= 256; dwt_b200.h): a call they cannot take raises
    NativeError with the library's reason and is never sent to another kernel family.  A bfloat16 NCHW x whose H*W is not
    a multiple of 8 (the bf16 kernels' TMA rows) runs the same kernels in float32 on an upcast copy, the result in
    bfloat16."""
    if x.dim() < 3:
        raise ValueError(f"switchable whitening expects [N, C, *] input (got {x.dim()}D input)")
    nv.require_cuda(x, bf16=True)
    mode = nv.MODE_TRAIN if training_stats else nv.MODE_EVAL
    args = (int(group_size), mode, float(eps), float(momentum), bool(update_running), tuple(running))
    return _apply_per_image(_SwitchFunction, x, mix.float(), *args)


class _LatentFunction(torch.autograd.Function):
    """Latent-domain whitening (dwt_whiten_latent_fwd / _bwd): every image of x [N, C, *] whitened by the statistics of
    n_domains latent domains under its row of weights [N, n_domains] (float32, on the device), per group of group_size
    channels, in the Cholesky basis.  The gradient of weights is returned.  Running buffers: (mean [D, C], second moment
    [D, C/gs, gs, gs]), one row per domain.  x is float32 or bfloat16, NCHW-contiguous or (4-D) channels-last; it goes to
    the kernels in its own layout and dtype."""

    @staticmethod
    def forward(ctx, x, weights, group_size, mode, eps, momentum, update_running, running):
        dev = nv.require_cuda(x, bf16=True)
        rm_t, rv_t = running
        nv.require_cuda(weights, rm_t, rv_t)
        lib = nv.lib()
        gs = group_size
        x, fmt = _tma_ready(x)
        n, c, hw = x.shape[0], x.shape[1], math.prod(x.shape[2:])
        k = weights.shape[1]
        w_c = _aligned(weights)
        need_running = (mode == nv.MODE_EVAL) or update_running
        if need_running:
            _check_param("running mean", rm_t, k * c)
            _check_param("running second moment", rv_t, k * c * gs)
        flags = mode | (nv.LAYOUT_NHWC if fmt == torch.channels_last else 0) | (nv.DTYPE_BF16 if x.dtype == torch.bfloat16 else 0)
        y = torch.empty_like(x)
        g = max(c // gs, 1)
        rec = gs * gs + gs
        save_mean = torch.empty(n, c, dtype=torch.float32, device=dev)
        save_w = torch.empty(n, g, gs, gs, dtype=torch.float32, device=dev)
        save_stats = torch.empty((n + k) * g * rec + k * g * gs * gs + k, dtype=torch.float32, device=dev)
        ws = nv.grow_workspace(dev, lib.dwt_latent_workspace_bytes(n, c, hw, gs, k))
        rm, rv = (nv.ptr(rm_t), nv.ptr(rv_t)) if need_running else (None, None)
        with torch.cuda.device(dev):
            rc = lib.dwt_whiten_latent_fwd(nv.ptr(x), nv.ptr(y), n, c, hw, gs, k, flags, eps, momentum, int(update_running),
                                           rm, rv, nv.ptr(w_c), nv.ptr(save_mean), nv.ptr(save_w), nv.ptr(save_stats),
                                           nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        nv.poll_status(dev)
        if update_running and mode == nv.MODE_TRAIN:
            _bump_versions([running])
        ctx.save_for_backward(x, w_c, save_mean, save_w, save_stats)
        ctx.cfg = (gs, flags, eps, n, c, hw, k, fmt)
        return y

    @staticmethod
    def backward(ctx, dout):
        lib = nv.lib()
        x, w_c, save_mean, save_w, save_stats = ctx.saved_tensors
        gs, flags, eps, n, c, hw, k, fmt = ctx.cfg
        dout, _ = _prepare_dout(ctx, dout, x, fmt, 16)
        dev = nv.require_cuda(dout, bf16=True)
        dx = torch.empty_like(x)
        dw = torch.empty(n, k, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        ws = nv.grow_workspace(dev, lib.dwt_latent_workspace_bytes(n, c, hw, gs, k))
        with torch.cuda.device(dev):
            rc = lib.dwt_whiten_latent_bwd(nv.ptr(x), nv.ptr(dout), nv.ptr(dx), n, c, hw, gs, k, flags, eps, nv.ptr(w_c),
                                           nv.ptr(save_mean), nv.ptr(save_w), nv.ptr(save_stats), nv.ptr(dw), nv.ptr(ws),
                                           ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        return dx, dw, None, None, None, None, None, None


def latent_domain_whiten(x, weights, *, group_size, training_stats, eps, momentum, update_running, running, weight=None,
                         bias=None, relu=False, residual=None):
    """Latent-domain whitening of x [N, C, *] under per-image domain weights [N, D] (used as given: no softmax, no value
    checks; cast to float32).  Per group of group_size channels, with each image's own mean and (biased) covariance
    m_n, C_n and s_d = sum_n w_nd:
        mu_d = sum_n w_nd m_n / s_d,  Sigma_d = sum_n w_nd [C_n + (m_n - mu_d)(m_n - mu_d)^T] / s_d
        (training_stats=False: the running buffers),  W_d = inverse(cholesky((1 - eps) Sigma_d + eps I)),
        y_n = sum_d w_nd W_d (x_n - mu_d).
    A domain whose weights sum to exactly 0 is skipped (its weights get gradient 0).  running = (mean [D, C], second
    moment [D, C/gs, gs, gs]): read when training_stats is False; updated with (mu_d, Sigma_d) by momentum when
    training_stats and update_running.  weights gets its gradient.
    Group sizes up to 4 run the register-resident kernels (dwt_whiten_latent_small_*; group sizes 1, 2, 4, any H*W):
    a channels-last x whose C is not a multiple of 4 runs as an NCHW copy, and a bfloat16 NCHW x whose H*W is not a
    multiple of 4 runs the float32 kernels on an upcast copy, the result in bfloat16.  Larger group sizes run the
    tensor-core kernels (group sizes 8, 16, 32, 64, H*W >= 256; dwt_whiten_latent_*): a bfloat16 NCHW x whose H*W is not
    a multiple of 8 (the bf16 kernels' TMA rows) runs them in float32 on an upcast copy, the result in bfloat16.  D <= 8
    either way; a call the kernels cannot take raises NativeError with the library's reason and is never sent to another
    kernel family."""
    what = "latent-domain whitening"
    if x.dim() < 3:
        raise ValueError(f"{what} expects [N, C, *] input (got {x.dim()}D input)")
    _check_weights(what, x, weights)
    _check_site(what, x, weight, bias, relu, residual)
    nv.require_cuda(x, bf16=True)
    mode = nv.MODE_TRAIN if training_stats else nv.MODE_EVAL
    args = (int(group_size), mode, float(eps), float(momentum), bool(update_running), tuple(running))
    if int(group_size) > 4:
        y = _apply_per_image(_LatentFunction, x, weights.float(), *args)
        if weight is None:
            return y
        # no fused epilogue on the tensor-core kernels: the site as tensor ops (DomainTripleNorm's rule there)
        shape = (1, -1) + (1,) * (x.dim() - 2)
        y = y * weight.view(shape) + bias.view(shape)
        return torch.relu(y + residual if residual is not None else y) if relu else y
    return _LatentBandwidthFunction.apply(*_bandwidth_ready(x, residual), weights.float(), weight, bias, nv.KIND_WHITEN,
                                          *args, bool(relu)).to(x.dtype)


def latent_domain_batch_norm(x, weights, weight, bias, *, training_stats, eps, momentum, update_running, running,
                             relu=False, residual=None):
    """Latent-domain batch norm of x [N, C, *] under per-image domain weights [N, D] (used as given: no softmax, no value
    checks; cast to float32).  Per channel, with each image's own mean and (biased) variance m_n, v_n and s_d = sum_n w_nd:
        mu_d = sum_n w_nd m_n / s_d,  sigma2_d = sum_n w_nd [v_n + (m_n - mu_d)^2] / s_d  (training_stats=False: the
        running buffers),  y_n = weight * sum_d w_nd (x_n - mu_d) / sqrt(sigma2_d + eps) + bias.
    weight / bias: [C]-sized or both None.  A domain whose weights sum to exactly 0 is skipped (its weights get gradient
    0).  running = (mean [D, C], var [D, C]): read when training_stats is False; updated with (mu_d, the unbiased sigma2_d)
    by momentum when training_stats and update_running.  x, weights, weight and bias get their gradients.
    The latent-domain batch-norm kernels (dwt_bn_latent_*; dwt_b200.h) take every shape.  A channels-last x whose C is not
    a multiple of 4 runs as an NCHW copy; a bfloat16 NCHW x whose H*W is not a multiple of 4 runs the float32 kernels on
    an upcast copy, the result in bfloat16.
    relu, residual (x's shape; needs relu and weight / bias): the norm site relu(y [+ residual]) in the same kernels
    (dwt_latent_site_*: ReLU and residual in registers, the ReLU mask recomputed or saved as one byte per 4 values)."""
    what = "latent-domain batch norm"
    if x.dim() < 2:
        raise ValueError(f"{what} expects [N, C, *] input (got {x.dim()}D input)")
    _check_weights(what, x, weights)
    _check_site(what, x, weight, bias, relu, residual)
    nv.require_cuda(x, bf16=True)
    mode = nv.MODE_TRAIN if training_stats else nv.MODE_EVAL
    args = (mode, float(eps), float(momentum), bool(update_running), tuple(running))
    return _LatentBandwidthFunction.apply(*_bandwidth_ready(x, residual), weights.float(), weight, bias, nv.KIND_BN, 1,
                                          *args, bool(relu)).to(x.dtype)


def _bandwidth_ready(x, residual=None):
    """-> (x, memory format, residual) as the latent-domain bandwidth passes take them: channels-last when x is and C % 4
    == 0, else NCHW-contiguous; a bfloat16 NCHW x whose H*W is not a multiple of 4 upcast to float32; data_ptr() 16-byte
    (bf16: 8-byte) aligned.  The residual gets x's dtype and layout."""
    fmt = torch.channels_last if _channels_last(x) and x.shape[1] % 4 == 0 else torch.contiguous_format
    xk = x
    if x.dtype == torch.bfloat16 and fmt == torch.contiguous_format and math.prod(x.shape[2:]) % 4:
        xk = x.float()
    align = 8 if xk.dtype == torch.bfloat16 else 16
    out = []
    for t in (xk, residual):
        if t is not None:
            t = t.to(xk.dtype).contiguous(memory_format=fmt)
            if t.data_ptr() % align:
                t = t.clone(memory_format=fmt)
        out.append(t)
    return out[0], fmt, out[1]


def _check_weights(what, x, weights):
    """A latent-domain layer's per-image domain weights: [N, n_domains], floating point, on x's device."""
    if weights.dim() != 2 or weights.shape[0] != x.shape[0]:
        raise ValueError(f"{what} expects weights of shape [N, n_domains] with N = {x.shape[0]} "
                         f"(got {list(weights.shape)})")
    if not weights.is_floating_point():
        raise TypeError(f"{what} expects floating-point weights (got {weights.dtype})")
    if weights.device != x.device:
        raise ValueError(f"{what} expects weights on x's device {x.device} (got {weights.device})")


def _check_site(what, x, weight, bias, relu, residual):
    """A latent-domain layer's site arguments: weight / bias together, relu and the residual only with them."""
    if (weight is None) != (bias is None):
        raise ValueError(f"{what} takes weight and bias together, or neither")
    if (relu or residual is not None) and weight is None:
        raise ValueError(f"{what}: a fused ReLU or residual needs weight and bias")
    if residual is not None:
        if not relu:
            raise ValueError(f"{what}: a fused residual needs relu=True (the site is relu(weight * y + bias + residual))")
        if residual.shape != x.shape or residual.device != x.device:
            raise ValueError(f"{what}: the residual must be shaped like x and on its device (got {list(residual.shape)})")


class _LatentBandwidthFunction(torch.autograd.Function):
    """Latent-domain batch norm (kind nv.KIND_BN) or small-group whitening (nv.KIND_WHITEN, group sizes 1, 2, 4) of x
    under weights on the bandwidth kernels (dwt_latent_site_fwd / _bwd), with the site out = relu(gamma * zhat + beta
    [+ residual]) in the same kernels.  gamma / beta are [C]-sized or both None (no epilogue: the layer alone); relu and
    the residual need them.  x and the residual as _bandwidth_ready leaves them.  Running buffers: (mean [D, C], var
    [D, C] or second moment [D, C/gs, gs, gs]).  Gradients of x, weights, gamma, beta and the residual.
    A channels-last residual saves the kernels' ReLU byte map; an NCHW one saves the output and forms dz = dout * (out >
    0) with one ATen pass (_NormFunction's rule)."""

    @staticmethod
    def forward(ctx, x, fmt, residual, weights, gamma, beta, kind, group_size, mode, eps, momentum, update_running,
                running, relu):
        dev = nv.require_cuda(x, residual, bf16=True)
        rm_t, rv_t = running
        nv.require_cuda(weights, gamma, beta, rm_t, rv_t)
        lib = nv.lib()
        gs = group_size
        n, c, hw = x.shape[0], x.shape[1], math.prod(x.shape[2:])
        k = weights.shape[1]
        w_c = _aligned(weights)
        need_running = (mode == nv.MODE_EVAL) or update_running
        if need_running:
            _check_param("running mean", rm_t, k * c)
            _check_param("running var" if kind == nv.KIND_BN else "running second moment", rv_t, k * c * gs)
        _check_param("gamma / weight", gamma, c)
        _check_param("beta / bias", beta, c)
        gamma_c, beta_c = ((None, None) if gamma is None
                           else (gamma.detach().reshape(-1).contiguous(), beta.detach().reshape(-1).contiguous()))
        nhwc = fmt == torch.channels_last
        epi = ((nv.EPI_AFFINE if gamma is not None else 0) | (nv.EPI_RELU if relu else 0)
               | (nv.EPI_RESIDUAL if residual is not None else 0))
        flags = mode | (nv.LAYOUT_NHWC if nhwc else 0) | (nv.DTYPE_BF16 if x.dtype == torch.bfloat16 else 0)
        y = torch.empty_like(x)
        mask = torch.empty(x.numel() // 4, dtype=torch.uint8, device=dev) if (residual is not None and nhwc) else None
        if kind == nv.KIND_BN:
            save_mean = save_w = None
            save = torch.empty((4 * n + 3 * k) * c, dtype=torch.float32, device=dev)
            ws_bytes = lib.dwt_bn_latent_workspace_bytes(n, c, hw, k)
        else:
            g = c // gs
            save_mean = torch.empty(n, c, dtype=torch.float32, device=dev)
            save_w = torch.empty(n, g, gs, gs, dtype=torch.float32, device=dev)
            save = torch.empty((n + k) * g * (gs * gs + gs) + k * g * gs * gs + k, dtype=torch.float32, device=dev)
            ws_bytes = lib.dwt_latent_small_workspace_bytes(n, c, hw, gs, k)
        ws = nv.grow_workspace(dev, ws_bytes)
        rm, rv = (nv.ptr(rm_t), nv.ptr(rv_t)) if need_running else (None, None)
        with torch.cuda.device(dev):
            rc = lib.dwt_latent_site_fwd(kind, nv.ptr(x), nv.ptr(y), n, c, hw, gs, k, flags, eps, momentum,
                                         int(update_running), rm, rv, nv.ptr(w_c), nv.ptr(gamma_c), nv.ptr(beta_c),
                                         nv.ptr(residual), nv.ptr(mask), epi, nv.ptr(save_mean), nv.ptr(save_w),
                                         nv.ptr(save), nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        nv.poll_status(dev)
        if update_running and mode == nv.MODE_TRAIN:
            _bump_versions([running])
        ctx.residual_mode = None
        extra = None
        if mask is not None:
            ctx.residual_mode, extra = "mask", mask
        elif residual is not None:
            ctx.residual_mode, extra, epi = "aten", y, nv.EPI_AFFINE
        ctx.save_for_backward(x, w_c, gamma_c, beta_c, save_mean, save_w, save, extra)
        ctx.cfg = (kind, gs, flags, eps, epi, n, c, hw, k, fmt, None if gamma is None else (gamma.shape, beta.shape))
        return y

    @staticmethod
    def backward(ctx, dout):
        lib = nv.lib()
        x, w_c, gamma_c, beta_c, save_mean, save_w, save, extra = ctx.saved_tensors
        kind, gs, flags, eps, epi, n, c, hw, k, fmt, shapes = ctx.cfg
        if ctx.residual_mode == "aten":
            dout2 = ctx.__dict__.pop("_dwt_extra_grad", None)
            if dout2 is not None:
                dout = dout + dout2
            dout = torch.ops.aten.threshold_backward(dout, extra, 0)
        dout, _ = _prepare_dout(ctx, dout, x, fmt, 8 if x.dtype == torch.bfloat16 else 16)
        dev = nv.require_cuda(dout, bf16=True)
        dx = torch.empty_like(x)
        dw = torch.empty(n, k, dtype=torch.float32, device=dev) if ctx.needs_input_grad[3] else None
        want_affine = ctx.needs_input_grad[4] or ctx.needs_input_grad[5]
        dgamma = torch.empty(c, dtype=torch.float32, device=dev) if want_affine else None
        dbeta = torch.empty(c, dtype=torch.float32, device=dev) if want_affine else None
        mask = d_res = None
        if ctx.residual_mode == "mask":
            mask, d_res = extra, torch.empty_like(x)     # dz, written even when the residual needs no gradient
        elif ctx.residual_mode == "aten":
            d_res = dout
        ws_bytes = (lib.dwt_bn_latent_workspace_bytes(n, c, hw, k) if kind == nv.KIND_BN
                    else lib.dwt_latent_small_workspace_bytes(n, c, hw, gs, k))
        ws = nv.grow_workspace(dev, ws_bytes)
        with torch.cuda.device(dev):
            rc = lib.dwt_latent_site_bwd(kind, nv.ptr(x), nv.ptr(dout), nv.ptr(dx), n, c, hw, gs, k, flags, eps,
                                         nv.ptr(w_c), nv.ptr(gamma_c), nv.ptr(beta_c), nv.ptr(mask),
                                         nv.ptr(d_res) if mask is not None else None, epi, nv.ptr(save_mean),
                                         nv.ptr(save_w), nv.ptr(save), nv.ptr(dw), nv.ptr(dgamma), nv.ptr(dbeta),
                                         nv.ptr(ws), ws.numel(), nv.stream_ptr(dev))
        nv.check(rc)
        if want_affine:
            dgamma, dbeta = dgamma.view(shapes[0]), dbeta.view(shapes[1])
        return (dx, None, d_res if ctx.needs_input_grad[2] else None, dw, dgamma, dbeta) + (None,) * 8


class _MecFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y):
        lib = nv.lib()
        if x.dim() != 2 or x.shape != y.shape:
            raise ValueError(f"expected two [N, K] logit tensors, got {tuple(x.shape)} and {tuple(y.shape)}")
        x, y = x.contiguous(), y.contiguous()
        dev = nv.require_cuda(x, y)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        gx, gy = torch.empty_like(x), torch.empty_like(y)
        with torch.cuda.device(dev):
            rc = lib.dwt_mec_fwd_bwd(nv.ptr(x), nv.ptr(y), x.shape[0], x.shape[1], nv.ptr(loss), nv.ptr(gx),
                                     nv.ptr(gy), nv.stream_ptr(dev))
        nv.check(rc)
        ctx.save_for_backward(gx, gy)
        return loss

    @staticmethod
    def backward(ctx, g):
        gx, gy = ctx.saved_tensors
        return g * gx, g * gy


def _upcast_logits(t):
    """bf16 logits (a Linear head under autocast) are [3B, K]: the losses upcast them, their gradient flows back as bf16."""
    return t.float() if t.dtype == torch.bfloat16 else t


def mec_loss(x, y):
    return _MecFunction.apply(_upcast_logits(x), _upcast_logits(y))


class _HeadLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, lam):
        lib = nv.lib()
        if logits.dim() != 2 or logits.shape[0] % 3 != 0 or labels.dim() != 1 or labels.shape[0] * 3 != logits.shape[0]:
            raise ValueError(f"expected logits [3B, K] and labels [B], got {tuple(logits.shape)} and {tuple(labels.shape)}")
        logits = logits.contiguous()
        dev = nv.require_cuda(logits)
        if not labels.is_cuda or labels.dtype != torch.int64:
            raise nv.NativeError("labels must be an int64 CUDA tensor")
        labels = labels.contiguous()
        losses = torch.empty(3, dtype=torch.float32, device=dev)
        grad = torch.empty_like(logits)
        with torch.cuda.device(dev):
            rc = lib.dwt_head_loss_fwd_bwd(nv.ptr(logits), nv.ptr(labels), labels.shape[0], logits.shape[1], float(lam),
                                           nv.ptr(losses), nv.ptr(grad), nv.status_ptr(dev), nv.stream_ptr(dev))
        nv.check(rc)
        nv.poll_status(dev)
        ctx.save_for_backward(grad)
        ctx.mark_non_differentiable(losses)
        return losses[0], losses

    @staticmethod
    def backward(ctx, g, _unused):
        (grad,) = ctx.saved_tensors
        return g * grad, None, None


def head_loss(logits, labels, lambda_mec):
    """-> (total loss (differentiable), tensor [total, classification, lambda*MEC])."""
    return _HeadLossFunction.apply(_upcast_logits(logits), labels, lambda_mec)
