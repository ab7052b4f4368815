"""ctypes binding of libdwt_b200.so (include/dwt_b200.h) -- the only way the Python layers
reach the GPU.  There is no CPU path: if the library is missing or the tensors are not on a
CUDA device the call fails loudly.
"""
from __future__ import annotations

import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# DWT_B200_LIB: another build of the same library (development: A/B timing of a kernel variant on one box)
LIB_PATH = os.environ.get("DWT_B200_LIB") or os.path.join(_HERE, "lib", "libdwt_b200.so")

ABI_VERSION = 10
MAX_DOMAINS = 4
MAX_GROUP_SIZE = 64
TC_MAX_GROUP_SIZE = 128            # the one wider group size: fp32 whitening on the tensor-core kernels only
MODE_TRAIN, MODE_EVAL = 0, 1
EPI_NONE, EPI_AFFINE, EPI_RELU, EPI_RESIDUAL = 0, 1, 2, 4
LAYOUT_NHWC = 0x100
DTYPE_BF16 = 0x200                 # bf16 activations (gs 1/2/4 and BN channels-last or NCHW, tensor-core gs 8..64; dwt_b200.h)
STATUS_NOT_PD, STATUS_BAD_LABEL = 1, 2
ZCA_MAX_ITERATIONS = 16            # Newton-Schulz iterations of the ZCA basis (dwt_whiten_zca_*): 1..16
EIGH = "eigh"                      # the exact ZCA basis (dwt_whiten_eigh_*) where a number of iterations goes
COLOR = "color"                    # the Cholesky basis coloured (dwt_whiten_color_*): functional._NormFunction's basis
KIND_WHITEN, KIND_BN = 0, 1

_c_float_p = ctypes.c_void_p
_PtrArray = ctypes.c_void_p * MAX_DOMAINS


class TailSite(ctypes.Structure):
    """dwt_tail_site: one of the two norm sites of dwt_tail2_fwd / dwt_tail2_bwd."""
    _fields_ = [("x", ctypes.c_void_p), ("eps", ctypes.c_float), ("momentum", ctypes.c_float),
                ("update_running", ctypes.c_int), ("running_mean", ctypes.POINTER(ctypes.c_void_p)),
                ("running_cov", ctypes.POINTER(ctypes.c_void_p)), ("gamma", ctypes.c_void_p), ("beta", ctypes.c_void_p),
                ("save_mean", ctypes.c_void_p), ("save_w", ctypes.c_void_p), ("dx", ctypes.c_void_p),
                ("dgamma", ctypes.c_void_p), ("dbeta", ctypes.c_void_p)]

_SIGNATURES = {
    "dwt_abi_version": (ctypes.c_int, []),
    "dwt_last_error": (ctypes.c_char_p, []),
    "dwt_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "dwt_whiten_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                      ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                      ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p),
                                      _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_int, _c_float_p,
                                      _c_float_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_whiten_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                      ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                      _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, _c_float_p,
                                      ctypes.c_int, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_size_t,
                                      ctypes.c_void_p]),
    "dwt_whiten_zca_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                          ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                          ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p),
                                          ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                          ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_whiten_zca_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                          ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                          ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                          ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_whiten_eigh_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                           ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                           ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p),
                                           _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_size_t,
                                           ctypes.c_void_p]),
    "dwt_whiten_eigh_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                           ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                           _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_size_t,
                                           ctypes.c_void_p]),
    "dwt_whiten_color_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                            ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                            ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p),
                                            _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_size_t,
                                            ctypes.c_void_p]),
    "dwt_whiten_color_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                            ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                            _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                            ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_instance_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int]),
    "dwt_whiten_instance_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                               ctypes.c_int, ctypes.c_int, ctypes.c_float, _c_float_p, _c_float_p,
                                               ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_whiten_instance_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                               ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_float, _c_float_p,
                                               _c_float_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_switch_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int]),
    "dwt_whiten_switch_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                             ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int,
                                             _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                             ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_whiten_switch_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                             ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_float, _c_float_p,
                                             _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                             ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_latent_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "dwt_whiten_latent_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                             ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                             ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                             _c_float_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_whiten_latent_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                             ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                             _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                             ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_latent_small_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int,
                                                           ctypes.c_int]),
    "dwt_whiten_latent_small_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                                   ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                                   ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                   _c_float_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_whiten_latent_small_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                                   ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                                   _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                                   ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_bn_latent_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int]),
    "dwt_bn_latent_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, _c_float_p, _c_float_p,
                                         _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_size_t,
                                         ctypes.c_void_p]),
    "dwt_bn_latent_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                         ctypes.c_int, ctypes.c_int, ctypes.c_float, _c_float_p, _c_float_p, _c_float_p,
                                         _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_size_t,
                                         ctypes.c_void_p]),
    "dwt_latent_site_fwd": (ctypes.c_int, [ctypes.c_int, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                           ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                           ctypes.c_float, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                           _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_int, _c_float_p, _c_float_p,
                                           _c_float_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_latent_site_bwd": (ctypes.c_int, [ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64,
                                           ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                           _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p, _c_float_p, ctypes.c_int,
                                           _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                           ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_bn_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                  ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int,
                                  ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p), _c_float_p,
                                  _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_int, _c_float_p, _c_float_p,
                                  ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_bn_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                  ctypes.c_int, ctypes.c_int, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                  ctypes.c_void_p, _c_float_p, ctypes.c_int, _c_float_p, _c_float_p, ctypes.c_void_p,
                                  ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_tail2_fwd": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(TailSite), _c_float_p, ctypes.c_void_p, ctypes.c_int64,
                                     ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_tail2_bwd": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(TailSite), _c_float_p, _c_float_p, ctypes.c_void_p,
                                     _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "dwt_mec_fwd_bwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, _c_float_p,
                                       _c_float_p, _c_float_p, ctypes.c_void_p]),
    "dwt_head_loss_fwd_bwd": (ctypes.c_int, [_c_float_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_float,
                                             _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_void_p]),
    "dwt_augment_pair": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, _c_float_p,
                                        ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), _c_float_p,
                                        _c_float_p, ctypes.c_int, ctypes.c_void_p]),
    "dwt_maxpool_fwd": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                       ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "dwt_maxpool_bwd": (ctypes.c_int, [_c_float_p, ctypes.c_void_p, _c_float_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                       ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "dwt_launch_count": (ctypes.c_int64, []),
    "dwt_profile_begin": (None, []),
    "dwt_profile_end": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
}


class ProfileEntry(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 48), ("launches", ctypes.c_int64), ("ms", ctypes.c_double),
                ("bytes", ctypes.c_double)]


def profile_begin():
    lib().dwt_profile_begin()


def profile_end():
    """-> {"family|C|HW|GS|D|N": dict(launches, ms, bytes)}; waits for the recorded events."""
    cap = 1024
    buf = (ProfileEntry * cap)()
    k = lib().dwt_profile_end(ctypes.cast(buf, ctypes.c_void_p), cap)
    return {buf[i].name.decode(): dict(launches=buf[i].launches, ms=buf[i].ms, bytes=buf[i].bytes) for i in range(k)}


def by_family(prof):
    """Collapse profile_end() output over geometries: {family: dict(launches, ms, bytes)}."""
    out = {}
    for name, v in prof.items():
        f = out.setdefault(name.split("|")[0], dict(launches=0, ms=0.0, bytes=0.0))
        for k in f:
            f[k] += v[k]
    return out


def launch_count() -> int:
    return int(lib().dwt_launch_count())
EXPORTS = tuple(_SIGNATURES)

_lib = None
_lock = threading.Lock()


class NativeError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load (once) and return the shared library; raise if it has not been built."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise NativeError(
                        f"{LIB_PATH} is missing: build it with `python {os.path.join(_HERE, 'build.py')}` "
                        "(dwt_b200 has no CPU or PyTorch fallback)")
                handle = ctypes.CDLL(LIB_PATH)
                for name, (res, args) in _SIGNATURES.items():
                    fn = getattr(handle, name)
                    fn.restype, fn.argtypes = res, args
                if handle.dwt_abi_version() != ABI_VERSION:
                    raise NativeError("libdwt_b200.so ABI version mismatch; rebuild it")
                _lib = handle
    return _lib


def channels_last_supported(channels: int, group_size: int) -> bool:
    """Mirror of cl_supports() in csrc/norm_cl.cu: group sizes 1/2/4 with C a multiple of 4 and C/4 at most 16384."""
    if group_size not in (1, 2, 4) or channels % 4:
        return False
    return 0 < channels // 4 <= 16384


def small_bf16_supported(hw: int, group_size: int) -> bool:
    """Mirror of the C ABI's bf16 rule for the NCHW register-resident kernels (csrc/api.cu, route(): the SMALL family):
    whitening at group sizes 1, 2, 4 and batch norm (group_size 1) take bf16 activations when HW is a multiple of 4 (a
    thread reads four pixels of a channel row as 8 bytes).  The tensors also need an 8-byte-aligned data_ptr()."""
    return group_size in (1, 2, 4) and hw % 4 == 0


def tensor_core_bf16_supported(n: int, channels: int, hw: int, group_size: int) -> bool:
    """Mirror of the C ABI's bf16 NCHW rule (csrc/api.cu, route(): the TC family, over tc_supports in
    csrc/norm_tc.cu): the
    tensor-core whitening kernels take bf16 activations for group sizes 8..64 dividing 64, HW >= 32 and a multiple of 8
    (16-byte TMA rows), and at least 4096 samples per domain (n = images per domain).  The tensors also need a
    16-byte-aligned data_ptr()."""
    return (group_size in (8, 16, 32, 64) and channels % group_size == 0 and hw >= 32 and hw % 8 == 0
            and n * hw >= 4096)


def tensor_core_nhwc_supported(n: int, channels: int, hw: int, group_size: int) -> bool:
    """Mirror of the C ABI's channels-last tensor-core rule (csrc/api.cu, route(): the TC family): whitening at group sizes
    8..64 dividing 64, and 128, runs on channels-last tensors when HW >= 32 and a multiple of 4 and there are at least
    4096 samples per domain (n = images per domain); fp32 and bf16 alike up to 64, fp32 only at 128 (bf16 upcasts).
    The tensors also need a 16-byte-aligned data_ptr()."""
    return (group_size in (8, 16, 32, 64, TC_MAX_GROUP_SIZE) and channels % group_size == 0 and hw >= 32 and hw % 4 == 0
            and n * hw >= 4096)


def check(rc: int) -> None:
    if rc != 0:
        raise NativeError(f"libdwt_b200 error {rc}: {lib().dwt_last_error().decode()}")


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def ptr_array(tensors):
    arr = _PtrArray()
    for i, t in enumerate(tensors):
        arr[i] = None if t is None else t.data_ptr()
    return ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p))


def require_cuda(*tensors, any_dtype=False, bf16=False) -> torch.device:
    """Device of the tensors (all CUDA, all on one device).  They must be float32 unless any_dtype; bf16=True also
    admits bfloat16 (activations: statistics, parameters and running buffers are always float32)."""
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise NativeError("dwt_b200 runs on CUDA tensors only (no CPU fallback); got a tensor on " + str(t.device))
        if t.dtype != torch.float32 and not any_dtype and not (bf16 and t.dtype == torch.bfloat16):
            raise NativeError("dwt_b200 computes in float32 (activations may also be bfloat16); got " + str(t.dtype))
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise NativeError(f"tensors on different devices: {dev} vs {t.device}")
    return dev


def stream_ptr(device) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


# One zero-initialised, grow-only workspace per (device, stream): kernels of one stream run in
# order, so they can share it; the arrival counters inside reset themselves.
_workspaces: dict = {}


def workspace(device, n, c, hw, gs, nd):
    if gs == TC_MAX_GROUP_SIZE and c % gs == 0:
        c, gs = 2 * c, MAX_GROUP_SIZE                # dwt_b200.h: the group-size-64 query on 2C channels covers it
    need = lib().dwt_workspace_bytes(n, c, hw, gs, nd)
    if need == 0:
        raise NativeError(f"invalid geometry for workspace: C={c} group_size={gs} domains={nd}")
    return grow_workspace(device, need)


def grow_workspace(device, nbytes):
    """The current stream's workspace, grown to at least nbytes (a new buffer has at least 8 MiB).  The per-image entry
    points size theirs by dwt_instance_workspace_bytes / dwt_switch_workspace_bytes / dwt_latent_workspace_bytes, and
    latent-domain batch norm by dwt_bn_latent_workspace_bytes, which give 0 for a geometry they refuse (the call then
    reports why)."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _workspaces.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.zeros(max(nbytes, 8 << 20), dtype=torch.uint8, device=device)
        _workspaces[key] = buf
    return buf


def status(device=None) -> int:
    """Device status word of the current stream's workspace (syncs).  Bit 0 (STATUS_NOT_PD): a covariance was
    not positive definite (the reference raises from torch.cholesky at that point); bit 1 (STATUS_BAD_LABEL): the
    head loss met a label outside [0, K) other than -100 (F.nll_loss device-asserts)."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    buf = _workspaces.get((device.index, torch.cuda.current_stream(device).cuda_stream))
    return 0 if buf is None else int(buf[:4].view(torch.int32).item())


def status_all(device=None) -> int:
    """OR of the status words of every stream's workspace on the device (syncs): CUDA-graph capture runs on its own
    stream and therefore on its own workspace."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    torch.cuda.synchronize(device)
    st = 0
    for (idx, _), buf in _workspaces.items():
        if idx == device.index:
            st |= int(buf[:4].view(torch.int32).item())
    return st


def status_ptr(device):
    """Device address of the current stream's status word (the head-loss kernel ORs its bit in there)."""
    return ctypes.c_void_p(workspace(device, 1, 4, 1, 1, 1).data_ptr())


def clear_status(device=None) -> None:
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    buf = _workspaces.get((device.index, torch.cuda.current_stream(device).cuda_stream))
    if buf is not None:
        buf[:4].zero_()


class NotPositiveDefiniteError(torch.linalg.LinAlgError):
    """What the reference's torch.cholesky raises at utils/whitening.py:53, raised late: the kernels never sync the
    host, so the failure is seen at the next poll (raise_on_status) or explicit check_status() call."""


_poll = {"every": 0, "count": 0}


def raise_on_status(every: int = 1) -> None:
    """Opt-in failure surfacing: every `every`-th layer call (forward of a whitening / BN / fused-site / head-loss
    layer) reads the status word -- one 4-byte device->host copy, i.e. a host sync -- and raises.  every=0 turns the
    polling off again (the default: the hot path never syncs).  Not for use while capturing a CUDA graph."""
    _poll["every"], _poll["count"] = max(0, int(every)), 0


def check_status(device=None) -> None:
    """Read the status word now (syncs) and raise if a kernel reported a failure; clears the word."""
    st = status(device)
    if st == 0:
        return
    clear_status(device)
    if st & STATUS_NOT_PD:
        raise NotPositiveDefiniteError(
            "cholesky: a whitening covariance was not positive definite (status word bit 0; the reference raises "
            "from torch.cholesky, utils/whitening.py:53); the affected group's output is NaN and its running-"
            "statistics update was skipped")
    if st & STATUS_BAD_LABEL:
        raise IndexError("head loss: a label was outside [0, num_classes) and is not ignore_index=-100 "
                         "(F.nll_loss asserts here); the row was dropped")
    raise NativeError(f"unknown status bits {st:#x}")


def poll_status(device) -> None:
    if _poll["every"]:
        _poll["count"] += 1
        if _poll["count"] >= _poll["every"]:
            _poll["count"] = 0
            check_status(device)
