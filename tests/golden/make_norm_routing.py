"""The argument-validation table of the norm entry points of the C ABI, and its fixture.

    python tests/golden/make_norm_routing.py      # builds the library if needed, writes tests/golden/norm_routing.json

Every case calls dwt_whiten_fwd/bwd, dwt_bn_fwd/bwd or dwt_tail2_fwd/bwd with fake device pointers and (but for the
misaligned-workspace cases) workspace_bytes = 1: a call that passes every argument check stops at DWT_E_WORKSPACE
("need N bytes"), any other at its refusal, and none reaches device memory, so the table runs without a GPU.  The
fixture records (return code, dwt_last_error text) of every case; the byte count of a "need N bytes" text depends on
the SM count and is masked.  tests/test_norm_routing.py checks the library against it.
"""
from __future__ import annotations

import ctypes
import hashlib
import itertools
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
FIXTURE = os.path.join(HERE, "norm_routing.json")

NHWC, BF16 = 0x100, 0x200
TRAIN, EVAL = 0, 1
AFFINE, RELU, RESIDUAL = 1, 2, 4
HUGE = 1 << 40                     # workspace_bytes of the misaligned-workspace cases: the size check passes

# group sizes and geometries (N per domain, C, HW, D) at every family edge
GROUP_SIZES = (1, 2, 3, 4, 8, 16, 32, 64, 96, 128)
GEOMETRIES = (
    (8, 384, 1024, 3),             # C divisible by every group size above, tensor-core geometry, C/4 not a power of two
    (8, 256, 1024, 2),             # C/4 a power of two
    (16, 320, 256, 1),             # C % 3, C % 96, C % 128 != 0
    (16, 66, 256, 3),              # C % 4 != 0
    (1, 65664, 4096, 1),           # C/4 > 16384 (and C/gs > 65535 at group size 1)
    (512, 384, 16, 3),             # HW < 32
    (8, 384, 1026, 3),             # HW % 4 != 0
    (8, 384, 1028, 3),             # HW % 8 != 0
    (3, 384, 1024, 3),             # N*HW < 4096 per domain
    (8, 384, 1024, 0),             # D outside 1..4
    (8, 384, 1024, 5),
    (0, 384, 1024, 3),             # empty tensor
)

# default pointers: fake, distinct, 256-byte aligned; the optional ones start absent
_ADDR = {name: (1 << 32) + k * (1 << 24) for k, name in enumerate((
    "x", "y", "dout", "dout2", "dx", "gamma", "beta", "residual", "relu_mask", "dresidual", "save_mean", "save_w",
    "dgamma", "dbeta", "ws", "rmean", "rcov", "dz",
    "s0.x", "s0.gamma", "s0.beta", "s0.save_mean", "s0.save_w", "s0.dx", "s0.dgamma", "s0.dbeta", "s0.rmean", "s0.rcov",
    "s1.x", "s1.gamma", "s1.beta", "s1.save_mean", "s1.save_w", "s1.dx", "s1.dgamma", "s1.dbeta", "s1.rmean", "s1.rcov"))}
_ABSENT = {"residual", "relu_mask", "dout2", "dresidual"}


def case(op, N, C, HW, gs, D, flags, mode=TRAIN, epi=0, upd=0, ws_bytes=1, **ptrs):
    """One call.  ptrs: name=None (null), name=k (the default address + k bytes; 0 makes an absent pointer present);
    rmean / rcov (and s0.rmean, ...) are host arrays of D device pointers: None (no array) or "hole" (entry 1 null).
    flags: layout | dtype of whiten / bn, DWT_DTYPE_BF16 | kind of the tail."""
    return dict(op=op, N=N, C=C, HW=HW, gs=gs, D=D, flags=flags, mode=mode, epi=epi, upd=upd, ws_bytes=ws_bytes,
                ptrs=dict(sorted(ptrs.items())))


def case_id(c):
    p = ",".join(f"{k}={v}" for k, v in c["ptrs"].items())
    return (f"{c['op']} N={c['N']} C={c['C']} HW={c['HW']} gs={c['gs']} D={c['D']} flags={c['flags']:#x} mode={c['mode']} "
            f"epi={c['epi']} upd={c['upd']} ws={c['ws_bytes']} [{p}]")


def _variations(op, base, fwd):
    """One argument at a time away from a passing base case (a dict of case() arguments)."""
    out = []

    def v(**kw):
        a = dict(base)
        a.update(kw)
        out.append(case(op, **a))

    for mode in (TRAIN, EVAL, 2):
        v(mode=mode)
    for epi in (0, 1, 2, 3, 7):
        extra = ("residual", "relu_mask") if fwd else ("relu_mask", "dresidual")
        for on in itertools.product((False, True), repeat=2):
            v(epi=epi, **{name: 0 for name, o in zip(extra, on) if o})
    acts = ("x", "y") if fwd else ("x", "dout", "dx")
    for name in acts:
        for off in (2, 4, 8):
            v(**{name: off})
    if fwd:
        for off in (2, 4, 8):
            v(epi=7, residual=off)
            v(epi=7, residual=0, relu_mask=off)
    else:
        for dout2 in (0, 4, 8):
            v(dout2=dout2)
        for off in (2, 4, 8):
            v(epi=7, relu_mask=0, dresidual=off)
    required = ("x", "y", "save_mean", "save_w", "ws") if fwd else ("x", "dout", "dx", "save_mean", "save_w", "ws")
    for name in required:
        v(**{name: None})
    v(epi=1, gamma=None)
    v(epi=1, beta=None)
    if fwd:
        v(upd=1, rmean=None)
        v(upd=1, rcov=None)
        v(upd=1, rmean="hole")
        v(mode=EVAL, rcov=None)
    else:
        v(dbeta=None)
        v(dgamma=None)
    v(ws=128, ws_bytes=HUGE)
    v(ws=None, ws_bytes=HUGE)
    return out


def _tail_variations(op, base, fwd):
    out = []

    def v(**kw):
        a = dict(base)
        a.update(kw)
        out.append(case(op, **a))

    names = ["s0.x", "s1.x", "s0.gamma", "s1.gamma", "s0.beta", "s1.beta", "s0.save_mean", "s1.save_mean", "s0.save_w",
             "s1.save_w", "relu_mask", "ws"]
    names += ["y"] if fwd else ["dout", "dz", "s0.dx", "s1.dx"]
    for name in names:
        v(**{name: None})
    for name in ["s0.x", "s1.x"] + (["y"] if fwd else ["dout", "dz", "s0.dx", "s1.dx"]):
        for off in (2, 4, 8):
            v(**{name: off})
    if fwd:
        for k in ("s0", "s1"):
            v(upd=1, **{f"{k}.rmean": None})
            v(upd=1, **{f"{k}.rcov": "hole"})
    else:
        for dout2 in (0, 4, 8):
            v(dout2=dout2)
        for k in ("s0", "s1"):
            v(**{f"{k}.dbeta": None})
    for kind in (2, 3):
        v(flags=(base["flags"] & BF16) | kind)
    v(ws=128, ws_bytes=HUGE)
    return out


def cases():
    out = []
    for layout, dtype, gs, (N, C, HW, D) in itertools.product((0, NHWC), (0, BF16), GROUP_SIZES, GEOMETRIES):
        for op in ("whiten_fwd", "whiten_bwd"):
            out.append(case(op, N, C, HW, gs, D, layout | dtype))
        if gs == 1:
            for op in ("bn_fwd", "bn_bwd"):
                out.append(case(op, N, C, HW, 1, D, layout | dtype))
        for kind in ((0, 1) if gs == 1 else (0,)) if layout == 0 else ():     # the tail has no layout argument
            for op in ("tail2_fwd", "tail2_bwd"):
                out.append(case(op, N, C, HW, gs, D, dtype | kind))
    geo = dict(N=8, C=384, HW=1024, D=3)
    bases = [(gs, flags) for flags in (0, BF16, NHWC, NHWC | BF16) for gs in (4, 3, 64, 128)]   # cl/small, tiled, tc, 128
    for gs, flags in bases:
        for fwd in (True, False):
            out += _variations("whiten_" + ("fwd" if fwd else "bwd"), dict(geo, gs=gs, flags=flags), fwd)
    for flags in (0, BF16, NHWC, NHWC | BF16):
        for fwd in (True, False):
            out += _variations("bn_" + ("fwd" if fwd else "bwd"), dict(geo, gs=1, flags=flags), fwd)
    for kind, gs, dtype in ((0, 4, 0), (0, 4, BF16), (1, 1, 0), (0, 2, BF16)):
        for fwd in (True, False):
            out += _tail_variations("tail2_" + ("fwd" if fwd else "bwd"), dict(geo, gs=gs, flags=dtype | kind), fwd)
    return list({case_id(c): c for c in out}.values())          # a variation may repeat its base case


def _lib():
    sys.path.insert(0, os.path.join(ROOT, "dwt-domain-adaptation_b200"))
    from dwt_b200 import _native as nv
    return nv, nv.lib()


def run(c, nv=None, lib=None):
    """-> (return code, dwt_last_error text with the byte count of "need N bytes" masked)."""
    if lib is None:
        nv, lib = _lib()
    P, D, keep = c["ptrs"], c["D"], []

    def ptr(name):
        if name in P:
            return None if P[name] is None else _ADDR[name] + P[name]
        return None if name in _ABSENT else _ADDR[name]

    def arr(name):
        if P.get(name, 0) is None:
            return None
        a = (ctypes.c_void_p * 4)(*[_ADDR[name] + 256 * d for d in range(4)])
        if P.get(name) == "hole":
            a[1] = None
        keep.append(a)
        return ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))

    op, N, C, HW, gs, f, mode, epi, upd, wsb = (c[k] for k in ("op", "N", "C", "HW", "gs", "flags", "mode", "epi", "upd", "ws_bytes"))
    if op == "whiten_fwd":
        rc = lib.dwt_whiten_fwd(ptr("x"), ptr("y"), N, C, HW, gs, D, mode | f, 1e-3, 0.1, upd, arr("rmean"), arr("rcov"),
                                ptr("gamma"), ptr("beta"), ptr("residual"), ptr("relu_mask"), epi, ptr("save_mean"),
                                ptr("save_w"), ptr("ws"), wsb, None)
    elif op == "bn_fwd":
        rc = lib.dwt_bn_fwd(ptr("x"), ptr("y"), N, C, HW, D, mode | f, 1e-5, 0.1, upd, arr("rmean"), arr("rcov"),
                            ptr("gamma"), ptr("beta"), ptr("residual"), ptr("relu_mask"), epi, ptr("save_mean"),
                            ptr("save_w"), ptr("ws"), wsb, None)
    elif op == "whiten_bwd":
        rc = lib.dwt_whiten_bwd(ptr("x"), ptr("dout"), ptr("dout2"), ptr("dx"), N, C, HW, gs, D, mode | f, 1e-3,
                                ptr("save_mean"), ptr("save_w"), ptr("gamma"), ptr("beta"), ptr("relu_mask"),
                                ptr("dresidual"), epi, ptr("dgamma"), ptr("dbeta"), ptr("ws"), wsb, None)
    elif op == "bn_bwd":
        rc = lib.dwt_bn_bwd(ptr("x"), ptr("dout"), ptr("dout2"), ptr("dx"), N, C, HW, D, mode | f, ptr("save_mean"),
                            ptr("save_w"), ptr("gamma"), ptr("beta"), ptr("relu_mask"), ptr("dresidual"), epi,
                            ptr("dgamma"), ptr("dbeta"), ptr("ws"), wsb, None)
    else:
        sites = (nv.TailSite * 2)()
        for k in range(2):
            s = f"s{k}."
            sites[k] = nv.TailSite(ptr(s + "x"), 1e-3, 0.1, upd, arr(s + "rmean"), arr(s + "rcov"), ptr(s + "gamma"),
                                   ptr(s + "beta"), ptr(s + "save_mean"), ptr(s + "save_w"), ptr(s + "dx"),
                                   ptr(s + "dgamma"), ptr(s + "dbeta"))
        if op == "tail2_fwd":
            rc = lib.dwt_tail2_fwd(f, sites, ptr("y"), ptr("relu_mask") if "relu_mask" in P else _ADDR["relu_mask"],
                                   N, C, HW, gs, D, ptr("ws"), wsb, None)
        else:
            rc = lib.dwt_tail2_bwd(f, sites, ptr("dout"), ptr("dout2"),
                                   ptr("relu_mask") if "relu_mask" in P else _ADDR["relu_mask"], ptr("dz"), N, C, HW,
                                   gs, D, ptr("ws"), wsb, None)
    return rc, re.sub(r"need \d+ bytes", "need N bytes", lib.dwt_last_error().decode())


def table():
    """-> (case ids, [(rc, text)]) of every case, in order."""
    nv, lib = _lib()
    cs = cases()
    return [case_id(c) for c in cs], [run(c, nv, lib) for c in cs]


def digest(ids):
    return hashlib.sha256("\n".join(ids).encode()).hexdigest()


def main():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    ids, results = table()
    assert len(set(ids)) == len(ids), "duplicate case"
    texts = sorted({t for _, t in results})
    index = {t: i for i, t in enumerate(texts)}
    doc = {"cases": len(ids), "digest": digest(ids), "texts": texts, "results": [[rc, index[t]] for rc, t in results]}
    with open(FIXTURE, "w") as fh:
        json.dump(doc, fh, separators=(",", ":"))
        fh.write("\n")
    codes = {}
    for rc, _ in results:
        codes[rc] = codes.get(rc, 0) + 1
    print(f"{FIXTURE}: {len(ids)} cases, {len(texts)} distinct texts, return codes {codes}")


if __name__ == "__main__":
    main()
