"""Channels-last norm sites at channel counts whose C/4 is not a power of two, on the channels-last kernels.

The channels-last family (norm_cl.cu) takes every C that is a multiple of 4 with C/4 <= 16384: cl_slabs() splits the
C/4 float4 columns into slabs of CW columns, cl_lane() gives each row lane LS >= CW threads (rpi = 256 / LS lanes), and
the threads left over sit the sweep out.
Compared here, with the tolerances of test_channels_last_fp64.py (whose fp64 composition, _check, runs the plain /
residual / two-site paths):

  * widths C/4 in {3, 5, 12, 24, 36, 48, 80, 100, 144, 250, 255, 257, 320, 384, 513, 1000, 16383}, group sizes 1, 2, 4
    and batch norm, epilogues none / affine / affine+relu / residual, against oracle/torch_port.py in float64 --
    output (channels-last), dx, d_identity, dgamma / dbeta, batch mean and covariance, running buffers,
    num_batches_tracked, status -- and from the launch profile: only cl_* families, x itself saved (no NCHW copy);
  * the two-site tail, row edges derived from the new rpi, eval / no-grad / replicated modes and fork_for_sum;
  * bf16 against the fp32 channels-last call on x.float(), bit for bit; the NCHW call on x.contiguous() to fp32 rounding;
  * the LeNet (conv2 site: C = 48) and a MobileNet-width DomainTripleNorm stack channels-last end to end;
  * the C ABI's return codes and workspace size; CUDA-graph replay of one site.
"""
import ctypes
import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

CL = torch.channels_last
BF = torch.bfloat16
THREADS = 256
STATS_UNROLL = 8
STATS_SLOTS = 3

_spec = importlib.util.spec_from_file_location("_cl_fp64", os.path.join(os.path.dirname(__file__), "test_channels_last_fp64.py"))
fp64 = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(fp64)

WIDTHS = [3, 5, 12, 24, 36, 48, 80, 100, 144, 250, 255, 257, 320, 384, 513, 1000, 16383]   # C/4
DEEP = {12, 36, 100, 257, 513}       # widths also swept at more rows than one chunk
KINDS = [("whiten", 1), ("whiten", 2), ("whiten", 4), ("bn", 1)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.init()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def worst(dev):
    table = {}
    yield table
    print("\nworst errors (norm-wise, max-elementwise):")
    for key in sorted(table):
        print("  %-28s %s" % (" / ".join(key), ", ".join(f"{k} {r:.1e} {m:.1e}" for k, (r, m) in sorted(table[key].items()))))


def recorded_slabs(c, dev):
    """The column-slab count (grid.y) the library launched cl_stats_kernel with at C channels, read from a recorded
    launch (torch.profiler's trace of one forward call)."""
    import json
    import tempfile

    import dwt_b200
    x = torch.randn(2, c, 2, 2, device=dev).contiguous(memory_format=CL)
    m = dwt_b200.WTransform2d(c, 1).to(dev).train()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        m(x)
        torch.cuda.synchronize(dev)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    grids = {tuple(e["args"]["grid"]) for e in events if e.get("cat") == "kernel" and "cl_stats_kernel" in e.get("name", "")}
    assert len(grids) == 1, grids
    return next(iter(grids))[1]


@pytest.fixture(scope="module")
def slab_counts(dev):
    """{C: recorded slab count} of every width this file derives launch shapes for, recorded once, up front."""
    cs = {4 * (1 << k) for k in (0, 3, 5, 8, 9, 10, 12)} | {4 * c4 for c4 in WIDTHS} | {96, 192, 576, 1280}
    cs |= {e[0] for e in EDGES}
    return {c: recorded_slabs(c, dev) for c in sorted(cs)}


def lane(c4, cw):
    """Threads per row lane of a slab cw columns wide (cl_lane in norm_cl.cu)."""
    if c4 < 8:
        return cw
    if cw <= 32:
        return max(8, 1 << (cw - 1).bit_length())
    return -(-cw // 32) * 32


def shape_of(c4, s):
    """(CW, LS, rpi, share of the CTA's threads that own a row lane and a column) with s slabs."""
    cw = -(-c4 // s)
    ls = lane(c4, cw)
    rpi = THREADS // ls
    return cw, ls, rpi, c4 * rpi / (s * THREADS)


def warp_runs(c4, s):
    """Lengths (columns) of the contiguous pieces of one row that a warp loads, over every slab."""
    cw, ls, rpi, _ = shape_of(c4, s)
    runs = []
    for slab in range(s):
        valid = min(cw, c4 - slab * cw)
        for w in range(THREADS // 32):
            pieces = {}
            for t in range(32 * w, 32 * w + 32):
                k, col = divmod(t, ls)
                if k < rpi and col < valid:
                    pieces.setdefault(k, []).append(col)
            for cols in pieces.values():
                assert cols == list(range(cols[0], cols[0] + len(cols)))
                assert c4 < 8 or cols[0] % 8 == 0
                runs.append(len(cols))
    return runs


def test_slab_shapes_of_the_library(slab_counts):
    """From recorded launches: power-of-two C/4 keeps min(C/4, 256)-column slabs; every other width has slabs of at
    least 8 columns, every warp's piece of a row is a run of >= 8 columns (128 bytes) from a multiple of 8, and most
    threads are busy.  The active fraction of each shape is printed."""
    for k in (0, 3, 5, 8, 9, 10, 12):
        c4 = 1 << k
        assert slab_counts[4 * c4] == max(1, c4 // 256)
    for c4 in WIDTHS + [96 // 4, 192 // 4, 576 // 4, 1280 // 4]:
        s = slab_counts[4 * c4]
        cw, ls, rpi, active = shape_of(c4, s)
        runs = warp_runs(c4, s)
        print(f"C/4 = {c4}: {s} slab(s) of {cw} columns, lanes of {ls} threads, rpi {rpi}, active {active:.3f}, "
              f"shortest warp run {min(runs)} columns")
        assert (s - 1) * cw < c4 and rpi >= 1
        if c4 >= 8:
            assert cw >= 8 and min(runs) >= 8, (c4, s, runs)
        assert active >= 0.74, (c4, active)


def _profiled(fn):
    from dwt_b200 import _native
    _native.profile_begin()
    try:
        out = fn()
    finally:
        fams = _native.by_family(_native.profile_end())
    return out, {k: v["launches"] for k, v in fams.items()}


def _only_cl(fams, bf16=False):
    assert fams, "no library launch recorded"
    for f in fams:
        assert f.startswith("cl_") or f == "eval_prep", fams
        assert f.endswith("_bf16") == bf16 or f == "eval_prep", fams


# --------------------------------------------------------------------------- every width, group size and epilogue
def _check_epi(dev, kind, c, gs, d, n, h, w, affine, relu, seed):
    """A site with epilogue none (affine False) or affine (relu False) against the fp64 composition."""
    from dwt_b200 import _native
    gen = torch.Generator(device=dev).manual_seed(seed)
    shape = (d * n, c, h, w)
    x = fp64._activation(gen, shape, d, dev).contiguous(memory_format=CL).requires_grad_(True)
    dy = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=CL)
    site = fp64._Site(kind, c, gs, d, "shared", gen, dev)
    _native.clear_status(dev)
    y, fams = _profiled(lambda: site.norm(x, site.mods, site.gamma if affine else None, site.beta if affine else None,
                                          relu=relu))
    assert y.is_contiguous(memory_format=CL) and y.grad_fn.cfg[3] & _native.LAYOUT_NHWC
    assert y.grad_fn.saved_tensors[0].data_ptr() == x.data_ptr(), "x was copied"
    save_mean, save_w = y.grad_fn.saved_tensors[1:3]
    _, fb = _profiled(lambda: y.backward(dy))
    _only_cl(fams)
    _only_cl(fb)
    status = _native.status(dev)
    err = {}

    def add(key, got, ref):
        err.setdefault(key, fp64._Err()).add(got, ref)
    out = y.detach()
    for di in range(d):
        sl = slice(di * n, (di + 1) * n)
        x64 = fp64._f64(x[sl]).requires_grad_(True)
        pre = site.ref[di](x64)
        if affine:
            pre = pre * site.g64 + site.b64
        if relu:
            m = (out[sl] > 0).double()
            ref = pre * m
        else:
            ref = pre
        add("out", out[sl], ref.detach())
        (ref * fp64._f64(dy[sl])).sum().backward()
        add("dx", x.grad[sl], x64.grad)
        with torch.no_grad():
            mu, cov = site.batch_stats(x64.detach())
            add("mean", save_mean[di], mu)
            add("cov", site.kernel_cov(save_w[di]), cov)
    if affine:
        add("dgamma", site.gamma.grad, site.g64.grad)
        add("dbeta", site.beta.grad, site.b64.grad)
    for o in site.buf32:
        add("running_mean", site.buf32[o][0], site.buf64[o][0])
        add("running_var", site.buf32[o][1], site.buf64[o][1])
    if kind == "bn":
        assert [int(m.num_batches_tracked) for m in site.mods] == [int(m.num_batches_tracked) for m in site.ref] == [3] * d
    assert status == 0, status
    res = {k: e.both() for k, e in err.items()}
    for k, (rel, mx) in res.items():
        loose = kind == "whiten" and not k.startswith(fp64.STAT_KEYS)
        assert rel < (fp64.TOL if loose else fp64.TOL_STAT), (k, rel, mx)
        assert mx < (fp64.TOL_MAX if loose else 5 * fp64.TOL_STAT), (k, rel, mx)
    return res


@pytest.mark.parametrize("c4", WIDTHS)
def test_every_width(c4, dev, worst):
    """Each width with group sizes 1, 2, 4 and batch norm, epilogues none / affine / affine+relu / residual."""
    c = 4 * c4
    # 18 rows per domain (one chunk of one CTA); at some widths 1152, several chunks over several CTAs
    h, w = (24, 24) if c4 in DEEP else (3, 3) if c4 < 16383 else (1, 4)
    failures = []
    for i, (kind, gs) in enumerate(KINDS):
        for epi in ("none", "affine", "relu", "residual"):
            label = f"C={c} {kind} gs{gs} {epi}"
            try:
                if epi in ("none", "affine"):
                    _check_epi(dev, kind, c, gs, 3, 2, h, w, affine=epi == "affine", relu=False, seed=c4 + i)
                else:
                    path = "plain" if epi == "relu" else "residual"
                    _, fams = _profiled(lambda: fp64._check(dev, worst, label, "widths", kind=kind, c=c, gs=gs, d=3, n=2,
                                                             h=h, w=w, path=path, fork=False, seed=c4 + i))
                    _only_cl(fams)
            except AssertionError as e:
                failures.append(f"{label}: {e}")
    assert not failures, "\n".join(failures)


# --------------------------------------------------------------------------- two-site tail, row edges, fork
@pytest.mark.parametrize("c", [48, 1284])
def test_two_site_tail(c, dev, worst):
    for i, layouts in enumerate([("shared", "shared"), ("distinct", "distinct"), ("mixed", "mixed")]):
        for kind, gs in (("whiten", 4), ("bn", 1)):
            _, fams = _profiled(lambda: fp64._check(dev, worst, f"tail2 C={c} {kind} {layouts}", "tail2", kind=kind, c=c,
                                                     gs=gs, d=3, n=2, h=4, w=4, path="tail2", fork=i == 1,
                                                     layouts=layouts, seed=c + i))
            _only_cl(fams)
            assert fams.get("cl_tail2_apply", 0) == 1, fams


def _edge_rows(rows, c, d, sms, s):
    """Rows per domain of a named launch edge, from the slab count s the library launches at C."""
    _, _, rpi, _ = shape_of(c // 4, s)
    cap = max(1, STATS_SLOTS * sms // (s * d))
    chunk = rpi * STATS_UNROLL
    if rows == "lt_rpi":
        assert rpi > 1
    n = {"lt_rpi": rpi - 1, "chunk": chunk, "chunk+1": chunk + 1, "ragged": (2 * cap + 7) * chunk - 5}[rows]
    if rows == "ragged":      # enough work for the capped grid, and a last round in which only some CTAs have a chunk
        assert n // (2 * chunk) >= cap and -(-n // chunk) % cap != 0
    return n


EDGES = [   # C, path, kind, gs, domains, rows
    (12, "plain", "whiten", 4, 1, "lt_rpi"),
    (12, "residual", "bn", 1, 3, "ragged"),
    (48, "tail2", "whiten", 2, 2, "chunk"),
    (48, "plain", "whiten", 4, 4, "chunk+1"),
    (20, "residual", "whiten", 1, 2, "lt_rpi"),
    (400, "plain", "bn", 1, 3, "chunk+1"),
    (400, "tail2", "whiten", 4, 1, "ragged"),
    (576, "residual", "whiten", 2, 4, "chunk"),
    (1028, "plain", "whiten", 4, 3, "ragged"),
    (1028, "residual", "bn", 1, 1, "chunk+1"),
    (2052, "tail2", "bn", 1, 3, "lt_rpi"),
]


@pytest.mark.parametrize("c,path,kind,gs,d,rows", EDGES, ids=[f"c{e[0]}-{e[1]}-{e[2]}-gs{e[3]}-d{e[4]}-{e[5]}" for e in EDGES])
def test_row_edges(c, path, kind, gs, d, rows, dev, worst, slab_counts):
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    m = _edge_rows(rows, c, d, sms, slab_counts[c])
    _, fams = _profiled(lambda: fp64._check(dev, worst, f"c{c} {path} {rows}={m}", "edges", kind=kind, c=c, gs=gs, d=d,
                                             n=1, h=1, w=m, path=path, fork=rows == "chunk",
                                             layouts=("mixed" if d >= 3 else "distinct", "shared"), seed=c + d))
    _only_cl(fams)


@pytest.mark.parametrize("c", [48, 576, 1000])
def test_fork_for_sum_equals_autograd_add(c, dev):
    """dout2 summed in the kernels == autograd adding the two gradients first, bit for bit."""
    import dwt_b200
    gen = torch.Generator(device=dev).manual_seed(c)
    shape = (6, c, 5, 4)
    x0 = fp64._activation(gen, shape, 3, dev).contiguous(memory_format=CL)
    g1 = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=CL)
    g2 = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=CL)
    outs = []
    for forked in (True, False):
        site = fp64._Site("whiten", c, 4, 3, "shared", torch.Generator(device=dev).manual_seed(1), dev)
        x = x0.clone().requires_grad_(True)
        y = site.norm(x, site.mods, site.gamma, site.beta, relu=True)
        if forked:
            u, v = dwt_b200.fork_for_sum(y)
            assert u.grad_fn is not None
            torch.autograd.backward([u, v], [g1, g2])
        else:
            y.backward(g1 + g2)
        outs.append((x.grad, site.gamma.grad, site.beta.grad))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# --------------------------------------------------------------------------- eval, no-grad, replicated
@pytest.mark.parametrize("c", [48, 1028])
@pytest.mark.parametrize("kind,gs", [("whiten", 4), ("bn", 1)])
def test_modes(c, kind, gs, dev):
    """Eval against the fp64 modules in eval mode; no-grad training == training; replicated against the NCHW call."""
    from dwt_b200 import _native
    gen = torch.Generator(device=dev).manual_seed(c + gs)
    shape = (6, c, 4, 4)
    x = fp64._activation(gen, shape, 3, dev).contiguous(memory_format=CL)
    site = fp64._Site(kind, c, gs, 3, "distinct", gen, dev)
    # eval
    for m in site.mods + site.ref:
        m.eval()
    y, fams = _profiled(lambda: site.norm(x, site.mods, site.gamma, site.beta, relu=True))
    _only_cl(fams)
    assert y.is_contiguous(memory_format=CL)
    ref = torch.cat([site.ref[di](fp64._f64(x[2 * di:2 * di + 2])) for di in range(3)]) * site.g64 + site.b64
    e = fp64._Err()
    e.add(y.detach(), ref.clamp_min(0).detach())
    rel, mx = e.both()
    assert rel < (fp64.TOL if kind == "whiten" else fp64.TOL_STAT) and mx < fp64.TOL_MAX, (rel, mx)
    # no-grad training == training, running buffers included
    results = []
    for grad in (True, False):
        s = fp64._Site(kind, c, gs, 3, "shared", torch.Generator(device=dev).manual_seed(9), dev)
        with torch.set_grad_enabled(grad):
            yy, fams = _profiled(lambda: s.norm(x, s.mods, s.gamma, s.beta, relu=True))
        _only_cl(fams)
        results.append([yy.detach()] + [t.clone() for o in s.buf32 for t in s.buf32[o]])
    assert all(torch.equal(a, b) for a, b in zip(*results))
    # replicated: the channels-last call against the NCHW call on the same values
    got = []
    for xin in (x, x.contiguous()):
        s = fp64._Site(kind, c, gs, 3, "shared", torch.Generator(device=dev).manual_seed(4), dev)
        yy = s.norm(xin, s.mods, s.gamma, s.beta, relu=True, replicated=True)
        assert yy.is_contiguous(memory_format=CL) == (xin is x)
        got.append(yy.detach().contiguous())
    assert (got[0] - got[1]).norm() / got[1].norm() < (1e-4 if kind == "whiten" else 1e-5)
    assert _native.status(dev) == 0


# --------------------------------------------------------------------------- bf16 and NCHW agreement
@pytest.mark.parametrize("c", [12, 48, 400, 1028])
@pytest.mark.parametrize("kind,gs", [("whiten", 2), ("whiten", 4), ("bn", 1)])
def test_bf16_equals_fp32_rounded(c, kind, gs, dev):
    """A bf16 channels-last call == the fp32 channels-last call on x.float(), rounded; only cl_*_bf16 families run."""
    from dwt_b200 import functional as F
    gen = torch.Generator(device=dev).manual_seed(c)
    shape = (6, c, 4, 4)
    x0 = fp64._activation(gen, shape, 3, dev).contiguous(memory_format=CL).to(BF)
    r0 = fp64._activation(gen, shape, 3, dev).contiguous(memory_format=CL).to(BF)
    dy = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=CL).to(BF)
    arms = []
    for dt in (BF, torch.float32):
        s = fp64._Site(kind, c, gs, 3, "shared", torch.Generator(device=dev).manual_seed(2), dev)
        x = x0.to(dt).detach().requires_grad_(True)
        r = r0.to(dt).detach().requires_grad_(True)
        second = "running_variance" if kind == "whiten" else "running_var"
        y, fams = _profiled(lambda: F.norm(x, s.gamma, s.beta, kind=kind, group_size=gs, n_domains=3, training_stats=True,
                                           eps=1e-5, momentum=0.1, update_running=True, relu=True, residual=r,
                                           running=[(m.running_mean, getattr(m, second)) for m in s.mods]))
        _only_cl(fams, bf16=dt == BF)
        assert y.dtype == dt and y.is_contiguous(memory_format=CL)
        stats = [t.clone() for t in y.grad_fn.saved_tensors[1:3]]
        _, fb = _profiled(lambda: y.backward(dy.to(dt)))
        _only_cl(fb, bf16=dt == BF)
        arms.append([y.detach(), x.grad, r.grad, s.gamma.grad, s.beta.grad] + stats +
                    [t.clone() for o in s.buf32 for t in s.buf32[o]])
    a, b = arms
    for i, (p, q) in enumerate(zip(a, b)):
        assert torch.equal(p, q.to(p.dtype)), i


@pytest.mark.parametrize("c", [12, 48, 400, 1028, 4 * 513])
@pytest.mark.parametrize("kind,gs", [("whiten", 4), ("bn", 1)])
def test_against_nchw_call(c, kind, gs, dev):
    """The channels-last call and the NCHW call on x.contiguous() agree to fp32 rounding."""
    gen = torch.Generator(device=dev).manual_seed(c)
    shape = (6, c, 5, 5)
    x0 = fp64._activation(gen, shape, 3, dev).contiguous(memory_format=CL)
    dy = torch.randn(shape, device=dev, generator=gen)
    res = []
    for xin in (x0, x0.contiguous()):
        s = fp64._Site(kind, c, gs, 3, "shared", torch.Generator(device=dev).manual_seed(2), dev)
        x = xin.clone(memory_format=torch.preserve_format).requires_grad_(True)
        y = s.norm(x, s.mods, s.gamma, s.beta, relu=True)
        y.backward(dy)
        res.append([y.detach(), x.grad, s.gamma.grad, s.beta.grad] + [t for o in s.buf32 for t in s.buf32[o]])
    tol = 1e-4 if kind == "whiten" else 1e-5
    for i, (p, q) in enumerate(zip(*res)):
        rel = ((p - q).norm() / q.norm().clamp_min(1e-30)).item()
        assert rel < tol, (i, rel)


# --------------------------------------------------------------------------- models
def test_lenet_channels_last_step(dev, monkeypatch):
    """The LeNet with channels-last input and conv weights: one training step within tolerance of the NCHW step, both
    whitening sites (C = 32 and the conv2 site, C = 48) on the channels-last kernels."""
    import copy

    import dwt_b200
    from harness.lenet_dwt import LeNetDWT
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)      # both steps convolve in full fp32
    torch.manual_seed(5)
    proto = LeNetDWT(dwt_b200).to(dev).train()
    images = torch.randn(2 * 64, 1, 28, 28, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    steps = []
    for cl in (True, False):
        model = copy.deepcopy(proto)
        x = images
        if cl:
            model = model.to(memory_format=CL)
            x = images.contiguous(memory_format=CL)
        seen = []
        hook = model.conv2.register_forward_hook(lambda m, i, o: seen.append(o.is_contiguous(memory_format=CL)))
        logits, fams = _profiled(lambda: model(x))
        loss = logits.logsumexp(1).mean()
        _, fb = _profiled(lambda: loss.backward())
        hook.remove()
        if cl:
            assert seen == [True]
            assert fams.get("cl_stats", 0) == 4 and fams.get("cl_apply", 0) == 4, fams       # 2 sites x 2 domains
            assert fb.get("cl_bwd_reduce", 0) == 4, fb
            assert not any(k.startswith(("small_", "tiled_", "tc_")) for k in list(fams) + list(fb)), (fams, fb)
        steps.append([logits.detach(), loss.detach()] + [p.grad for p in model.parameters()])
    # a gradient that cancels to nearly nothing (beta1: site 2 removes per-channel shifts) is held to the step's scale
    scale = torch.cat([q.reshape(-1) for q in steps[1][2:]]).norm()
    for i, (p, q) in enumerate(zip(*steps)):
        err = (p - q).norm()
        assert err < 1e-3 * q.norm() + 1e-5 * scale, (i, err.item(), q.norm().item())


def test_mobilenet_width_stack(dev):
    """DomainTripleNorm sites at MobileNet-style widths between 1x1 convolutions: channels-last end to end, every
    site on the channels-last kernels, forward and backward."""
    import dwt_b200
    torch.manual_seed(0)
    widths = [24, 96, 144, 192, 320, 576]
    convs = torch.nn.ModuleList([torch.nn.Conv2d(a, b, 1, bias=False) for a, b in zip([16] + widths[:-1], widths)])
    convs = convs.to(dev).to(memory_format=CL)
    sites = []
    for i, c in enumerate(widths):
        kind, gs = ("whiten", 4) if i % 2 == 0 else ("bn", 1)
        mods = [dwt_b200.WTransform2d(c, gs) if kind == "whiten" else
                dwt_b200.BatchNorm2d(c, torch.zeros(c, device=dev), torch.ones(c, device=dev), affine=False) for _ in range(3)]
        mods = [m.to(dev).train() for m in mods]
        sites.append((dwt_b200.DomainTripleNorm(kind, c, gs, n_domains=3), mods,
                      torch.ones(c, 1, 1, device=dev, requires_grad=True), torch.zeros(c, 1, 1, device=dev, requires_grad=True)))
    x = torch.randn(6, 16, 14, 14, device=dev).contiguous(memory_format=CL)

    def run():
        h = x
        for conv, (norm, mods, g, b) in zip(convs, sites):
            h = norm(conv(h), mods, g, b, relu=True)
            assert h.is_contiguous(memory_format=CL) and not h.is_contiguous()
        return h
    y, fams = _profiled(run)
    _, fb = _profiled(lambda: y.square().mean().backward())
    _only_cl(fams)
    _only_cl(fb)
    assert fams["cl_stats"] == len(widths) and fb["cl_bwd_reduce"] == len(widths), (fams, fb)
    assert all(torch.isfinite(g.grad).all() for _, _, g, _ in sites)


# --------------------------------------------------------------------------- the C ABI
def test_c_abi_return_codes(dev):
    from dwt_b200 import _native
    lib = _native.lib()
    assert lib.dwt_abi_version() == 10
    n, hw, d = 2, 16, 1
    V = ctypes.c_void_p

    def call(c, gs=4, offset=0, ws_bytes=None, bwd=False):
        buf = torch.zeros(n * c * hw + 64, device=dev)
        x = buf.data_ptr() + offset
        out = torch.zeros_like(buf)
        st = torch.zeros(4 * c * gs, device=dev)
        gb = _native.ptr(st)
        rm = _native.ptr_array([st] * d)
        ws = torch.zeros((lib.dwt_workspace_bytes(n, c, hw, gs, d) if c % gs == 0 else 1 << 20) // 4 + 64, device=dev)
        nbytes = ws.numel() * 4 if ws_bytes is None else ws_bytes
        if bwd:
            return lib.dwt_whiten_bwd(V(x), V(x), None, _native.ptr(out), n, c, hw, gs, d, _native.LAYOUT_NHWC, 1e-3, gb,
                                      gb, None, None, None, None, 0, None, None, _native.ptr(ws), nbytes, _native.stream_ptr(dev))
        return lib.dwt_whiten_fwd(V(x), _native.ptr(out), n, c, hw, gs, d, _native.LAYOUT_NHWC, 1e-3, 0.1, 0, rm, rm, gb,
                                  gb, None, None, 0, gb, gb, _native.ptr(ws), nbytes, _native.stream_ptr(dev))
    for c in (48, 1028, 4 * 16383):
        assert lib.dwt_workspace_bytes(n, c, hw, 4, d) > 0
        assert call(c) == 0 and call(c, bwd=True) == 0, lib.dwt_last_error()
        assert call(c, ws_bytes=lib.dwt_workspace_bytes(n, c, hw, 4, d) // 2) == -2
    assert call(4 * 16384 + 8, gs=2) == -4                    # C/4 > 16384 (C divisible by gs: refused on layout)
    assert b"C/4 <= 16384" in lib.dwt_last_error()
    assert call(50, gs=2) == -4                               # C % 4 != 0
    assert call(48, offset=4) == -1                           # misaligned NHWC tensor
    torch.cuda.synchronize(dev)
    _native.clear_status(dev)


# --------------------------------------------------------------------------- CUDA graphs
def test_graph_capture(dev):
    """One C = 144 site (gs 4, AFFINE|RELU, distinct buffers) forward + backward captured and replayed twice: bit for
    bit the eager step, running buffers included."""
    gen = torch.Generator(device=dev).manual_seed(3)
    shape = (6, 144, 8, 8)
    x = fp64._activation(gen, shape, 3, dev).contiguous(memory_format=CL)
    dy = torch.randn(shape, device=dev, generator=gen).contiguous(memory_format=CL)
    site = fp64._Site("whiten", 144, 4, 3, "distinct", gen, dev)
    running = [t for o in sorted(site.buf32) for t in site.buf32[o]]
    r0 = [t.clone() for t in running]

    def step():
        xi = x.detach().requires_grad_(True)
        y = site.norm(xi, site.mods, site.gamma, site.beta, relu=True)
        return (y,) + torch.autograd.grad(y, (xi, site.gamma, site.beta), dy)
    eager = [t.detach().clone() for t in step()]
    r1 = [t.clone() for t in running]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = step()
    for _ in range(2):
        for t, v in zip(running, r0):
            t.copy_(v)
        g.replay()
        torch.cuda.synchronize(dev)
        assert all(torch.equal(p, q) for p, q in zip(got, eager))
        assert all(torch.equal(p, q) for p, q in zip(running, r1))
