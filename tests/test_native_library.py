"""CPU-side checks of the C-ABI library and the Python boundary (no kernel is launched)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    import __graft_entry__ as entry
    entry.build()
    from dwt_b200 import _native
    return _native


def test_library_exports_every_declared_symbol(built_lib):
    header = open(os.path.join(ROOT, "include", "dwt_b200.h")).read()
    declared = set(re.findall(r"DWT_API\s+[\w\s\*]+?\b(dwt_\w+)\s*\(", header))
    assert declared == set(built_lib.EXPORTS), declared ^ set(built_lib.EXPORTS)
    handle = ctypes.CDLL(built_lib.LIB_PATH)
    for name in declared:
        assert hasattr(handle, name), name
    assert built_lib.lib().dwt_abi_version() == built_lib.ABI_VERSION


def test_library_has_no_torch_dependency(built_lib):
    import subprocess
    out = subprocess.run(["ldd", built_lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "torch" not in out and "libc10" not in out, out


def test_workspace_size_query(built_lib):
    lib = built_lib.lib()
    assert lib.dwt_workspace_bytes(64, 64, 3136, 4, 3) > 0
    assert lib.dwt_workspace_bytes(64, 64, 3136, 5, 3) == 0        # 64 % 5 != 0
    assert lib.dwt_workspace_bytes(64, 256, 3136, 128, 1) == 0     # group size above the built maximum


def test_argument_validation_needs_no_gpu(built_lib):
    lib = built_lib.lib()
    rc = lib.dwt_mec_fwd_bwd(None, None, 4, 5, None, None, None, None)
    assert rc == -1 and b"null" in lib.dwt_last_error()


def test_no_cpu_fallback(built_lib):
    import dwt_b200
    with pytest.raises(built_lib.NativeError, match="no CPU fallback"):
        dwt_b200.WTransform2d(8, 4)(torch.zeros(2, 8, 3, 3))
    with pytest.raises(built_lib.NativeError, match="no CPU fallback"):
        dwt_b200.MinEntropyConsensusLoss(5, "cpu")(torch.zeros(2, 5), torch.zeros(2, 5))
    with pytest.raises(built_lib.NativeError, match="no CPU fallback"):
        dwt_b200.BatchNorm2d(8, torch.zeros(8), torch.ones(8))(torch.randn(2, 8, 3, 3))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "dwt-domain-adaptation_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f
                assert not re.search(r"sys\.path\.(insert|append)", src), f     # no path games -> no reference imports


def test_module_surface_matches_reference():
    """Constructor signatures, attributes, buffer names/shapes, error texts (SURVEY.md §8b)."""
    import batch_norm
    import consensus_loss
    import whitening
    sig = inspect.signature(whitening.WTransform2d.__init__)
    assert list(sig.parameters)[1:] == ["num_features", "group_size", "running_m", "running_var", "momentum",
                                        "track_running_stats", "eps", "alpha"]
    assert sig.parameters["momentum"].default == 0.1 and sig.parameters["eps"].default == 1e-3
    m = whitening.WTransform2d(8, 16)                      # group size clamps to C
    assert (m.group_size, m.num_groups) == (8, 1)
    assert tuple(m.running_mean.shape) == (1, 8, 1, 1) and tuple(m.running_variance.shape) == (1, 8, 8)
    assert torch.all(m.running_variance == 1) and list(dict(m.named_parameters())) == []
    rm, rv = torch.zeros(1, 8, 1, 1), torch.ones(2, 4, 4)
    a, b = whitening.WTransform2d(8, 4, running_m=rm, running_var=rv), whitening.WTransform2d(8, 4, running_m=rm, running_var=rv)
    assert a.running_mean.data_ptr() == b.running_mean.data_ptr() == rm.data_ptr()      # registered, not copied
    with pytest.raises(ValueError, match=r"expected 4D input \(got 3D input\)"):
        m(torch.zeros(2, 8, 3))
    with pytest.raises(ValueError, match="expected number of channels divisible by group_size"):
        whitening.WTransform2d(48, 32)(torch.zeros(2, 48, 3, 3))

    sig = inspect.signature(batch_norm.BatchNorm2d.__init__)
    assert list(sig.parameters)[1:] == ["num_features", "running_m", "running_v", "eps", "momentum", "affine",
                                        "track_running_stats"]
    rmean, rvar = torch.zeros(6), torch.ones(6)
    bn = batch_norm.BatchNorm2d(num_features=6, running_m=rmean, running_v=rvar, affine=False)
    assert bn.running_mean.data_ptr() == rmean.data_ptr() and bn.weight is None and int(bn.num_batches_tracked) == 0
    assert set(bn.state_dict()) == {"running_mean", "running_var", "num_batches_tracked"}
    assert "6, eps=1e-05, momentum=0.1, affine=False" in repr(bn)
    for cls, bad, msg in [(batch_norm.BatchNorm1d, (2, 6, 3, 3), "expected 2D or 3D input"),
                          (batch_norm.BatchNorm2d, (2, 6, 3), "expected 4D input"),
                          (batch_norm.BatchNorm3d, (2, 6, 3, 3), "expected 5D input")]:
        with pytest.raises(ValueError, match=msg):
            cls(6, torch.zeros(6), torch.ones(6))(torch.zeros(*bad))
    old = {"running_mean": torch.zeros(6), "running_var": torch.ones(6)}               # v1 checkpoint: no counter
    bn.load_state_dict(old)
    crit = consensus_loss.MinEntropyConsensusLoss(num_classes=65, device="cpu")
    assert crit.num_classes == 65 and crit.device == "cpu"


def test_tensor_core_objects_contain_hopper_instructions(built_lib):
    """The large-group kernels must really be TMA + wgmma code: their sm_90a objects carry the SASS mnemonics of
    warpgroup tf32 MMAs (HGMMA ... TF32), bulk tensor loads (UTMALDG) and transaction mbarriers (SYNCS); an
    mma.sync/FFMA fallback would show none."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    lib_dir = os.path.dirname(built_lib.LIB_PATH)
    want = {"norm_tc.o": ["HGMMA.64x64x8.F32.TF32", "UTMALDG", "SYNCS.PHASECHK.TRANS64.TRYWAIT"],
            "norm_tc_apply.o": ["HGMMA.64x64x8.F32.TF32", "UTMALDG", "SYNCS.PHASECHK.TRANS64.TRYWAIT"]}
    for obj, mnemonics in want.items():
        sass = subprocess.run([cuobjdump, "-sass", os.path.join(lib_dir, obj)], capture_output=True, text=True).stdout
        assert "sm_90a" in sass, obj
        for m in mnemonics:
            assert m in sass, f"{obj}: no {m} in SASS"


def test_extensions_refuse_cpu_tensors_too(built_lib):
    """The extension entry points (fused site, head loss, augmentation) have no CPU path either."""
    import dwt_b200
    mods = [dwt_b200.WTransform2d(8, 4).train() for _ in range(3)]
    g, b = torch.ones(8, 1, 1), torch.zeros(8, 1, 1)
    with pytest.raises(built_lib.NativeError):
        dwt_b200.DomainTripleNorm("whiten", 8, 4)(torch.randn(6, 8, 4, 4), mods, g, b)
    with pytest.raises(built_lib.NativeError):
        dwt_b200.DomainTripleNorm("whiten", 8, 4)(torch.randn(2, 8, 4, 4), mods, g, b, replicated=True)
    with pytest.raises(built_lib.NativeError):
        dwt_b200.HeadLoss(5, 0.1)(torch.randn(6, 5), torch.zeros(2, dtype=torch.int64))
    with pytest.raises(built_lib.NativeError):
        dwt_b200.PairedAugment(crop=4)(torch.zeros(2, 6, 6, 3, dtype=torch.uint8),
                                       crop_plain=torch.zeros(2, 2, dtype=torch.int32), want_aug=False)


def test_replicated_site_bookkeeping_errors_and_counters(built_lib):
    """Host logic of the statistics-collection site that runs before any kernel: a running_mean shared by branches
    whose second-moment buffers differ cannot be folded into one update (ValueError); BN branch counters advance
    once per branch (utils/batch_norm.py:57-58) even though the site is evaluated once."""
    import dwt_b200
    rm, rv1, rv2 = torch.zeros(1, 8, 1, 1), torch.eye(4).repeat(2, 1, 1), torch.eye(4).repeat(2, 1, 1)
    mods = [dwt_b200.WTransform2d(8, 4, running_m=rm, running_var=v).train() for v in (rv1, rv2, rv2)]
    with pytest.raises(ValueError, match="paired"):
        dwt_b200.DomainTripleNorm("whiten", 8, 4)(torch.randn(2, 8, 4, 4), mods, torch.ones(8, 1, 1), torch.zeros(8, 1, 1),
                                                  replicated=True)
    bm, bv = torch.zeros(8), torch.ones(8)
    bns = [dwt_b200.BatchNorm2d(8, bm, bv, affine=False).train() for _ in range(3)]
    with pytest.raises(built_lib.NativeError):          # CPU tensors: refused by the kernel call, after the bookkeeping
        dwt_b200.DomainTripleNorm("bn", 8)(torch.randn(2, 8, 4, 4), bns, torch.ones(8, 1, 1), torch.zeros(8, 1, 1),
                                           replicated=True)
    assert [int(m.num_batches_tracked) for m in bns] == [1, 1, 1]


def test_fork_for_sum_is_the_identity_without_a_site_output():
    """fork_for_sum only changes how gradients are summed when its argument is the output of one of the package's norm
    sites; anything else (and anything under no_grad) comes back as the same object twice, so autograd adds as usual."""
    import torch
    import dwt_b200
    t = (torch.randn(3, 4, requires_grad=True) * 2.0)
    a, b = dwt_b200.fork_for_sum(t)
    assert a is t and b is t
    (a.sum() + (b * b).sum()).backward()
    with torch.no_grad():
        u = torch.randn(2, 2)
        a, b = dwt_b200.fork_for_sum(u)
        assert a is u and b is u
