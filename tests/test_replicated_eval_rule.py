"""What DomainTripleNorm asks of functional.norm in every module mode, replicated or not (no GPU: norm is stubbed).

The reference's statistics-collection pass feeds cat((data, data, data)) through the three domain modules
(resnet50_dwt_mec_officehome.py:380-389).  Through eval-mode modules each third is normalised with its module's running
statistics and no buffer moves; the replicated site stands for that with one copy of the batch, so its output -- the
first third -- must be normalised with mods[0]'s running buffers, never with the batch's statistics.  In training, every
distinct buffer pair gets one launch with the k-fold EMA factor 1 - (1 - m)^k; modules that track no running statistics
normalise with the batch and update nothing.
"""
import pytest
import torch

C, GS, N = 8, 4, 2
OWNERS = {"shared": [0, 0, 0], "distinct": [0, 1, 2], "mixed": [0, 1, 1]}


@pytest.fixture
def calls(monkeypatch):
    from dwt_b200 import functional as F
    seen = []

    def fake_norm(x, gamma, beta, **kw):
        seen.append(dict(kw, x=x))
        return x.clone()
    monkeypatch.setattr(F, "norm", fake_norm)
    return seen


def _site(kind, layout, mode, momentum=0.1, nbt=0, track=True):
    """(DomainTripleNorm, the three domain modules, their buffer pairs) with buffers aliased as `layout` says."""
    import dwt_b200
    bufs = {}
    mods = []
    for o in OWNERS[layout]:
        if o not in bufs:
            bufs[o] = ((torch.zeros(1, C, 1, 1), torch.eye(GS).repeat(C // GS, 1, 1)) if kind == "whiten"
                       else (torch.zeros(C), torch.ones(C)))
        rm, rv = bufs[o] if track else (None, None)
        if kind == "whiten":
            m = dwt_b200.WTransform2d(C, GS, running_m=rm, running_var=rv, momentum=momentum, track_running_stats=track)
        else:
            m = dwt_b200.BatchNorm2d(C, rm, rv, affine=False, momentum=momentum, track_running_stats=track)
            if track:
                m.num_batches_tracked.fill_(nbt)
        mods.append(m.train(mode == "train"))
    return dwt_b200.DomainTripleNorm(kind, C, GS), mods, [bufs[o] for o in sorted(bufs)]


def _second(kind, m):
    return m.running_variance if kind == "whiten" else m.running_var


def _args(kind):
    """gamma, beta of the site."""
    return torch.ones(C, 1, 1), torch.zeros(C, 1, 1)


@pytest.mark.parametrize("layout", list(OWNERS))
@pytest.mark.parametrize("kind", ["whiten", "bn"])
def test_replicated_eval_normalises_with_the_first_modules_running_buffers(kind, layout, calls):
    site, mods, pairs = _site(kind, layout, "eval", nbt=5)
    x = torch.randn(N, C, 4, 4)
    site(x, mods, *_args(kind), replicated=True)
    assert len(calls) == 1, calls
    kw = calls[0]
    assert kw["training_stats"] is False and kw["update_running"] is False and kw["momentum"] == 0.0
    assert kw["n_domains"] == 1 and kw["x"] is x
    (rm, rv), = kw["running"]
    assert rm is mods[0].running_mean and rv is _second(kind, mods[0])
    if kind == "bn":
        assert [int(m.num_batches_tracked) for m in mods] == [5, 5, 5]       # eval modules count no batches
    # the three-domain call on the same modules agrees: running statistics, nothing updated
    calls.clear()
    site(torch.randn(3 * N, C, 4, 4), mods, *_args(kind))
    assert len(calls) == 1 and calls[0]["training_stats"] is False and calls[0]["update_running"] is False


@pytest.mark.parametrize("layout", list(OWNERS))
@pytest.mark.parametrize("kind", ["whiten", "bn"])
def test_replicated_train_folds_k_updates_per_buffer_pair(kind, layout, calls):
    momentum = None if kind == "bn" else 0.1
    site, mods, pairs = _site(kind, layout, "train", momentum=momentum, nbt=2)
    site(torch.randn(N, C, 4, 4), mods, *_args(kind), replicated=True)
    f = 1.0 / 3.0 if kind == "bn" else 0.1              # momentum=None after the bump to 3: cumulative average
    owners = sorted(set(OWNERS[layout]))             # pairs in order of first use: the order of the launches
    assert len(calls) == len(pairs) == len(owners)
    for kw, o, (rm, rv) in zip(calls, owners, pairs):
        assert kw["training_stats"] is True and kw["update_running"] is True and kw["n_domains"] == 1
        assert kw["momentum"] == pytest.approx(1.0 - (1.0 - f) ** OWNERS[layout].count(o), rel=1e-12)
        assert kw["running"][0][0] is rm and kw["running"][0][1] is rv
    if kind == "bn":
        assert [int(m.num_batches_tracked) for m in mods] == [3, 3, 3]


def test_replicated_train_without_counting_batches(calls):
    """count_batches=False: the caller has bumped every counter already (the model's one multi-tensor launch)."""
    site, mods, pairs = _site("bn", "mixed", "train", momentum=None, nbt=3)
    site(torch.randn(N, C, 4, 4), mods, *_args("bn"), replicated=True, count_batches=False)
    assert [int(m.num_batches_tracked) for m in mods] == [3, 3, 3]
    assert [kw["momentum"] for kw in calls] == pytest.approx([1.0 / 3.0, 1.0 - (2.0 / 3.0) ** 2], rel=1e-12)


@pytest.mark.parametrize("replicated", [False, True])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("kind", ["whiten", "bn"])
def test_untracked_modules_use_batch_statistics_and_update_nothing(kind, mode, replicated, calls):
    site, mods, _ = _site(kind, "distinct", mode, track=False)
    site(torch.randn(N if replicated else 3 * N, C, 4, 4), mods, *_args(kind), replicated=replicated)
    assert len(calls) == 1
    assert calls[0]["training_stats"] is True and calls[0]["update_running"] is False


@pytest.mark.parametrize("layout", list(OWNERS))
@pytest.mark.parametrize("kind", ["whiten", "bn"])
def test_three_domain_site_modes(kind, layout, calls):
    """Not replicated: one call over the three domains with every branch's buffer pair, in domain order."""
    for mode in ("train", "eval"):
        calls.clear()
        site, mods, _ = _site(kind, layout, mode, nbt=2)
        site(torch.randn(3 * N, C, 4, 4), mods, *_args(kind))
        assert len(calls) == 1
        kw = calls[0]
        assert kw["training_stats"] is (mode == "train") and kw["update_running"] is (mode == "train")
        assert kw["n_domains"] == 3
        assert all(r[0] is m.running_mean and r[1] is _second(kind, m) for r, m in zip(kw["running"], mods))
        if mode == "train":
            assert kw["momentum"] == 0.1
        if kind == "bn":
            assert [int(m.num_batches_tracked) for m in mods] == [2 + (mode == "train")] * 3
