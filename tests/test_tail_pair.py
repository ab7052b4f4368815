"""The two-site residual tail of a downsampling Bottleneck (DomainTripleNorm.forward_with_downsample on channels-last
tensors: dwt_tail2_fwd / dwt_tail2_bwd) against the two-call composition it replaces, bit for bit: the output, the
ReLU byte map, both sites' running buffers and every gradient."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


def _modules(kind, c, gs, dev, seed):
    """Three domain modules on ONE shared buffer pair (as in the model), the pair filled with non-trivial values."""
    import dwt_b200
    g = torch.Generator().manual_seed(seed)
    rm = torch.randn(c, generator=g) * 0.1
    if kind == "whiten":
        a = torch.randn(c // gs, gs, gs, generator=g) * 0.1
        rv = (a @ a.transpose(1, 2) + torch.eye(gs)).to(dev)
        rm = rm.view(1, c, 1, 1).to(dev)
        return [dwt_b200.WTransform2d(c, gs, running_m=rm, running_var=rv).to(dev).train() for _ in range(3)]
    rm, rv = rm.to(dev), (torch.rand(c, generator=g) + 0.5).to(dev)
    return [dwt_b200.BatchNorm2d(c, rm, rv, affine=False).to(dev).train() for _ in range(3)]


def _buffers(mods):
    return [b.clone() for b in mods[0].buffers()]


@pytest.mark.parametrize("fork", [False, True], ids=["single", "forked"])
@pytest.mark.parametrize("kind,c,gs,hw", [("whiten", 256, 4, 14), ("bn", 512, 1, 7)], ids=["layer1", "layer2"])
def test_tail_pair_equals_two_call_composition(kind, c, gs, hw, fork, dev):
    import dwt_b200
    n = 2                                                    # images per domain
    torch.manual_seed(c + hw)
    cl = torch.channels_last
    x3 = (torch.randn(3 * n, c, hw, hw, device=dev) * 1.5 + 0.3).contiguous(memory_format=cl)
    xd = (torch.randn(3 * n, c, hw, hw, device=dev) * 0.7 - 0.2).contiguous(memory_format=cl)
    g3, b3 = torch.rand(c, 1, 1, device=dev) + 0.5, torch.randn(c, 1, 1, device=dev) * 0.1
    gd, bd = torch.rand(c, 1, 1, device=dev) + 0.5, torch.randn(c, 1, 1, device=dev) * 0.1
    w1 = torch.randn(3 * n, c, hw, hw, device=dev).contiguous(memory_format=cl)
    w2 = torch.randn(3 * n, c, hw, hw, device=dev).contiguous(memory_format=cl)
    site, down = dwt_b200.DomainTripleNorm(kind, c, gs), dwt_b200.DomainTripleNorm(kind, c, gs)

    def run(pair):
        mods3, modsd = _modules(kind, c, gs, dev, 1), _modules(kind, c, gs, dev, 2)
        leaves = [t.clone().requires_grad_(True) for t in (x3, xd, g3, b3, gd, bd)]
        a3, ad, ga3, ba3, gad, bad = leaves
        if pair:
            y = site.forward_with_downsample(a3, mods3, ga3, ba3, ad, down, modsd, gad, bad)
            mask = y.grad_fn.saved_tensors[2]
        else:
            identity = down(ad, modsd, gad, bad, relu=False)
            y = site(a3, mods3, ga3, ba3, True, residual=identity)
            mask = y.grad_fn.saved_tensors[5]
        assert type(y.grad_fn).__name__.startswith("_TailPairFunction") == pair
        if fork:                                             # the output feeds the next block twice
            u, v = dwt_b200.fork_for_sum(y)
            loss = (u * w1).sum() + (v * w2).sum()
        else:
            loss = (y * w1).sum()
        loss.backward()
        return dict(out=y.detach(), mask=mask, buffers=_buffers(mods3) + _buffers(modsd), grads=[t.grad for t in leaves])

    ref, got = run(False), run(True)
    assert torch.equal(got["out"], ref["out"])
    assert torch.equal(got["mask"], ref["mask"])
    for a, b in zip(got["buffers"], ref["buffers"]):
        assert torch.equal(a, b)
    names = ["dx3", "dxd", "dgamma3", "dbeta3", "dgamma_d", "dbeta_d"]
    for name, a, b in zip(names, got["grads"], ref["grads"]):
        assert torch.equal(a, b), (name, (a - b).abs().max().item())


def test_tail_pair_falls_back_to_composition_for_nchw(dev):
    """NCHW tensors take the two-call composition (no two-site kernels exist for that layout)."""
    import dwt_b200
    c, gs = 16, 4
    x3, xd = torch.randn(6, c, 4, 4, device=dev), torch.randn(6, c, 4, 4, device=dev)
    g, b = torch.ones(c, 1, 1, device=dev), torch.zeros(c, 1, 1, device=dev)
    site = dwt_b200.DomainTripleNorm("whiten", c, gs)
    y = site.forward_with_downsample(x3, _modules("whiten", c, gs, dev, 1), g, b, xd, dwt_b200.DomainTripleNorm("whiten", c, gs),
                                     _modules("whiten", c, gs, dev, 2), g, b)
    identity = site(xd, _modules("whiten", c, gs, dev, 2), g, b, relu=False)
    assert torch.equal(y, site(x3, _modules("whiten", c, gs, dev, 1), g, b, True, residual=identity))
