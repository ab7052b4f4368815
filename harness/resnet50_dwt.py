"""ResNet-50-DWT measurement harness (the model the hot-path layers drop into).

The reference model lives in its experiment script
(/root/reference/resnet50_dwt_mec_officehome.py:40-378), which cannot travel to
the GPU box and is out of scope to rebuild (SURVEY.md §2).  This file re-states
only its *topology* so that ``bench.py`` and the parity tests have something to
drop the layers into: a torchvision-style ResNet-50 whose every norm site is a
domain triple (source | target | target-aug), whitening in the stem and layer1,
domain batch-norm in layers 2-4, one shared gamma/beta per site.

Parameter and buffer names match the reference model one-for-one, so a state
dict produced for one loads into the other (``tests/test_harness_vs_reference``
checks logits/loss/grads against the unmodified reference script in the build
container).  The norm layers come from a ``layers`` namespace -- the product
package ``dwt_b200`` by default, the CPU oracle port in CPU tests:

    layers.WTransform2d, layers.BatchNorm2d           (reference-compatible ctors)
    layers.DomainTripleNorm (optional)                (fused site, SURVEY.md §8f-1)

``site_mode``:
    "modules"  reference composition: split/3 -> 3 modules -> cat -> *gamma+beta -> relu
               (resnet50_dwt_mec_officehome.py:220-222,335-337)
    "fused"    one DomainTripleNorm call per site (needs layers.DomainTripleNorm)
"""
from __future__ import annotations

import torch
import torch.nn as nn

_STAGES = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))   # planes, blocks, stride
_DOMAINS = ("s", "t", "t_aug")                                   # bns*, bnt*, bnt*_aug
EXPANSION = 4


_REPLICATED = [False]          # set by collect_stats(): one copy of the batch stands for all three branches
_BATCHED_COUNTERS = [False]    # set inside ResNet50DWT.forward (fused sites): the model has bumped every BN step counter itself


class WhitenScaleShift(nn.Module):
    """Same role and attribute names as the reference's ``whitening_scale_shift``
    (resnet50_dwt_mec_officehome.py:40-63): ``.wh`` is the whitening transform,
    optional per-channel ``gamma``/``beta``."""

    def __init__(self, layers, planes, group_size, running_mean, running_variance,
                 track_running_stats=True, affine=True):
        super().__init__()
        self.planes, self.group_size, self.affine = planes, group_size, affine
        self.wh = layers.WTransform2d(planes, group_size, running_m=running_mean,
                                      running_var=running_variance,
                                      track_running_stats=track_running_stats)
        if affine:
            self.gamma = nn.Parameter(torch.ones(planes, 1, 1))
            self.beta = nn.Parameter(torch.zeros(planes, 1, 1))

    def forward(self, x):
        y = self.wh(x)
        return y * self.gamma + self.beta if self.affine else y


class _SiteOwner(nn.Module):
    """Mixin: registers a domain-triple norm site under the reference's flat names
    (``bns1/bnt1/bnt1_aug/gamma1/beta1`` ...) and runs it."""

    def _add_site(self, layers, tag, key, planes, whiten, group_size, stats, site_mode):
        # tag: "1"/"2"/"3" -> bns{tag}, gamma{tag};  "downsample" -> downsample_bns, downsample_gamma
        pre, post = ("downsample_", "") if tag == "downsample" else ("", tag)
        names = [f"{pre}bn{d}{post}" if d != "t_aug" else f"{pre}bnt{post}_aug" for d in _DOMAINS]
        if whiten:
            rm, rv = stats[key + ".wh.running_mean"], stats[key + ".wh.running_variance"]
            gamma, beta = stats[key + ".gamma"], stats[key + ".beta"]
            mods = [WhitenScaleShift(layers, planes, group_size, rm, rv, affine=False) for _ in names]
        else:
            rm, rv = stats[key + ".running_mean"], stats[key + ".running_var"]
            gamma, beta = stats[key + ".weight"].view(-1, 1, 1), stats[key + ".bias"].view(-1, 1, 1)
            mods = [layers.BatchNorm2d(num_features=planes, running_m=rm, running_v=rv, affine=False)
                    for _ in names]
        for n, m in zip(names, mods):
            setattr(self, n, m)
        gname = f"{pre}gamma{post}" if pre == "" else "downsample_gamma"
        bname = f"{pre}beta{post}" if pre == "" else "downsample_beta"
        setattr(self, gname, nn.Parameter(gamma))
        setattr(self, bname, nn.Parameter(beta))
        if not hasattr(self, "_sites"):
            self._sites = {}
        self._sites[tag] = (names, gname, bname, whiten)
        if site_mode == "fused":
            # not registered as a submodule: it owns no state, only borrows the
            # three modules' buffers and the site's gamma/beta at call time.
            object.__setattr__(self, f"_fused_{tag}", layers.DomainTripleNorm(
                kind="whiten" if whiten else "bn", num_features=planes,
                group_size=group_size if whiten else 1))

    def _site(self, tag, x, relu, residual=None):
        """residual: the Bottleneck tail `relu(site(x) + identity)`; folded into the kernel by the fused site,
        applied with ATen ops otherwise."""
        names, gname, bname, whiten = self._sites[tag]
        gamma, beta = getattr(self, gname), getattr(self, bname)
        if residual is not None:
            fused = getattr(self, f"_fused_{tag}", None) if self.training else None
            if fused is not None:
                mods = [getattr(self, n) for n in names]
                return fused(x, [m.wh if whiten else m for m in mods], gamma, beta, True, residual=residual,
                             replicated=_REPLICATED[0], count_batches=not _BATCHED_COUNTERS[0])
            return torch.relu_(self._site(tag, x, relu=False) + residual)
        if self.training:
            fused = getattr(self, f"_fused_{tag}", None)
            mods = [getattr(self, n) for n in names]
            if fused is not None:
                return fused(x, [m.wh if whiten else m for m in mods], gamma, beta, relu, replicated=_REPLICATED[0],
                             count_batches=not _BATCHED_COUNTERS[0])
            if _REPLICATED[0]:
                raise RuntimeError("replicated statistics collection needs site_mode='fused'")
            parts = torch.split(x, x.shape[0] // 3, dim=0)
            s, t, a = (m(p) for m, p in zip(mods, parts))
            out = torch.cat((s, torch.cat((t, a), dim=0)), dim=0) * gamma + beta
        else:
            out = getattr(self, names[1])(x) * gamma + beta      # target branch only (:241-260)
        return torch.relu_(out) if relu else out


class Bottleneck(_SiteOwner):
    def __init__(self, layers, inplanes, planes, layer, sub_layer, stats, group_size, stride,
                 downsample, site_mode):
        super().__init__()
        whiten = layer == 1
        key = f"layer{layer}.{sub_layer}"
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self._add_site(layers, "1", key + ".bn1", planes, whiten, group_size, stats, site_mode)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride=stride, padding=1, bias=False)
        self._add_site(layers, "2", key + ".bn2", planes, whiten, group_size, stats, site_mode)
        self.conv3 = nn.Conv2d(planes, planes * EXPANSION, 1, bias=False)
        self._add_site(layers, "3", key + ".bn3", planes * EXPANSION, whiten, group_size, stats, site_mode)
        self.downsample = downsample
        if downsample is not None:
            self._add_site(layers, "downsample", f"layer{layer}.0.downsample_bn", planes * EXPANSION,
                           whiten, group_size, stats, site_mode)
        # x feeds the first convolution AND the identity (or downsample) branch: with the fused sites the two gradients
        # are summed inside the producing site's backward kernels instead of by an autograd `add` (layers.fork_for_sum)
        object.__setattr__(self, "_fork", getattr(layers, "fork_for_sum", None) if site_mode == "fused" else None)

    def forward(self, x):
        xa, xb = self._fork(x) if (self._fork is not None and self.training) else (x, x)
        out = self._site("1", self.conv1(xa), relu=True)
        out = self._site("2", self.conv2(out), relu=True)
        identity = xb if self.downsample is None else self._site("downsample", self.downsample(xb), relu=False)
        return self._site("3", self.conv3(out), relu=True, residual=identity)


class ResNet50DWT(_SiteOwner):
    def __init__(self, layers, state_dict, num_classes=65, group_size=4, site_mode="modules", stem_pad=0, stem_nchw=False,
                 stem_s2d=False):
        super().__init__()
        # stem_s2d: evaluate the 7x7 / stride-2 / pad-3 stem convolution as the 4x4 / stride-1 convolution of the 2x2
        # space-to-depth rearrangement of the image (12 channels) -- see _stem_s2d.  Same sums of the same products; the
        # 12-channel operand gives cuDNN a tensor-core implicit-GEMM kernel where the 3-channel one only has legacy
        # engines.
        self.stem_s2d = stem_s2d
        # stem_nchw: run ONLY the 3-channel 7x7 stem convolution in NCHW (its weight stays NCHW-contiguous, the image is
        # viewed / copied to NCHW, the 64-channel result is copied to channels-last once) -- cuDNN's NHWC engines for a
        # 3-channel input are legacy kernels; same arithmetic, different cuDNN kernel
        self.stem_nchw = stem_nchw
        # stem_pad = 4 / 8: feed the 7x7 stem convolution a zero-padded 4- / 8-channel image and the equally padded
        # weight -- identical arithmetic (the extra products are exact zeros), but cuDNN has no tensor-core kernel for
        # a 3-channel NHWC tensor and falls back to a legacy engine.  The parameter keeps the reference's [64, 3, 7, 7]
        # shape.
        self.stem_pad = stem_pad
        if site_mode not in ("modules", "fused"):
            raise ValueError("site_mode must be 'modules' or 'fused'")
        stats = {k: v for k, v in state_dict.items() if "bn" in k or "downsample" in k}
        self.site_mode = site_mode
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self._add_site(layers, "1", "bn1", 64, True, group_size, stats, site_mode)
        self.maxpool = nn.MaxPool2d(3, stride=2, padding=1)       # resnet50_dwt_mec_officehome.py:295
        inplanes = 64
        for li, (planes, blocks, stride) in enumerate(_STAGES, start=1):
            seq = []
            for b in range(blocks):
                down = None
                if b == 0 and (stride != 1 or inplanes != planes * EXPANSION):
                    down = nn.Sequential(nn.Conv2d(inplanes, planes * EXPANSION, 1, stride=stride, bias=False))
                # the reference's _make_layer never forwards ResNet's group_size (:316,325,328): always 4
                seq.append(Bottleneck(layers, inplanes, planes, li, b, stats, 4, stride if b == 0 else 1,
                                      down, site_mode))
                inplanes = planes * EXPANSION
            setattr(self, f"layer{li}", nn.Sequential(*seq))
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc_out = nn.Linear(512 * EXPANSION, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def _stem_s2d(self, x):
        """conv(x, w; k=7, s=2, p=3)[o, i, j] = sum_{c,u,v} w[o,c,u,v] xp[c, 2i+u, 2j+v]   (xp: x padded by 3).
        Write u = 2u' + a, v = 2v' + b (a, b in {0,1}; u', v' in 0..3; the taps u = 7 / v = 7 get a zero weight):
            = sum_{(c,a,b),u',v'} w4[o,(c,a,b),u',v'] xs[(c,a,b), i+u', j+v']
        with xs[(c,a,b), p, q] = xp[c, 2p+a, 2q+b] and w4[o,(c,a,b),u',v'] = w[o,c,2u'+a,2v'+b]: a 4x4 stride-1
        convolution of a 4C-channel image.  The parameter keeps the reference's [64, 3, 7, 7] shape (autograd carries
        the weight gradient back through the rearrangement); one copy of the image and of the weight per call."""
        n, c, h, w = x.shape
        if h % 2 or w % 2:
            return self.conv1(x)
        cl = x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous()
        xp = torch.nn.functional.pad(x, (3, 3, 3, 3))
        hp, wp = (h + 6) // 2, (w + 6) // 2
        wt = torch.nn.functional.pad(self.conv1.weight, (0, 1, 0, 1))
        o = wt.shape[0]
        if cl:      # build the NHWC memory order directly: [n, p, q, (c, a, b)]
            xs = xp.view(n, c, hp, 2, wp, 2).permute(0, 2, 4, 1, 3, 5).reshape(n, hp, wp, 4 * c).permute(0, 3, 1, 2)
            w4 = wt.view(o, c, 4, 2, 4, 2).permute(0, 2, 4, 1, 3, 5).reshape(o, 4, 4, 4 * c).permute(0, 3, 1, 2)
        else:
            xs = xp.view(n, c, hp, 2, wp, 2).permute(0, 1, 3, 5, 2, 4).reshape(n, 4 * c, hp, wp)
            w4 = wt.view(o, c, 4, 2, 4, 2).permute(0, 1, 3, 5, 2, 4).reshape(o, 4 * c, 4, 4)
        return torch.nn.functional.conv2d(xs, w4)

    def _stem(self, x):
        if self.stem_s2d:
            return self._stem_s2d(x)
        if self.stem_nchw:
            return self.conv1(x.contiguous()).contiguous(memory_format=torch.channels_last)
        if not self.stem_pad or x.shape[1] >= self.stem_pad:
            return self.conv1(x)
        extra = self.stem_pad - x.shape[1]
        fmt = torch.channels_last if (x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous()) \
            else torch.contiguous_format
        xp = torch.zeros((x.shape[0], self.stem_pad) + tuple(x.shape[2:]), dtype=x.dtype, device=x.device).contiguous(memory_format=fmt)
        xp[:, :x.shape[1]] = x
        w = torch.nn.functional.pad(self.conv1.weight, (0, 0, 0, 0, 0, extra))
        if fmt == torch.channels_last:
            w = w.contiguous(memory_format=torch.channels_last)
        c = self.conv1
        return torch.nn.functional.conv2d(xp, w, None, c.stride, c.padding, c.dilation, c.groups)

    def _bump_counters(self):
        """All 126 `num_batches_tracked += 1` (batch_norm.py:58) of a fused-site training forward as one launch."""
        cs = getattr(self, "_bn_counters", None)
        if cs is None:
            cs = [m.num_batches_tracked for m in self.modules()
                  if hasattr(m, "num_batches_tracked") and m.num_batches_tracked is not None and getattr(m, "track_running_stats", False)]
            object.__setattr__(self, "_bn_counters", cs)
        if cs:
            torch._foreach_add_(cs, 1)

    def forward(self, x):
        batched = self.training and self.site_mode == "fused"
        if batched:
            self._bump_counters()
        _BATCHED_COUNTERS[0] = batched
        try:
            x = self.maxpool(self._site("1", self._stem(x), relu=True))
            x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        finally:
            _BATCHED_COUNTERS[0] = False
        return self.fc_out(torch.flatten(self.avgpool(x), 1))


def build_resnet50_dwt(state_dict, layers, site_mode="modules", num_classes=65, channels_last=False, stem_pad=0,
                       stem_nchw=False, stem_s2d=False):
    """state_dict uses the reference checkpoint's key names *without* the 7-char
    ``module.`` prefix (resnet50_dwt_mec_officehome.py:370-376).  channels_last=True converts the
    convolution weights to torch.channels_last so that, fed channels-last images, every activation
    stays NHWC (no cuDNN NCHW<->NHWC copies); results are identical, only strides change."""
    model = ResNet50DWT(layers, state_dict, num_classes=num_classes, site_mode=site_mode, stem_pad=stem_pad,
                        stem_nchw=stem_nchw and channels_last, stem_s2d=stem_s2d)
    model.load_state_dict(state_dict, strict=False)
    if channels_last and hasattr(layers, "MaxPool2d"):
        model.maxpool = layers.MaxPool2d(3, stride=2, padding=1)    # the library's channels-last kernel pair (no state)
    if channels_last:
        # only the convolution weights: Module.to(memory_format=...) would also re-stride the [1,C,1,1]
        # running-mean buffers into fresh tensors and silently break the aliasing of the three domain branches
        for m in model.modules():
            if isinstance(m, nn.Conv2d) and not (model.stem_nchw and m is model.conv1):
                m.weight.data = m.weight.data.contiguous(memory_format=torch.channels_last)
    return model


def collect_stats(model, batches, passes=1, replicated=True):
    """The reference's pre-evaluation pass (resnet50_dwt_mec_officehome.py:380-389): train-mode forwards
    under no_grad that fold target batches into every branch's running statistics.  replicated=False is
    the reference's own form, ``model(cat((data, data, data)))``; replicated=True (fused sites only) feeds
    the single copy and lets each site apply the three identical updates at once (SURVEY.md §8f-3)."""
    was_training = model.training
    model.train(True)
    out = None
    try:
        with torch.no_grad():
            for _ in range(passes):
                for data in batches:
                    if replicated:
                        _REPLICATED[0] = True
                        out = model(data)
                    else:
                        out = model(torch.cat((data, data, data), dim=0))
    finally:
        _REPLICATED[0] = False
        model.train(was_training)
    return out
