"""Edge-case fixture for the paired target augmentation, produced by the UNMODIFIED reference functions.

    python tests/golden/make_golden_augment_edges.py     # needs /root/reference, cv2, torchvision, PIL

Same pipeline as make_golden_augment.py (torchvision crop / hflip / to_tensor / normalize around the reference's
cv2.warpAffine call and its `_gaussian_blur`, resnet50_dwt_mec_officehome.py:481-492, 526-542), but every 2x3 matrix
is chosen here and handed to cv2.warpAffine directly, as that script's "strong" case does, and the geometry goes
where the GPU kernel and the numpy oracle have their edges:

  translate   translations of both signs, up to +- the crop, with and without a linear part
  reflect     negative determinants
  rot90       quarter turns about the origin and about the crop centre
  singular    near-singular matrices, and exactly singular ones (D = 0: the inverse is taken as all zeros)
  zoom        x4 and x0.25, about the origin and about the centre
  tall, wide  non-square sources (SH != SW), the crop as large as the shorter side
  full        crop = source size
  pixel       crop = 1
  corners     crops at all four corners, each with and without the flip
  saturated   images at 0 and at 255 everywhere, and half and half

Writes tests/golden/augment_edges.npz (tests/golden/augment.npz is left as it is).  Every array is a deterministic
function of the seed, so rerunning the script reproduces the fixture exactly.
"""
from __future__ import annotations

import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
warnings.filterwarnings("ignore")
os.chdir(REF)
sys.path.insert(0, REF)
sys.modules.setdefault("matplotlib", types.ModuleType("matplotlib"))
sys.modules.setdefault("matplotlib.pyplot", types.ModuleType("matplotlib.pyplot"))
import resnet50_dwt_mec_officehome as ref     # noqa: E402  (the experiment script, unmodified)
import cv2                                    # noqa: E402
from PIL import Image                         # noqa: E402
import torchvision.transforms.functional as TF  # noqa: E402

assert ref.__file__.startswith(REF)
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def smooth_image(rng, h, w):
    """Natural-image-like content: low-frequency colour gradients + texture, uint8."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([127 + 100 * np.sin(xx / (5 + 3 * k) + rng.random() * 6) * np.cos(yy / (7 + 2 * k) + rng.random() * 6)
                    for k in range(3)], axis=-1)
    img += rng.normal(0, 12, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def lin(a, b, c, d, tx=0.0, ty=0.0):
    return [[a, b, tx], [c, d, ty]]


def cases(rng):
    """-> [(name, SH, SW, crop, [(top, left, flip, 2x3 matrix), ...])]; the plain view's corners are drawn."""
    out = []
    c = 16
    out.append(("translate", 20, 20, c, [
        (2, 3, 0, lin(1, 0, 0, 1, c, 0)), (0, 0, 1, lin(1, 0, 0, 1, -c, 0)), (4, 4, 0, lin(1, 0, 0, 1, 0, c)),
        (1, 2, 1, lin(1, 0, 0, 1, 0, -c)), (3, 0, 0, lin(1, 0, 0, 1, 7.5, -3.25)), (0, 4, 1, lin(1, 0, 0, 1, -0.4, 0.7)),
        (2, 2, 0, lin(1.1, -0.2, 0.15, 0.9, -5.3, 9.7)), (4, 1, 1, lin(0.93, 0.05, -0.08, 1.07, 15.9, -15.9)),
        (1, 1, 0, lin(1, 0, 0, 1, c - 0.03125, -(c - 0.03125))), (3, 3, 1, lin(1, 0, 0, 1, 1e-3, -1e-3))]))
    out.append(("reflect", 18, 18, c, [
        (0, 0, 0, lin(-1, 0, 0, 1, c - 1, 0)), (2, 1, 1, lin(1, 0, 0, -1, 0, c - 1)), (1, 2, 0, lin(-1, 0, 0, -1, c - 1, c - 1)),
        (2, 2, 1, lin(0, 1, 1, 0)), (0, 1, 0, lin(0.9, 0.2, 0.3, -1.1, 1.0, 14.0)), (1, 0, 1, lin(-1, 0, 0, 1))]))
    out.append(("rot90", 17, 17, c, [
        (0, 0, 0, lin(0, -1, 1, 0, c - 1, 0)), (1, 1, 1, lin(0, 1, -1, 0, 0, c - 1)), (0, 1, 0, lin(0, -1, 1, 0)),
        (1, 0, 1, lin(0, 1, -1, 0)), (1, 1, 0, lin(0, -1, 1, 0, c, 0)), (0, 0, 1, lin(-1, 0, 0, -1, c, c))]))
    out.append(("singular", 20, 20, c, [
        (0, 0, 0, lin(1, 2, 0.5, 1)), (1, 2, 1, lin(0, 0, 0, 0, 3, -2)), (2, 1, 0, lin(2, 4, 1, 2, -1.5, 2.5)),
        (3, 3, 1, lin(1, 0, 0, 0, 4, 0)), (4, 0, 0, lin(1, 2, 0.5, 1.001)), (0, 4, 1, lin(1, 1, 1, 1.0078125, 2, -3)),
        (2, 3, 0, lin(0.01, 0, 0, 1)), (1, 1, 1, lin(1e-3, 0.5, -0.25, 2e-3, 8, 8))]))
    out.append(("zoom", 20, 20, c, [
        (0, 0, 0, lin(4, 0, 0, 4)), (2, 2, 1, lin(0.25, 0, 0, 0.25)), (1, 3, 0, lin(4, 0, 0, 4, -1.5 * c, -1.5 * c)),
        (3, 1, 1, lin(0.25, 0, 0, 0.25, 0.375 * c, 0.375 * c)), (4, 4, 0, lin(4, 0, 0, 0.25, -c, 2)),
        (0, 2, 1, lin(0.25, 0.1, -0.1, 4, 3, -20))]))
    sig = lambda: [rng.normal(0.0, 0.1) for _ in range(4)]                          # noqa: E731
    ref_like = lambda: (lambda n: lin(1 + n[0], n[1], n[2], 1 + n[3]))(sig())       # noqa: E731
    out.append(("tall", 24, 17, 12, [(12, 5, 0, ref_like()), (0, 0, 1, ref_like()), (7, 3, 1, lin(1, 0, 0, 1, 2, -5)),
                                     (3, 1, 0, lin(0, -1, 1, 0, 11, 0))]))
    out.append(("wide", 13, 30, 13, [(0, 17, 1, ref_like()), (0, 0, 0, ref_like()), (0, 9, 1, lin(-1, 0, 0, 1, 12, 0)),
                                     (0, 4, 0, lin(1.5, 0, 0, 0.75, -3, 1))]))
    out.append(("full", 11, 11, 11, [(0, 0, 1, ref_like()), (0, 0, 0, ref_like()), (0, 0, 1, lin(0.5, 0, 0, 2, 5, -5)),
                                     (0, 0, 0, lin(1, 0, 0, 1))]))
    out.append(("pixel", 5, 7, 1, [(0, 0, 0, lin(1, 0, 0, 1)), (4, 6, 1, ref_like()), (2, 3, 0, lin(1, 0, 0, 1, 0.5, 0.25)),
                                    (0, 6, 1, lin(1, 0, 0, 1, -0.5, -0.75)), (4, 0, 0, lin(3, 1, -1, 2, 0.1, 0.9))]))
    corner = []
    for flip in (0, 1):
        for top, left in ((0, 0), (0, 14), (10, 0), (10, 14)):
            corner.append((top, left, flip, ref_like() if (top + left + flip) % 2 else lin(1, 0, 0, 1, 1.5, -2.5)))
    out.append(("corners", 19, 23, 9, corner))
    out.append(("saturated", 14, 14, 12, [(0, 0, 0, ref_like()), (2, 2, 1, ref_like()), (1, 0, 0, ref_like()),
                                          (0, 2, 1, lin(0.8, 0.3, -0.3, 0.8, 2, 1))]))
    return out


def main():
    rng = np.random.default_rng(23)
    fixture, names = {}, []
    for name, sh, sw, crop, views in cases(rng):
        names.append(name)
        B = len(views)
        imgs = np.stack([smooth_image(rng, sh, sw) for _ in range(B)])
        if name == "saturated":
            imgs[0] = 0
            imgs[1] = 255
            imgs[2, :, : sw // 2] = 0
            imgs[2, :, sw // 2:] = 255
            imgs[3, : sh // 2] = 255
        crop_plain = rng.integers(0, [sh - crop + 1, sw - crop + 1], (B, 2)).astype(np.int32)
        crop_aug = np.int32([[v[0], v[1]] for v in views])
        flip = np.uint8([v[2] for v in views])
        mats = np.float32([v[3] for v in views])
        assert (crop_aug >= 0).all() and (crop_aug[:, 0] <= sh - crop).all() and (crop_aug[:, 1] <= sw - crop).all()
        plains, augs = [], []
        for b in range(B):
            pil = Image.fromarray(imgs[b])
            # plain view: :526-531
            p = TF.normalize(TF.to_tensor(TF.crop(pil, int(crop_plain[b, 0]), int(crop_plain[b, 1]), crop, crop)), MEAN, STD)
            # augmented view: :534-542, the matrix given instead of drawn (the body of _random_affine_augmentation)
            a = TF.crop(pil, int(crop_aug[b, 0]), int(crop_aug[b, 1]), crop, crop)
            if flip[b]:
                a = TF.hflip(a)
            a = TF.to_tensor(a)
            a = torch.from_numpy(np.transpose(cv2.warpAffine(np.transpose(a.numpy(), [1, 2, 0]), mats[b], (crop, crop)),
                                              [2, 0, 1]).reshape(3, crop, crop))
            # unmodified reference function; cv2 drops the trailing axis of a 1-channel Mat (crop = 1), hence the reshape
            a = ref._gaussian_blur(a).reshape(3, crop, crop)
            a = TF.normalize(a, MEAN, STD)
            plains.append(p.numpy())
            augs.append(a.numpy())
        for k, v in dict(images=imgs, crop_plain=crop_plain, crop_aug=crop_aug, flip=flip, affine=mats,
                         plain=np.stack(plains), aug=np.stack(augs), crop=np.int32(crop)).items():
            fixture[f"{name}/{k}"] = v
    fixture["cases"] = np.array(names)
    fixture["versions"] = np.array([f"cv2 {cv2.__version__}", f"torch {torch.__version__}"])
    path = os.path.join(HERE, "augment_edges.npz")
    np.savez_compressed(path, **fixture)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
