"""CPU oracle for the paired target augmentation (TEST INFRASTRUCTURE, never the product path).

Restates, in numpy, what the reference's two target-domain transform pipelines do to one resized uint8
image (paths relative to /root/reference):

  plain  resnet50_dwt_mec_officehome.py:526-531   RandomCrop -> ToTensor -> Normalize
  aug    resnet50_dwt_mec_officehome.py:534-542   RandomCrop -> RandomHorizontalFlip -> ToTensor ->
         _random_affine_augmentation (:481-487, cv2.warpAffine) -> _gaussian_blur (:489-492) -> Normalize
  both applied to the same image by utils/folder.py:127-147 (`transform`, `transform_aug`).

The random draws are inputs here (crop corner, flip flag, the 2x3 matrix), so the functions are deterministic.

Third-party arithmetic restated (not under /root/reference; versions probed in the build container):
  * OpenCV 4.13.0 `cv2.warpAffine(src, M, dsize)` with its defaults INTER_LINEAR / BORDER_CONSTANT(0) on a
    CV_32FC3 image: M (float32) is widened to double and inverted in double; destination pixel (x, y) samples
    the source at fixed-point coordinates  X = (rint((m1*y + m2)*1024) + 16 + rint(m0*x*1024)) >> 5  (likewise Y),
    integer part X >> 5, fraction (X & 31)/32; the four taps are blended in float32 with weights
    (1-fy)(1-fx), (1-fy)fx, fy(1-fx), fy*fx (products rounded to float32) summed left to right, taps outside
    the image contributing 0.
  * `cv2.GaussianBlur(x, (k, k), sigma)` with k = int(sigma + 0.5)*8 + 1: the reference's sigma = 0.1 gives
    k = 1, a 1x1 kernel -- the identity.  Other sigmas are not restated (ValueError).
  * torchvision 0.26 `to_tensor` (uint8 -> float32 true division by 255), `normalize` ((x - mean) / std),
    `hflip`, `crop`.

Parity pin: tests/golden/augment.npz holds outputs of the unmodified reference functions + torchvision
(tests/golden/make_golden_augment.py); tests/test_oracle_vs_golden.py requires BIT-EXACT agreement.  The same holds
for tests/golden/augment_edges.npz (translations, reflections, singular and zoom matrices, non-square sources, crops
of 1 and of the whole source; tests/test_pool_augment_exact.py).  Crop corners must lie in [0, src - crop]: numpy
slicing would shorten the crop, the GPU kernel clamps the corner, torchvision pads.
"""
from __future__ import annotations

import numpy as np

MEAN = np.float32([0.485, 0.456, 0.406])      # resnet50_dwt_mec_officehome.py:530
STD = np.float32([0.229, 0.224, 0.225])


def invert_affine(m23):
    """cv2.invertAffineTransform as warpAffine applies it internally: float32 [2,3] -> six doubles."""
    M = np.asarray(m23, dtype=np.float32).astype(np.float64).reshape(6)
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    m = np.zeros(6)
    m[0], m[1], m[3], m[4] = A11, M[1] * (-D), M[3] * (-D), A22
    m[2] = -m[0] * M[2] - m[1] * M[5]
    m[5] = -m[3] * M[2] - m[4] * M[5]
    return m


def warp_affine(img, m23):
    """cv2.warpAffine(img, M, (W, H)) for a float32 [H, W, C] image, bit for bit."""
    img = np.asarray(img, dtype=np.float32)
    H, W = img.shape[:2]
    m = invert_affine(m23)
    xs, ys = np.arange(W), np.arange(H)
    adelta = np.rint(m[0] * xs * 1024.0).astype(np.int64)
    bdelta = np.rint(m[3] * xs * 1024.0).astype(np.int64)
    X0 = np.rint((m[1] * ys + m[2]) * 1024.0).astype(np.int64) + 16
    Y0 = np.rint((m[4] * ys + m[5]) * 1024.0).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = X >> 5, Y >> 5
    fx = (X & 31).astype(np.float32) / np.float32(32)
    fy = (Y & 31).astype(np.float32) / np.float32(32)

    def tap(yy, xx):
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        v = img[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        return np.where(ok[..., None], v, np.float32(0))

    one = np.float32(1)
    w00, w01 = ((one - fy) * (one - fx))[..., None], ((one - fy) * fx)[..., None]
    w10, w11 = (fy * (one - fx))[..., None], (fy * fx)[..., None]
    return ((tap(sy, sx) * w00 + tap(sy, sx + 1) * w01) + tap(sy + 1, sx) * w10) + tap(sy + 1, sx + 1) * w11


def gaussian_blur(x, sigma=0.1):
    if int(sigma + 0.5) * 8 + 1 != 1:
        raise ValueError("only the reference's sigma (kernel size 1, the identity) is restated")
    return x


def to_tensor_normalize(hwc_float, mean=MEAN, std=STD):
    """[H,W,3] float32 in [0,1] -> normalised [3,H,W]."""
    return np.transpose((hwc_float - mean) / std, (2, 0, 1)).astype(np.float32)


def plain_view(img_u8, top, left, crop, mean=MEAN, std=STD):
    """The un-augmented view: crop -> /255 -> normalise.  img_u8: [H,W,3] uint8 (already resized)."""
    c = img_u8[top:top + crop, left:left + crop].astype(np.float32) / np.float32(255)
    return to_tensor_normalize(c, mean, std)


def aug_view(img_u8, top, left, crop, flip, m23, mean=MEAN, std=STD):
    """The augmented view: crop -> (flip) -> /255 -> affine warp -> blur (identity) -> normalise."""
    c = img_u8[top:top + crop, left:left + crop]
    if flip:
        c = c[:, ::-1]
    f = c.astype(np.float32) / np.float32(255)
    return to_tensor_normalize(gaussian_blur(warp_affine(f, m23)), mean, std)


def paired(images_u8, crop_plain, crop_aug, flip, affine, crop, mean=MEAN, std=STD):
    """Batch form used by the tests: images [B,H,W,3] uint8 -> (plain [B,3,c,c], aug [B,3,c,c])."""
    p = np.stack([plain_view(im, int(cp[0]), int(cp[1]), crop, mean, std) for im, cp in zip(images_u8, crop_plain)])
    a = np.stack([aug_view(im, int(ca[0]), int(ca[1]), crop, bool(f), m, mean, std)
                  for im, ca, f, m in zip(images_u8, crop_aug, flip, affine)])
    return p, a
