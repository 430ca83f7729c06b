"""numpy restatement of the segmentation data path (`TextSegmentationData.process_images`, Dataloader.py:66-74) that
`csrc/seg_data.cu` implements.  Tests pin it bit-exactly against the reference's own code (Pillow, torchvision) and pin the
kernels bit-exactly against it.

Parameters of one image (int32, `PARAM_INTS` per image, the layout of `pcb_seg_params`):
  [0:4]  crop box top, left, height, width (RandomResizedCrop.get_params: i, j, h, w)
  [4]    1 when ColorJitter applies brightness before contrast (their relative order in torch.randperm(4))
  [5:7]  float32 bits of the brightness and contrast factors
  [7]    unused (0)
On an `L` image ColorJitter's saturation (a blend of the image with itself) and hue (returns the image) are the identity, so
only brightness and contrast act.
"""
import numpy as np

from oracle import inpaint_data as OI

PARAM_INTS = 8
SCALE = (0.1, 2.0)                          # RandomResizedCrop.get_params(scale=...) of process_images
JITTER = (0.8, 1.2)                         # ColorJitter(brightness=0.2, contrast=0.2): 1 -/+ 0.2


def params_row(box, brightness_first, b, c):
    p = np.zeros(PARAM_INTS, np.int32)
    p[0:4] = box
    p[4] = int(bool(brightness_first))
    p[5:7] = np.array([b, c], np.float32).view(np.int32)
    return p


def factors(p):
    """(brightness, contrast) float32 of a parameter row."""
    b, c = np.asarray(p[5:7], np.int32).view(np.float32)
    return np.float32(b), np.float32(c)


# ------------------------------------------------------------------------------------------------------- ColorJitter on L
def blend(d, x, f):
    """Pillow's Image.blend(degenerate d, image x, f) on 8-bit values: float32 d + f * (x - d) (two roundings, no FMA),
    truncated and clipped to [0, 255]."""
    x = np.asarray(x, np.int64)
    t = np.float32(d) + np.float32(f) * (x - d).astype(np.float32)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.trunc(t))).astype(np.uint8)


def contrast_mean(img):
    """ImageEnhance.Contrast's degenerate level: int(ImageStat mean + 0.5), the mean an exact integer sum over the count."""
    return int(int(np.asarray(img, np.int64).sum()) / img.size + 0.5)


def jitter(page, brightness_first, b, c):
    """ColorJitter(0.2, 0.2, 0.2, 0.2) of an `L` image with the drawn order and factors: adjust_brightness = blend(0, img, b),
    adjust_contrast = blend(int(mean + 0.5), img, c)."""
    if brightness_first:
        page = blend(0, page, b)
        return blend(contrast_mean(page), page, c)
    page = blend(contrast_mean(page), page, c)
    return blend(0, page, b)


def process(page, mask, p, out):
    """One image: (jittered page uint8 [out, out], resized mask uint8 [out, out]).  The reference's tensors are their
    to_tensor (value / 255.f, fp32 [1, out, out])."""
    box = [int(v) for v in p[:4]]
    pg = OI.resized_crop(page[..., None], box, out)[..., 0]
    m = OI.resized_crop(mask[..., None], box, out)[..., 0]
    b, c = factors(p)
    return jitter(pg, int(p[4]), b, c), m


def to_tensor(u8):
    return u8.astype(np.float32)[None] / np.float32(255)


# ------------------------------------------------------------------------------------------------------- sampler
def crop_from_uniforms(H, W, u, scale=SCALE):
    """RandomResizedCrop.get_params(scale, ratio=(3/4, 4/3)) with its draws taken from u[0:40]: per attempt a the scale value
    lo + (hi - lo) u[4a] in float32 (as torch's uniform_ works with float32 bounds), the log-aspect value from u[4a+1] and the
    top / left offsets from u[4a+2], u[4a+3]; the centre-crop fallback when no attempt fits."""
    lo = np.float32(scale[0])
    span = np.float32(np.float32(scale[1]) - lo)
    area = H * W
    for a in range(10):
        s = lo + span * np.float32(u[4 * a])
        r = OI.LOG_RATIO0 + OI.LOG_RATIO_SPAN * np.float32(u[4 * a + 1])
        target = area * float(s)
        aspect = float(np.float32(np.exp(np.float64(r))))
        w = int(np.rint(np.sqrt(target * aspect)))
        h = int(np.rint(np.sqrt(target / aspect)))
        if 0 < w <= W and 0 < h <= H:
            return OI._randint(u[4 * a + 2], 0, H - h), OI._randint(u[4 * a + 3], 0, W - w), h, w
    in_ratio = float(W) / float(H)
    if in_ratio < 0.75:
        w, h = W, int(np.rint(W / 0.75))
    elif in_ratio > 4.0 / 3.0:
        h, w = H, int(np.rint(H * (4.0 / 3.0)))
    else:
        w, h = W, H
    return (H - h) // 2, (W - w) // 2, h, w


def jitter_from_uniforms(u):
    """(brightness_first, b, c) from u[40:43]: the order flag u[40] < 0.5, the factors lo + (hi - lo) u in float32."""
    lo = np.float32(JITTER[0])
    span = np.float32(np.float32(JITTER[1]) - lo)
    return int(np.float32(u[40]) < np.float32(0.5)), lo + span * np.float32(u[41]), lo + span * np.float32(u[42])


def params_from_uniforms(H, W, u):
    return params_row(crop_from_uniforms(H, W, u), *jitter_from_uniforms(u))


def sample(seed, counter, sizes):
    """What the device sampler draws for images of `sizes` [(H, W), ...] at step `counter`."""
    u = OI.uniforms(seed, counter, len(sizes))
    return np.stack([params_from_uniforms(H, W, u[k]) for k, (H, W) in enumerate(sizes)])
