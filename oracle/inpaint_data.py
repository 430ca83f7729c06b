"""numpy restatement of the inpainting data path (`ImageInpaintingData.process_images`, Dataloader.py:110-132) that
`csrc/inpaint_data.cu` implements.  Tests pin it bit-exactly against the reference's own code (PIL, cv2, torchvision) and pin
the kernels bit-exactly against it.

Parameters of one image (int32, `PARAM_INTS` per image, the layout of `pcb_inpaint_params`):
  [0:4]  crop box top, left, height, width (RandomResizedCrop.get_params: i, j, h, w)
  [4]    grayscale flag
  [5]    number of lines, [6] number of ellipses
  [7:32] 5 lines  x0, y0, x1, y1, width
  [32:52] 5 ellipses x0, y0, x1, y1 (ImageDraw.ellipse's box, both corners inclusive)
"""
import numpy as np

PARAM_INTS = 52
PB = 22                                     # Pillow's PRECISION_BITS for 8-bit images
MAX_STROKES = 5
LINE0, ELL0 = 7, 32
# float32 log of (3/4, 4/3) as torch.log(torch.tensor(ratio)) computes it, and their float32 difference
LOG_RATIO0, LOG_RATIO1, LOG_RATIO_SPAN = np.float32(-0.28768208622932434), np.float32(0.28768211603164673), np.float32(0.5753642320632935)
NSLOTS = 88                                 # uniform draws per image (philox groups of 4)


# ------------------------------------------------------------------------------------------------------- crop + resize
def _cubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(insize, outsize):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for box (0, insize): list of (first tap, int weights)."""
    scale = insize / outsize
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ss = 1.0 / fs
    out = []
    for xx in range(outsize):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), insize) - xmin
        k = [_cubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = sum(k)
        k = [v / ww if ww != 0.0 else v for v in k]
        out.append((xmin, [int(-0.5 + v * (1 << PB)) if v < 0 else int(0.5 + v * (1 << PB)) for v in k]))
    return out


def _pass(img, cs):
    """Resample axis 1 of img [A, B, C] uint8 with coefficient list cs -> [A, len(cs), C] uint8."""
    o = np.empty((img.shape[0], len(cs), img.shape[2]), np.uint8)
    for xx, (xmin, kk) in enumerate(cs):
        acc = np.full((img.shape[0], img.shape[2]), 1 << (PB - 1), np.int64)
        for t, k in enumerate(kk):
            acc += img[:, xmin + t, :].astype(np.int64) * k
        o[:, xx, :] = np.clip(acc >> PB, 0, 255)
    return o


def resized_crop(img, box, out):
    """PIL `img.crop((j, i, j+w, i+h)).resize((out, out), BICUBIC)` for img [H, W, C] uint8: horizontal pass over every row
    of the box, uint8 intermediate, then the vertical pass."""
    i, j, h, w = box
    crop = img[i:i + h, j:j + w]
    t = _pass(crop, coeffs(w, out))                       # [h, out, C]
    return _pass(t.transpose(1, 0, 2), coeffs(h, out)).transpose(1, 0, 2)


# ------------------------------------------------------------------------------------------------------- per-pixel steps
def grayscale(rgb):
    """PIL convert('L') replicated to 3 channels (torchvision rgb_to_grayscale on PIL input)."""
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    l = ((19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16).astype(np.uint8)
    return np.repeat(l[..., None], 3, axis=2)


def dilate10(hole):
    """cv2.dilate(., ones(10, 10)) of a boolean map: max over rows y-5..y+4 and columns x-5..x+4, outside pixels ignored."""
    H, W = hole.shape
    p = np.zeros((H + 9, W + 9), bool)
    p[5:5 + H, 5:5 + W] = hole
    r = np.zeros((H + 9, W), bool)
    for d in range(10):
        r |= p[:, d:d + W]
    o = np.zeros((H, W), bool)
    for d in range(10):
        o |= r[d:d + H]
    return o


def ellipse_px(size, x0, y0, x1, y1):
    """Stroke rule for ImageDraw.ellipse([x0, y0, x1, y1]): the pixel centre lies inside the ellipse inscribed in
    [x0, x1+1) x [y0, y1+1).  Integer form: (2x - x0 - x1)^2 B^2 + (2y - y0 - y1)^2 A^2 <= A^2 B^2, A = x1-x0+1, B = y1-y0+1."""
    yy, xx = np.mgrid[0:size, 0:size].astype(np.int64)
    A, B = x1 - x0 + 1, y1 - y0 + 1
    dx, dy = 2 * xx - x0 - x1, 2 * yy - y0 - y1
    return dx * dx * B * B + dy * dy * A * A <= A * A * B * B


def line_px(size, x0, y0, x1, y1, w):
    """Stroke rule for ImageDraw.line([x0, y0, x1, y1], width=w): the pixel (integer coordinates) lies in the butt-capped
    rectangle of width w around the segment: 0 <= <p-p0, d> <= |d|^2 and 4 cross(p-p0, d)^2 <= w^2 |d|^2.  A zero-length line
    is the single pixel (x0, y0), as Pillow draws it."""
    yy, xx = np.mgrid[0:size, 0:size].astype(np.int64)
    dx, dy = x1 - x0, y1 - y0
    if dx == 0 and dy == 0:
        return (xx == x0) & (yy == y0)
    L2 = dx * dx + dy * dy
    dot = (xx - x0) * dx + (yy - y0) * dy
    cr = (xx - x0) * dy - (yy - y0) * dx
    return (dot >= 0) & (dot <= L2) & (4 * cr * cr <= w * w * L2)


def strokes_px(size, p):
    m = np.zeros((size, size), bool)
    for k in range(int(p[5])):
        m |= line_px(size, *(int(v) for v in p[LINE0 + 5 * k:LINE0 + 5 * k + 5]))
    for k in range(int(p[6])):
        m |= ellipse_px(size, *(int(v) for v in p[ELL0 + 4 * k:ELL0 + 4 * k + 4]))
    return m


def process(rgb, mask, p, out, strokes=True):
    """One image: (clean uint8 [out, out, 3] after the grayscale draw, hole bool [out, out] after the dilation).
    The reference's tensors are clean/255.f (fp32), binary = 1 - 255*hole/255.f, corrupted = clean * binary."""
    box = [int(v) for v in p[:4]]
    clean = resized_crop(rgb, box, out)
    if p[4]:
        clean = grayscale(clean)
    m = resized_crop(mask[..., None], box, out)[..., 0]
    hole = m >= 103                                          # mask > 0.4 * 255
    if strokes:
        hole |= strokes_px(out, p)                           # drawn at 255 before the threshold
    return clean, dilate10(hole)


def to_tensors(clean_u8, hole):
    """ToTensor and the masking of Dataloader.py:124-131: (corrupted, binary, clean) fp32 CHW."""
    clean = np.transpose(clean_u8, (2, 0, 1)).astype(np.float32) / np.float32(255)
    m = hole.astype(np.float32) * np.float32(255) / np.float32(255)
    binary = np.float32(1) - m
    return clean * binary[None], np.repeat(binary[None], 3, 0), clean


# ------------------------------------------------------------------------------------------------------- sampler
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_U32 = np.uint64(0xFFFFFFFF)


def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint64 arrays holding 32-bit values."""
    c = [np.asarray(v, np.uint64) & _U32 for v in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & _U32, np.uint64(k1) & _U32
    for r in range(10):
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & _U32, p1 & _U32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & _U32, p0 & _U32]
        if r < 9:
            k0, k1 = (k0 + np.uint64(_W0)) & _U32, (k1 + np.uint64(_W1)) & _U32
    return c


def uniforms(seed, counter, n):
    """[n, NSLOTS] float32 uniforms in [0, 1) (24 bits) of images 0..n-1 at step `counter`: philox counter = (group, image,
    counter lo, counter hi), key = (seed lo, seed hi)."""
    g, img = np.meshgrid(np.arange(NSLOTS // 4, dtype=np.uint64), np.arange(n, dtype=np.uint64))
    words = philox(g, img, counter & 0xFFFFFFFF, counter >> 32, seed & 0xFFFFFFFF, seed >> 32)
    u = np.stack(words, -1).reshape(n, NSLOTS)                # slot 4 * group + lane
    return (u >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)


def _randint(u, lo, hi):
    """lo..hi inclusive (random.randint / torch.randint(lo, hi + 1)) from one uniform."""
    return lo + int(np.float64(u) * (hi - lo + 1))


def crop_from_uniforms(H, W, u):
    """RandomResizedCrop.get_params(scale=(0.5, 2.0), ratio=(3/4, 4/3)) with its draws taken from u[0:40]: per attempt a the
    scale value 0.5 + 1.5 u[4a], the log-aspect value LOG_RATIO0 + span u[4a+1] (float32, as torch draws them) and the
    top / left offsets from u[4a+2], u[4a+3]."""
    area = H * W
    for a in range(10):
        s = np.float32(0.5) + np.float32(1.5) * np.float32(u[4 * a])
        r = LOG_RATIO0 + LOG_RATIO_SPAN * np.float32(u[4 * a + 1])
        target = area * float(s)
        aspect = float(np.float32(np.exp(np.float64(r))))
        w = int(np.rint(np.sqrt(target * aspect)))
        h = int(np.rint(np.sqrt(target / aspect)))
        if 0 < w <= W and 0 < h <= H:
            return _randint(u[4 * a + 2], 0, H - h), _randint(u[4 * a + 3], 0, W - w), h, w
    in_ratio = float(W) / float(H)
    if in_ratio < 0.75:
        w, h = W, int(np.rint(W / 0.75))
    elif in_ratio > 4.0 / 3.0:
        h, w = H, int(np.rint(H * (4.0 / 3.0)))
    else:
        w, h = W, H
    return (H - h) // 2, (W - w) // 2, h, w


def strokes_from_uniforms(size, u, p):
    """random_masks(size, offset=10) (Dataloader.py:142-162) with its draws taken from u[41:88], written into p."""
    off = 10
    p[5] = _randint(u[41], 1, 5)
    for k in range(MAX_STROKES):
        b = 42 + 5 * k
        x0, y0, x1, y1 = (_randint(u[b + t], off, size - 1) for t in range(4))
        x1 = min(max(x1, x0 - 75), x0 + 75)
        y1 = min(max(y1, y0 - 75), y0 + 75)
        p[LINE0 + 5 * k:LINE0 + 5 * k + 5] = (x0, y0, x1, y1, _randint(u[b + 4], 15, 20)) if k < p[5] else 0
    p[6] = _randint(u[67], 1, 5)
    for k in range(MAX_STROKES):
        b = 68 + 4 * k
        c0, c1 = sorted(_randint(u[b + t], off, size - off - 1) for t in range(2))
        e0 = min(max(c0 + _randint(u[b + 2], 20, 69), off), size - off)
        e1 = min(max(c1 + _randint(u[b + 3], 20, 69), off), size - off)
        p[ELL0 + 4 * k:ELL0 + 4 * k + 4] = (c0, c1, e0, e1) if k < p[6] else 0


def params_from_uniforms(H, W, size, u, strokes=True):
    p = np.zeros(PARAM_INTS, np.int32)
    p[0:4] = crop_from_uniforms(H, W, u)
    p[4] = int(np.float64(u[40]) < 0.4)                  # RandomGrayscale(p=0.4): torch.rand(1) < p
    if strokes:
        strokes_from_uniforms(size, u, p)
    return p


def sample(seed, counter, sizes, size, strokes=True):
    """What the device sampler draws for images of `sizes` [(H, W), ...] at step `counter`."""
    u = uniforms(seed, counter, len(sizes))
    return np.stack([params_from_uniforms(H, W, size, u[k], strokes) for k, (H, W) in enumerate(sizes)])
