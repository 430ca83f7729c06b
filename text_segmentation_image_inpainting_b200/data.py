"""Training batches prepared on the GPU from decoded source bytes: the reference's `process_images` for a whole batch.

  * `InpaintBatcher`: `ImageInpaintingData.process_images` (Dataloader.py:110-162), csrc/inpaint_data.cu.
  * `InpaintPairBatcher`: `TestDataset.process_images` (Dataloader.py:165-222), the masks derived from raw/clean page pairs,
    csrc/inpaint_data.cu.
  * `SegBatcher`: `TextSegmentationData.process_images` (Dataloader.py:66-74), csrc/seg_data.cu.

Both share the host side (`_SourceStager`): the host decodes files and calls `stage(samples)`, which copies the uint8 bytes
into pinned memory and uploads them on a copy stream; `prepare()` then runs the parameter sampler (Philox with the seed and
step counter in device memory) and the batcher's kernels.  The output buffers, the descriptor table and the parameters live at
fixed addresses, so the training steps of engine.py capture the whole thing in their CUDA graph; any mix of source sizes
within the capacity replays without recapture.  Source bytes are double buffered: the upload of the next batch overlaps the
current step.

InpaintBatcher and InpaintPairBatcher return the reference's triplet, batched, in the layouts the training step consumes:

  * corrupted: `[n, 3, s, s]` view of an 8-channel-padded NHWC buffer in the compute dtype (TrainStep._prepare's layout),
  * mask:      `HoleMask` over one uint8 plane `[n, s, s]` (1 = valid), 3 channels,
  * clean:     fp32 NCHW `[n, 3, s, s]` (the ToTensor output).

SegBatcher returns (x, target):

  * x:      `[n, 3, s, s]` view of an 8-channel-padded NHWC buffer in the compute dtype: the jittered gray page in all three
            channels (the networks take RGB; for an `L` page this is `to_tensor(page.convert("RGB"))`), optionally normalized,
  * target: fp32 NCHW `[n, 1, s, s]`, the mask's ToTensor (soft: the bicubic resize leaves up to 256 levels).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .masks import HoleMask

PARAM_INTS = 52                 # int32 fields of pcb_inpaint_params
SEG_PARAM_INTS = 8              # int32 fields of pcb_seg_params
_SRC_BYTES = 32                 # sizeof(pcb_inpaint_src), sizeof(pcb_seg_src)
_ALIGN = 256


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _up(v):
    return (v + _ALIGN - 1) // _ALIGN * _ALIGN


class _SourceStager:
    """The host side of a GPU batcher: a pinned double buffer of decoded sources, uploaded on a copy stream, each slot
    beginning with the descriptor table the kernels read (per image: two source pointers, height, width, two row strides).
    Subclasses set `_channels` (bytes per pixel of the two sources) and `_validate` (the C entry point that checks a table)."""

    _channels = (3, 1)
    _validate = "pcb_inpaint_validate"

    def _init_staging(self, seed):
        dev, n = self.device, self.batch
        ca, cb = self._channels
        self._table_bytes = _up(n * _SRC_BYTES)
        self._slot_bytes = self._table_bytes + n * (_up(self.cap_h * self.cap_w * ca) + _up(self.cap_h * self.cap_w * cb))
        self._host = [torch.empty(self._slot_bytes, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self._dev = [torch.empty(self._slot_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
        self._h2d_done = [None, None]       # event: the upload from host slot i finished (host may rewrite it)
        self._consumed = [None, None]       # event: the kernels that read device slot i were enqueued before it
        self._ready = None
        self._slot = 1
        self._host_table = None
        self.table = torch.zeros(self._table_bytes, dtype=torch.uint8, device=dev)       # what the kernels read
        self.rng = torch.tensor([int(seed), 0], dtype=torch.int64, device=dev)
        self._copy = torch.cuda.Stream(device=dev)

    def _check_sample(self, i, a, b):
        raise NotImplementedError

    # ------------------------------------------------------------------------------------------------------------ staging
    def reseed(self, seed: int, counter: int = 0):
        """Restart the device generator: the same seed reproduces the same sequence of parameters."""
        self.rng.copy_(torch.tensor([int(seed), int(counter)], dtype=torch.int64))

    def stage(self, samples):
        """Upload one batch of `batch` decoded source pairs (numpy arrays or CPU tensors; see the subclass).  Returns at once;
        the copy runs on a copy stream while the device works on the previous batch."""
        if len(samples) != self.batch:
            raise ValueError(f"stage() takes {self.batch} samples, got {len(samples)}")
        slot = self._slot ^ 1
        if self._h2d_done[slot] is not None:
            self._h2d_done[slot].synchronize()          # the upload from this pinned buffer two batches ago has finished
        host, base = self._host[slot].numpy(), self._dev[slot].data_ptr()
        ca, cb = self._channels
        table = np.zeros(self.batch, dtype=[("a", "<u8"), ("b", "<u8"), ("h", "<i4"), ("w", "<i4"), ("sa", "<i4"), ("sb", "<i4")])
        off, used = self._table_bytes, self._table_bytes
        for i, (a, b) in enumerate(samples):
            a, b = np.asarray(a), np.asarray(b)
            self._check_sample(i, a, b)
            h, w = b.shape[:2]
            if h > self.cap_h or w > self.cap_w:
                raise ValueError(f"sample {i} is {h}x{w}, capacity {self.cap_h}x{self.cap_w}")
            na, nb = h * w * ca, h * w * cb
            host[off:off + na] = a.reshape(-1)
            host[off + na:off + na + nb] = b.reshape(-1)
            table[i] = (base + off, base + off + na, h, w, ca * w, cb * w)
            off += _up(na + nb)
            used = off
        host[:table.nbytes] = table.view(np.uint8)
        _lib.check(getattr(_lib.load(), self._validate)(table.ctypes.data, None, self.batch, self.batch, self.cap_h, self.cap_w,
                                                        self.size))
        if self._consumed[slot] is not None:
            self._copy.wait_event(self._consumed[slot])     # the kernels that read this device slot two batches ago are done
        with torch.cuda.stream(self._copy):
            self._dev[slot][:used].copy_(self._host[slot][:used], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy)
        self._h2d_done[slot] = self._ready = ev
        self._slot, self._host_table = slot, table

    def activate(self):
        """Order the current stream after the last stage() and point the kernels' table at its slot (eager prepare() and the
        training steps of engine.py call this; it is never captured)."""
        if self._ready is None:
            raise RuntimeError("stage() a batch first")
        cur = torch.cuda.current_stream()
        cur.wait_event(self._ready)
        self.table.copy_(self._dev[self._slot][:self._table_bytes], non_blocking=True)

    def release(self):
        """Mark the staged slot as read by everything enqueued so far on the current stream."""
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self._consumed[self._slot] = ev


class InpaintBatcher(_SourceStager):
    """GPU `process_images` for batches of `batch` images of at most `max_hw = (height, width)` pixels (at most 8x
    `image_size`).  `add_random_masks` draws random_masks' strokes; `seed` seeds the device generator.  `stage(samples)` takes
    `batch` pairs (RGB uint8 [h, w, 3], text mask uint8 [h, w])."""

    _sample, _prepare = "pcb_inpaint_sample", "pcb_inpaint_prepare"
    _TMP_PIXEL_BYTES = 4            # the horizontal pass's intermediate (pcb_inpaint_prepare's tmp)

    def __init__(self, batch: int, max_hw: Tuple[int, int], image_size: int = 512, add_random_masks: bool = True, seed: int = 0,
                 compute_dtype=torch.bfloat16, device=None):
        if compute_dtype not in (torch.bfloat16, torch.float32):
            raise ValueError("compute_dtype must be torch.bfloat16 or torch.float32")
        self.batch, self.cap_h, self.cap_w = int(batch), int(max_hw[0]), int(max_hw[1])
        self.size, self.strokes, self.dtype = int(image_size), bool(add_random_masks), compute_dtype
        if not 1 <= self.batch <= 1024:
            raise ValueError("batch must be 1..1024")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        _lib.load()
        if self.cap_h > 8 * self.size or self.cap_w > 8 * self.size or self.size < 32:
            raise ValueError(f"capacity {max_hw} must be at most 8x the output size {image_size} (>= 32)")
        dev, n, s = self.device, self.batch, self.size
        self._init_staging(seed)
        self.params = torch.zeros((n, PARAM_INTS), dtype=torch.int32, device=dev)
        self._tmp = torch.empty(n * self.cap_h * s * self._TMP_PIXEL_BYTES, dtype=torch.uint8, device=dev)
        self._xbuf = torch.empty((n, 8, s, s), dtype=compute_dtype, device=dev, memory_format=torch.channels_last).zero_()
        self.corrupted = self._xbuf[:, :3]
        self.plane = torch.zeros((n, s, s), dtype=torch.uint8, device=dev)
        self.clean = torch.zeros((n, 3, s, s), dtype=torch.float32, device=dev)

    def _check_sample(self, i, rgb, mask):
        if rgb.dtype != np.uint8 or mask.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3 or mask.shape != rgb.shape[:2]:
            raise ValueError(f"sample {i}: expected uint8 RGB [h, w, 3] and uint8 mask [h, w], got {rgb.shape} {rgb.dtype} / "
                             f"{mask.shape} {mask.dtype}")

    # ------------------------------------------------------------------------------------------------------------ the batch
    def prepare(self, params: Optional[np.ndarray] = None):
        """(corrupted, HoleMask, clean) of the staged batch.  `params` (int32 [batch, 52], the pcb_inpaint_params layout:
        crop box top, left, height, width; grayscale flag; line and ellipse counts; 5 lines x0, y0, x1, y1, width; 5 ellipses
        x0, y0, x1, y1) replaces the device draws, e.g. to replay the reference's own random stream.  The returned tensors are
        the batcher's buffers, overwritten by the next call."""
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            self.activate()
        lib, st = _lib.load(), _stream()
        if params is None:
            _lib.check(getattr(lib, self._sample)(self.table.data_ptr(), self.batch, self.size, int(self.strokes), self.rng.data_ptr(),
                                                  self.params.data_ptr(), st))
        else:
            if capturing:
                raise RuntimeError("explicit parameters cannot be captured; prepare(params) runs eagerly")
            p = np.ascontiguousarray(params, dtype=np.int32)
            if p.shape != (self.batch, PARAM_INTS):
                raise ValueError(f"params must be int32 [{self.batch}, {PARAM_INTS}]")
            _lib.check(getattr(lib, self._validate)(self._host_table.ctypes.data, p.ctypes.data, self.batch, self.batch, self.cap_h,
                                                    self.cap_w, self.size))
            self.params.copy_(torch.from_numpy(p))
        _lib.check(getattr(lib, self._prepare)(self.table.data_ptr(), self.params.data_ptr(), self.batch, self.cap_h, self.cap_w,
                                               self.size, int(self.strokes), self._tmp.data_ptr(), self._xbuf.data_ptr(),
                                               _lib.PCB_BF16 if self.dtype == torch.bfloat16 else _lib.PCB_F32, self.plane.data_ptr(),
                                               self.clean.data_ptr(), st))
        if not capturing:
            self.release()
        return self.corrupted, HoleMask.from_plane(self.plane, 3), self.clean


class InpaintPairBatcher(InpaintBatcher):
    """GPU `TestDataset.process_images` (Dataloader.py:201-222): inpainting batches from raw/clean page pairs, the mask being
    where the two differ.  Both pages are cropped and resized with the one box drawn on raw; their `L` conversions are
    subtracted (ImageChops.difference), the strokes (`add_random_masks`) are drawn at 255 on the difference, and the result is
    thresholded at 0.4 * 255 and dilated 10x10.  There is no grayscale draw.  `prepare()` returns the same triplet as
    InpaintBatcher (`params` rows must have the grayscale flag 0), so the training steps and engine.InpaintEvalStep take
    either batcher.  The device draws the same crop boxes and strokes as an InpaintBatcher with the same seed and counter.

    `stage(samples)` takes `batch` pairs (raw RGB uint8 [h, w, 3], clean RGB uint8 [h, w, 3]) of equal size.  Decoding and
    pairing the files stay with the caller.  Note that `TestDataset.__getitem__` globs `clean/*` and derives the raw path
    with `re.sub("raw", "clean", ...)`, which leaves a path without "raw" in it unchanged, so the reference as written often
    pairs a file with itself (an empty mask).  This batcher takes whatever pair the caller decoded."""

    _channels = (3, 3)
    _validate = "pcb_inpaint_pair_validate"
    _sample, _prepare = "pcb_inpaint_pair_sample", "pcb_inpaint_pair_prepare"
    _TMP_PIXEL_BYTES = 8            # raw RGB0 | clean RGB0

    def _check_sample(self, i, raw, clean):
        if raw.dtype != np.uint8 or clean.dtype != np.uint8 or raw.ndim != 3 or raw.shape[2] != 3 or clean.shape != raw.shape:
            raise ValueError(f"sample {i}: expected a uint8 RGB [h, w, 3] raw page and a clean page of the same shape and dtype, got "
                             f"{raw.shape} {raw.dtype} / {clean.shape} {clean.dtype}")


def seg_params(rows) -> np.ndarray:
    """int32 [n, SEG_PARAM_INTS] parameter rows (the pcb_seg_params layout) for `SegBatcher.prepare(params)` from
    (top, left, height, width, brightness_first, brightness, contrast) tuples, e.g. what the reference's
    RandomResizedCrop.get_params and ColorJitter.get_params returned.  The factors are stored as float32 bit patterns."""
    rows = list(rows)
    p = np.zeros((len(rows), SEG_PARAM_INTS), np.int32)
    for k, (top, left, h, w, bfirst, b, c) in enumerate(rows):
        p[k, :5] = (top, left, h, w, int(bool(bfirst)))
        p[k, 5:7] = np.array([b, c], np.float32).view(np.int32)
    return p


class SegBatcher(_SourceStager):
    """GPU `TextSegmentationData.process_images` for batches of `batch` gray pages of at most `max_hw = (height, width)` pixels
    (at most 8x `image_size`).  `stage(samples)` takes `batch` pairs (page uint8 [h, w], text mask uint8 [h, w]): the files
    decoded and converted to `L` on the host.  `seed` seeds the device generator.

    `normalize=(mean, std)` (three values each) applies torchvision's Normalize to x in fp32 before the store: the input
    convention of the published checkpoints (demo_segmentation.py).  The default None is the reference's data path."""

    _channels = (1, 1)
    _validate = "pcb_seg_validate"

    def __init__(self, batch: int, max_hw: Tuple[int, int], image_size: int = 256, seed: int = 0, compute_dtype=torch.bfloat16,
                 device=None, normalize: Optional[Tuple[Sequence[float], Sequence[float]]] = None):
        if compute_dtype not in (torch.bfloat16, torch.float32):
            raise ValueError("compute_dtype must be torch.bfloat16 or torch.float32")
        self.batch, self.cap_h, self.cap_w = int(batch), int(max_hw[0]), int(max_hw[1])
        self.size, self.dtype = int(image_size), compute_dtype
        if not 1 <= self.batch <= 1024:
            raise ValueError("batch must be 1..1024")
        if self.size < 16 or self.size > 4096 or self.cap_h > 8 * self.size or self.cap_w > 8 * self.size:
            raise ValueError(f"capacity {max_hw} must be at most 8x the output size {image_size} (16..4096)")
        self._norm = None
        if normalize is not None:
            mean, std = (tuple(float(v) for v in t) for t in normalize)
            if len(mean) != 3 or len(std) != 3:
                raise ValueError("normalize takes (mean, std) with three values each")
            self._norm = (ctypes.c_float * 6)(*mean, *std)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        _lib.load()
        dev, n, s = self.device, self.batch, self.size
        self._init_staging(seed)
        self.params = torch.zeros((n, SEG_PARAM_INTS), dtype=torch.int32, device=dev)
        self._tmp = torch.empty(n * self.cap_h * s * 2, dtype=torch.uint8, device=dev)
        self._planes = torch.empty(2 * n * s * s, dtype=torch.uint8, device=dev)
        self._hist = torch.zeros(n * 256, dtype=torch.int32, device=dev)
        self._xbuf = torch.empty((n, 8, s, s), dtype=compute_dtype, device=dev, memory_format=torch.channels_last).zero_()
        self.x = self._xbuf[:, :3]
        self.target = torch.zeros((n, 1, s, s), dtype=torch.float32, device=dev)

    def _check_sample(self, i, page, mask):
        if page.dtype != np.uint8 or mask.dtype != np.uint8 or page.ndim != 2 or mask.shape != page.shape:
            raise ValueError(f"sample {i}: expected uint8 page [h, w] and uint8 mask [h, w], got {page.shape} {page.dtype} / "
                             f"{mask.shape} {mask.dtype}")

    def prepare(self, params: Optional[np.ndarray] = None):
        """(x, target) of the staged batch.  `params` (int32 [batch, 8], see `seg_params`: crop box top, left, height, width;
        brightness-first flag; float32 bits of the brightness and contrast factors) replaces the device draws, e.g. to replay the
        reference's own random stream.  The returned tensors are the batcher's buffers, overwritten by the next call."""
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            self.activate()
        lib, st = _lib.load(), _stream()
        if params is None:
            _lib.check(lib.pcb_seg_sample(self.table.data_ptr(), self.batch, self.rng.data_ptr(), self.params.data_ptr(), st))
        else:
            if capturing:
                raise RuntimeError("explicit parameters cannot be captured; prepare(params) runs eagerly")
            p = np.ascontiguousarray(params, dtype=np.int32)
            if p.shape != (self.batch, SEG_PARAM_INTS):
                raise ValueError(f"params must be int32 [{self.batch}, {SEG_PARAM_INTS}]")
            _lib.check(lib.pcb_seg_validate(self._host_table.ctypes.data, p.ctypes.data, self.batch, self.batch, self.cap_h, self.cap_w,
                                            self.size))
            self.params.copy_(torch.from_numpy(p))
        _lib.check(lib.pcb_seg_prepare(self.table.data_ptr(), self.params.data_ptr(), self.batch, self.cap_h, self.cap_w, self.size,
                                       self._tmp.data_ptr(), self._planes.data_ptr(), self._hist.data_ptr(), self._norm,
                                       self._xbuf.data_ptr(), _lib.PCB_BF16 if self.dtype == torch.bfloat16 else _lib.PCB_F32,
                                       self.target.data_ptr(), st))
        if not capturing:
            self.release()
        return self.x, self.target
