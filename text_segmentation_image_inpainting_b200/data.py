"""Inpainting training batches prepared on the GPU: `ImageInpaintingData.process_images` (Dataloader.py:110-162) for a batch.

The host decodes files and calls `stage(samples)`, which copies the uint8 bytes into pinned memory and uploads them on a copy
stream; `prepare()` then runs csrc/inpaint_data.cu: the parameter sampler (crop box, grayscale draw, strokes from Philox with
the seed and step counter in device memory), Pillow's bicubic crop + resize of image and text mask, strokes, threshold, 10x10
dilation, ToTensor and the masking.  It returns the reference's triplet, batched, in the layouts the training step consumes:

  * corrupted: `[n, 3, s, s]` view of an 8-channel-padded NHWC buffer in the compute dtype (TrainStep._prepare's layout),
  * mask:      `HoleMask` over one uint8 plane `[n, s, s]` (1 = valid), 3 channels,
  * clean:     fp32 NCHW `[n, 3, s, s]` (the ToTensor output).

The output buffers, the descriptor table and the parameters live at fixed addresses, so `engine.InpaintTrainStep` captures the
whole thing in its CUDA graph; any mix of source sizes within the capacity replays without recapture.  Source bytes are double
buffered: the upload of the next batch overlaps the current step.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .masks import HoleMask

PARAM_INTS = 52                 # int32 fields of pcb_inpaint_params
_SRC_BYTES = 32                 # sizeof(pcb_inpaint_src)
_ALIGN = 256


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _up(v):
    return (v + _ALIGN - 1) // _ALIGN * _ALIGN


class InpaintBatcher:
    """GPU `process_images` for batches of `batch` images of at most `max_hw = (height, width)` pixels (at most 8x
    `image_size`).  `add_random_masks` draws random_masks' strokes; `seed` seeds the device generator."""

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
        self._table_bytes = _up(n * _SRC_BYTES)
        self._slot_bytes = self._table_bytes + n * (_up(self.cap_h * self.cap_w * 3) + _up(self.cap_h * self.cap_w))
        self._host = [torch.empty(self._slot_bytes, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self._dev = [torch.empty(self._slot_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
        self._h2d_done = [None, None]       # event: the upload from host slot i finished (host may rewrite it)
        self._consumed = [None, None]       # event: the kernels that read device slot i were enqueued before it
        self._ready = None
        self._slot = 1
        self._host_table = None
        self.table = torch.zeros(self._table_bytes, dtype=torch.uint8, device=dev)       # what the kernels read
        self.rng = torch.tensor([int(seed), 0], dtype=torch.int64, device=dev)
        self.params = torch.zeros((n, PARAM_INTS), dtype=torch.int32, device=dev)
        self._tmp = torch.empty(n * self.cap_h * s * 4, dtype=torch.uint8, device=dev)
        self._xbuf = torch.empty((n, 8, s, s), dtype=compute_dtype, device=dev, memory_format=torch.channels_last).zero_()
        self.corrupted = self._xbuf[:, :3]
        self.plane = torch.zeros((n, s, s), dtype=torch.uint8, device=dev)
        self.clean = torch.zeros((n, 3, s, s), dtype=torch.float32, device=dev)
        self._copy = torch.cuda.Stream(device=dev)

    # ------------------------------------------------------------------------------------------------------------ staging
    def reseed(self, seed: int, counter: int = 0):
        """Restart the device generator: the same seed reproduces the same sequence of parameters."""
        self.rng.copy_(torch.tensor([int(seed), int(counter)], dtype=torch.int64))

    def stage(self, samples: Sequence[Tuple[np.ndarray, np.ndarray]]):
        """Upload one batch: `batch` pairs (RGB uint8 [h, w, 3], text mask uint8 [h, w]) of decoded sources (numpy arrays or CPU
        tensors).  Returns at once; the copy runs on a copy stream while the device works on the previous batch."""
        if len(samples) != self.batch:
            raise ValueError(f"stage() takes {self.batch} samples, got {len(samples)}")
        slot = self._slot ^ 1
        if self._h2d_done[slot] is not None:
            self._h2d_done[slot].synchronize()          # the upload from this pinned buffer two batches ago has finished
        host, base = self._host[slot].numpy(), self._dev[slot].data_ptr()
        table = np.zeros(self.batch, dtype=[("rgb", "<u8"), ("mask", "<u8"), ("h", "<i4"), ("w", "<i4"), ("rs", "<i4"), ("ms", "<i4")])
        off, used = self._table_bytes, self._table_bytes
        for i, (rgb, mask) in enumerate(samples):
            rgb, mask = np.asarray(rgb), np.asarray(mask)
            if rgb.dtype != np.uint8 or mask.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3 or mask.shape != rgb.shape[:2]:
                raise ValueError(f"sample {i}: expected uint8 RGB [h, w, 3] and uint8 mask [h, w], got {rgb.shape} {rgb.dtype} / "
                                 f"{mask.shape} {mask.dtype}")
            h, w = mask.shape
            if h > self.cap_h or w > self.cap_w:
                raise ValueError(f"sample {i} is {h}x{w}, capacity {self.cap_h}x{self.cap_w}")
            nb = h * w * 3
            host[off:off + nb] = rgb.reshape(-1)
            host[off + nb:off + nb + h * w] = mask.reshape(-1)
            table[i] = (base + off, base + off + nb, h, w, 3 * w, w)
            off += _up(nb + h * w)
            used = off
        host[:table.nbytes] = table.view(np.uint8)
        _lib.check(_lib.load().pcb_inpaint_validate(table.ctypes.data, None, self.batch, self.batch, self.cap_h, self.cap_w, self.size))
        if self._consumed[slot] is not None:
            self._copy.wait_event(self._consumed[slot])     # the kernels that read this device slot two batches ago are done
        with torch.cuda.stream(self._copy):
            self._dev[slot][:used].copy_(self._host[slot][:used], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy)
        self._h2d_done[slot] = self._ready = ev
        self._slot, self._host_table = slot, table

    def activate(self):
        """Order the current stream after the last stage() and point the kernels' table at its slot (eager prepare() and
        engine.InpaintTrainStep call this; it is never captured)."""
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
            _lib.check(lib.pcb_inpaint_sample(self.table.data_ptr(), self.batch, self.size, int(self.strokes), self.rng.data_ptr(),
                                              self.params.data_ptr(), st))
        else:
            if capturing:
                raise RuntimeError("explicit parameters cannot be captured; prepare(params) runs eagerly")
            p = np.ascontiguousarray(params, dtype=np.int32)
            if p.shape != (self.batch, PARAM_INTS):
                raise ValueError(f"params must be int32 [{self.batch}, {PARAM_INTS}]")
            _lib.check(lib.pcb_inpaint_validate(self._host_table.ctypes.data, p.ctypes.data, self.batch, self.batch, self.cap_h,
                                                self.cap_w, self.size))
            self.params.copy_(torch.from_numpy(p))
        _lib.check(lib.pcb_inpaint_prepare(self.table.data_ptr(), self.params.data_ptr(), self.batch, self.cap_h, self.cap_w, self.size,
                                           int(self.strokes), self._tmp.data_ptr(), self._xbuf.data_ptr(),
                                           _lib.PCB_BF16 if self.dtype == torch.bfloat16 else _lib.PCB_F32, self.plane.data_ptr(),
                                           self.clean.data_ptr(), st))
        if not capturing:
            self.release()
        # a new view object per call: the layers tag an input plane with the event that made it ready (ops._pconv_launch), and
        # this plane is rewritten in place by every call
        return self.corrupted, HoleMask.from_plane(self.plane.view(self.plane.shape), 3), self.clean
