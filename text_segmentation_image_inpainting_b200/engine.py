"""Training-step engine for the partial-conv U-Nets: flat fp32 parameter / gradient arenas, one fused SGD
launch, optional data-parallel gradient all-reduce (NCCL over NVLink) and whole-step CUDA-graph capture.
Inference engines (InferStep, SegInferStep): graph-captured eval-mode forward with the BatchNorm + activation passes fused
into the convolution epilogues.  InpaintEvalStep: held-out evaluation of an inpainting U-Net on a GPU batcher, loss included,
in one graph that coexists with a captured training step on the same network; SegEvalStep: the same for a segmentation network,
with its loss and the pixel average precision (metrics.PixelAveragePrecision) in the graph.  TextRemovalStep: text removal from
pages in one graph -- segmentation, the demo's mask, the dilated holes, inpainting and the composite.

The reference has no train script (SURVEY 3): its recipe is prose -- SGD + Nesterov momentum, weight decay,
cyclic LR (checkpoints/ReadME.md:4).  One step here = forward + loss + backward (+ all-reduce) + SGD update,
the unit BASELINE.json's images/sec is quoted on.  `TrainStep(..., lr_schedule=CyclicLR(...))` runs the recipe's schedule on
the device, inside the captured step; `TrainStep.state_dict()` / `load_state_dict()` save and resume a run.
"""
from __future__ import annotations

import contextlib
import copy
import math
import numbers
import os
from collections import OrderedDict
from typing import List, Optional

import torch

from . import _lib, ops
from .masks import HoleMask

CL = torch.channels_last


def _flat_view(flat: torch.Tensor, off: int, like: torch.Tensor) -> torch.Tensor:
    """A view into `flat` with the same logical shape AND physical element order as `like`."""
    n = like.numel()
    seg = flat[off:off + n]
    if like.dim() == 4 and like.is_contiguous(memory_format=CL) and not like.is_contiguous():
        co, ci, kh, kw = like.shape
        return seg.view(co, kh, kw, ci).permute(0, 3, 1, 2)
    return seg.view(like.shape)


class FlatParams:
    """All trainable parameters of a module re-pointed into one fp32 arena (and their grads into another).

    `retrainable` (a module or parameters of `module`): parameters that get a slot even while frozen, so that their storage moves
    once, here, and a later `set_trainable()` can train them without moving anything.  `params` lists every slot in
    `module.parameters()` order; `ranges` the [start, end) arena runs of the slots that are trainable now."""

    def __init__(self, module: torch.nn.Module, retrainable=None):
        if retrainable is None:
            self.params: List[torch.nn.Parameter] = [p for p in module.parameters() if p.requires_grad]
        else:
            every = list(module.parameters())
            extra = {id(p) for p in (retrainable.parameters() if isinstance(retrainable, torch.nn.Module) else retrainable)}
            if not extra <= {id(p) for p in every}:
                raise ValueError("retrainable: every parameter must belong to the network")
            self.params = [p for p in every if p.requires_grad or id(p) in extra]
        dev = self.params[0].device
        total = sum(p.numel() for p in self.params)
        # pad every tensor to a multiple of 4 elements so all views stay 16-byte aligned
        self.offsets = []
        off = 0
        for p in self.params:
            self.offsets.append(off)
            off += (p.numel() + 3) // 4 * 4
        self.numel = off
        self.flat_p = torch.zeros(off, dtype=torch.float32, device=dev)
        self.flat_g = torch.zeros(off, dtype=torch.float32, device=dev)
        self.flat_m = torch.zeros(off, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for p, o in zip(self.params, self.offsets):
                v = _flat_view(self.flat_p, o, p.data)
                v.copy_(p.data)
                p.data = v
                p.grad = _flat_view(self.flat_g, o, p.data)
        self.true_numel = total
        self._sink_made = {}            # slot -> its GradSink, kept across set_trainable() calls
        self.set_trainable()

    def set_trainable(self):
        """Gradient sinks and SGD ranges over the slots whose parameter requires a gradient now."""
        # Gradient sinks (ops.GradSink): the weight-gradient kernels (4-D convolution weights) and the BatchNorm backward
        # (1-D scale / shift) write straight into the arena -- no gradient tensor, no autograd accumulation kernel.
        self.sinks = []
        self.sink_of = {}
        self.ranges = []                # [start, end) arena runs of consecutive trainable slots
        for i, p in enumerate(self.params):
            if not p.requires_grad:
                p.__dict__.pop("_pcb_grad_sink", None)
                continue
            end = self.offsets[i + 1] if i + 1 < len(self.params) else self.numel
            if self.ranges and self.ranges[-1][1] == self.offsets[i]:
                self.ranges[-1][1] = end
            else:
                self.ranges.append([self.offsets[i], end])
            ok4 = p.dim() == 4 and p.grad.is_contiguous(memory_format=CL) and (p.grad.data_ptr() % 16) == 0
            ok1 = p.dim() == 1
            if ok4 or ok1:
                if i not in self._sink_made:
                    self._sink_made[i] = ops.GradSink(p.grad)
                    self._sink_made[i].prezeroed = True  # TrainStep zeroes the whole gradient arena at the start of every step
                p._pcb_grad_sink = self._sink_made[i]
                self.sinks.append(p._pcb_grad_sink)
                self.sink_of[i] = p._pcb_grad_sink


class CyclicLR:
    """The reference's cyclical learning rate (models/utils/cls.py, `CyclicLR`) as a TrainStep schedule: the same arguments and
    defaults, without the optimizer.  The rate is computed on the device at every update (ops.lr_cyclic), so a captured step
    follows it.  Modes: "triangular", "triangular2" (amplitude halved every cycle), "exp_range" (amplitude times
    gamma ** iteration).  A custom `scale_fn` cannot run on the device and is refused.

    `last_batch_iteration=k` resumes as the reference documents: the first update runs iteration k + 1."""

    MODES = {"triangular": _lib.CLR_TRIANGULAR, "triangular2": _lib.CLR_TRIANGULAR2, "exp_range": _lib.CLR_EXP_RANGE}

    def __init__(self, base_lr=1e-3, max_lr=6e-3, step_size=2000, mode="triangular", gamma=1.0, scale_fn=None,
                 scale_mode="cycle", last_batch_iteration=-1):
        if scale_fn is not None:
            raise ValueError("CyclicLR: a custom scale_fn cannot run on the device; use mode='triangular', 'triangular2' or "
                             "'exp_range'")
        if mode not in self.MODES:
            raise ValueError(f"CyclicLR: mode must be one of {sorted(self.MODES)}, got {mode!r}")
        for name, v in (("base_lr", base_lr), ("max_lr", max_lr), ("step_size", step_size), ("gamma", gamma)):
            if not isinstance(v, numbers.Real) or isinstance(v, bool) or not math.isfinite(v):
                raise ValueError(f"CyclicLR: {name} must be a finite real number (one parameter group), got {v!r}")
        if step_size <= 0:
            raise ValueError(f"CyclicLR: step_size must be positive, got {step_size!r}")
        if not isinstance(last_batch_iteration, numbers.Integral) or isinstance(last_batch_iteration, bool) or last_batch_iteration < -1:
            raise ValueError(f"CyclicLR: last_batch_iteration must be an integer >= -1, got {last_batch_iteration!r}")
        self.base_lr, self.max_lr, self.step_size = float(base_lr), float(max_lr), step_size
        self.mode, self.gamma, self.last_batch_iteration = mode, float(gamma), int(last_batch_iteration)

    def rate(self, iteration: int) -> float:
        """The rate of `iteration` on the host, in the reference's fp64 order (the device computes the same)."""
        step = float(self.step_size)
        cycle = math.floor(1 + iteration / (2 * step))
        x = abs(iteration / step - 2 * cycle + 1)
        height = (self.max_lr - self.base_lr) * max(0.0, 1 - x)
        if self.mode == "triangular2":
            scale = 0.0 if cycle - 1 > 1023 else 1 / (2.0 ** (cycle - 1))
        elif self.mode == "exp_range":
            scale = self.gamma ** iteration
        else:
            scale = 1.0
        return self.base_lr + height * scale


class TrainStep:
    """One training step: forward, loss, backward, (data parallel: gradient all-reduce,) SGD with momentum, Nesterov and weight
    decay, captured in one CUDA graph by `warmup_and_capture()`.

    Learning rate: the constant `lr`, or with `lr_schedule=CyclicLR(...)` a rate computed on the device before every update
    (the counter and the rate live in device memory, so each graph replay advances the schedule; `lr` is then unused and
    assigning it raises).  Every update counts, the eager warm-up updates of `warmup_and_capture()` included.
    `iteration` is the schedule iteration the next update runs, `last_lr` the rate of the last one (device fp64 scalar).

    Checkpoints: `state_dict()` / `load_state_dict()` save and restore the parameters, module buffers, momentum, schedule counter
    and the batcher's generator; see there.

    Frozen parameters (`requires_grad` False) are never updated: no weight decay, no momentum, as torch.optim.SGD leaves a
    parameter without a gradient.  Their BatchNorm layers keep training mode and running statistics, and their operand buffers
    are laid out once instead of at every step.  `retrainable` (a module or parameters of `net`) opts in to training in stages
    on one step: those parameters get an arena slot even while frozen; after changing `requires_grad` (e.g.
    ``net.encoder.requires_grad_(True)``), `update_trainable()` switches the step over in place."""

    def __init__(self, net: torch.nn.Module, compute_dtype=torch.bfloat16, lr=2e-4, momentum=0.9, weight_decay=1e-4,
                 nesterov=True, process_group=None, use_graph=True, bucket_mb=32, overlap_allreduce=None,
                 lr_schedule: Optional[CyclicLR] = None, retrainable=None):
        self.net = net.train()
        self.dtype = compute_dtype
        if lr_schedule is not None and not isinstance(lr_schedule, CyclicLR):
            raise TypeError("lr_schedule must be an engine.CyclicLR")
        self.lr_schedule = lr_schedule
        self._lr, self.momentum, self.wd, self.nesterov = lr, momentum, weight_decay, nesterov
        self.retrainable = retrainable is not None
        self.flat = FlatParams(net, retrainable)
        if lr_schedule is not None:
            dev = self.flat.flat_p.device
            start = lr_schedule.last_batch_iteration + 1
            self._lr_iter = torch.tensor([start], dtype=torch.int64, device=dev)
            self._lr32 = torch.zeros(1, dtype=torch.float32, device=dev)
            # before the first update: the rate that update will use, as the reference's CyclicLR sets it at construction
            self._lr64 = torch.tensor(lr_schedule.rate(start), dtype=torch.float64, device=dev)
        self._caches = [c for _, _, c in ops.operand_caches(net)]
        self._scope = ops.StepScope(self.flat.flat_g.device, training=True)
        self.pg = process_group
        self.world = torch.distributed.get_world_size(process_group) if process_group is not None else 1
        # data parallel: ranks exchange the SUM of their gradient arenas; the 1/world of the mean is folded into the optimiser
        # kernel (no scaling pass over the 131 MB arena)
        self.grad_scale = 1.0 / self.world
        self.use_graph = use_graph
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.static_x = self.static_m = self.static_loss = None
        self.first = True
        self.bucket_elems = bucket_mb * (1 << 20) // 4
        self.launches_per_step = 0
        self.graph_update = None
        self._captured_operands = None
        is_cuda = self.flat.flat_p.is_cuda
        if overlap_allreduce is None:
            overlap_allreduce = os.environ.get("PCB_DDP_OVERLAP", "1") != "0"
        self.overlap = bool(overlap_allreduce) and self.world > 1 and is_cuda
        self.overlap_active = False
        self._comm_stream = torch.cuda.Stream(device=self.flat.flat_p.device) if (self.world > 1 and is_cuda) else None
        self._hooks_installed = False
        self._hooked = set()            # slots with a post-accumulate hook (a hook cannot be removed, only ignored)
        self._make_buckets()
        if self.pg is not None:
            self._sync_replicas()

    @property
    def lr(self):
        return self._lr

    @lr.setter
    def lr(self, value):
        if self.lr_schedule is not None:
            raise AttributeError("this TrainStep follows its lr_schedule: the rate is computed on the device at every update")
        self._lr = value

    @property
    def iteration(self) -> Optional[int]:
        """The schedule iteration the next update runs (the reference's `last_batch_iteration + 1`); None without a schedule.
        Reading it synchronises with the device."""
        return int(self._lr_iter.item()) if self.lr_schedule is not None else None

    @property
    def last_lr(self) -> Optional[torch.Tensor]:
        """The rate of the last update as a device fp64 scalar, overwritten by the next update (reading it does not
        synchronise); before the first update, the rate that update will use.  None without a schedule."""
        return self._lr64 if self.lr_schedule is not None else None

    def _sync_replicas(self, momentum=False):
        """Data parallel start-up and resume: every rank adopts rank 0's parameters, schedule counter and module buffers
        (BatchNorm running statistics, `num_batches_tracked`), like torch DDP does, so replicas built from different seeds or
        checkpoints cannot silently diverge; every rank then computes the same rate from the same counter.  `momentum`: the
        momentum arena too (after a load; at construction it is zeros on every rank).  BatchNorm batch statistics stay
        rank-local afterwards (the reference has no SyncBN); running statistics therefore drift per rank during training and
        rank 0's are the ones to checkpoint.  Frozen parameters without an arena slot are broadcast one by one."""
        dist = torch.distributed
        src = dist.get_global_rank(self.pg, 0)
        dist.broadcast(self.flat.flat_p, src=src, group=self.pg)
        slotted = {id(p) for p in self.flat.params}
        for p in self.net.parameters():
            if id(p) not in slotted:
                dist.broadcast(p.data, src=src, group=self.pg)
        if momentum:
            dist.broadcast(self.flat.flat_m, src=src, group=self.pg)
        if self.lr_schedule is not None:
            dist.broadcast(self._lr_iter, src=src, group=self.pg)
            dist.broadcast(self._lr64, src=src, group=self.pg)
        for b in self.net.buffers():
            dist.broadcast(b, src=src, group=self.pg)
        ops.bump_weight_epoch()

    # -- frozen layers -----------------------------------------------------------------------------
    def _sync_cache_modes(self, refresh_frozen=False):
        """Give every operand cache of the network the mode of its weight: `frozen` (ops.OperandCache) while the weight requires
        no gradient, so prefetch_weights() skips it and a captured step has no refresh for it.  A cache that changes mode, and
        with `refresh_frozen` every frozen one, is rewritten in place once from the weight's current values (the buffers a
        captured graph reads stay the same); `refresh_frozen` also rewrites every frozen record the captured step holds, in
        case an eager forward has since given its cache a new one.  Modes change only outside a capture: a refresh captured
        into the step would run again on every replay (warmup_and_capture() sets the modes before it captures)."""
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            return
        done = set()
        for _, _, cache in ops.operand_caches(self.net):
            rec = cache.current
            if rec is None:
                continue
            frozen = not rec.weight.requires_grad
            if frozen != cache.frozen or (frozen and refresh_frozen):
                cache.frozen = frozen
                cache.refresh(rec)
                done.add(id(rec))
        if refresh_frozen:
            for rec in self._captured_operands or ():
                if id(rec) not in done and not rec.weight.requires_grad:
                    rec.refresh()

    def update_trainable(self):
        """Switch to the parameters' current `requires_grad` in place, after a stage change such as
        ``net.encoder.requires_grad_(True)`` or ``net.encoder.freeze_params(k)``: SGD ranges, gradient sinks and all-reduce
        buckets are rebuilt over the trainable slots, frozen layers' operands are laid out once, and the captured graph is
        dropped (the next `warmup_and_capture()` recaptures; its warm-up updates count in the schedule).  No parameter moves:
        a parameter that requires a gradient but has no arena slot (see `retrainable`) is refused before anything changes.
        Momentum, schedule counter and batcher generator carry over; a slot trained for the first time starts from zeros."""
        slotted = {id(p) for p in self.flat.params}
        missing = [n for n, p in self.net.named_parameters() if p.requires_grad and id(p) not in slotted]
        if missing:
            raise ValueError(f"update_trainable: {missing[:5]} require a gradient but have no arena slot; construct the step "
                             "with retrainable= covering them")
        self.close()
        self.flat.set_trainable()
        self._make_buckets()
        self._hooks_installed = False
        self._sync_cache_modes(refresh_frozen=True)

    # -- gradient exchange ---------------------------------------------------------------------------
    def _make_buckets(self):
        """Buckets of ~bucket_elems consecutive arena elements, cut at parameter boundaries.  Backward produces gradients
        roughly from the END of the arena (decoder) to its start (encoder), so buckets complete tail first.  Only trainable
        slots are exchanged: a bucket never crosses the end of a trainable range."""
        fp = self.flat
        self.buckets = []               # [start, end, [param indices]]
        i = 0
        for rs, re_ in fp.ranges:
            start, members = rs, []
            while i < len(fp.offsets) and fp.offsets[i] < re_:
                end = fp.offsets[i + 1] if i + 1 < len(fp.offsets) else fp.numel
                if fp.offsets[i] >= rs:
                    members.append(i)
                    if end - start >= self.bucket_elems or end == re_:
                        self.buckets.append([start, end, members])
                        start, members = end, []
                i += 1
        self._bucket_of = {}
        for b, (_, _, mem) in enumerate(self.buckets):
            for i in mem:
                self._bucket_of[i] = b

    def _install_hooks(self):
        """A parameter reports ONCE per step (its sink's first write, or its autograd accumulation).  A weight used twice in one
        forward would therefore be exchanged before its second contribution lands: the reference's networks share no weights;
        construct with overlap_allreduce=False for models that do."""
        if self._hooks_installed:
            return
        self._hooks_installed = True
        for i, p in enumerate(self.flat.params):
            if not p.requires_grad:
                continue
            sink = self.flat.sink_of.get(i)
            if sink is not None:
                sink.on_written = (lambda idx: (lambda: self._param_ready(idx)))(i)
            # parameters whose gradient still arrives through autograd (or a sink that was refused and fell back to it)
            if i not in self._hooked:
                self._hooked.add(i)
                p.register_post_accumulate_grad_hook((lambda idx: (lambda _p: self._param_ready(idx)))(i))

    def _param_ready(self, idx):
        if not self._overlap_armed or idx not in self._bucket_of:
            return
        b = self._bucket_of[idx]
        if idx in self._pending[b]:
            self._pending[b].discard(idx)
            if not self._pending[b]:
                self._launch_bucket(b)

    def _launch_bucket(self, b):
        """All-reduce (sum) of bucket b on the communication stream, ordered after everything issued so far on the compute
        stream (BatchNorm / bias gradients, autograd accumulations) and on the auxiliary streams the step has used (the
        weight-gradient side stream)."""
        if self._launched[b]:
            return
        self._launched[b] = True
        s, e, _ = self.buckets[b]
        comm = self._comm_stream
        comm.wait_stream(torch.cuda.current_stream())
        for st in self._scope.streams:
            comm.wait_stream(st)
        with torch.cuda.stream(comm):
            torch.distributed.all_reduce(self.flat.flat_g[s:e], group=self.pg)

    def _arm_overlap(self, on: bool):
        self._overlap_armed = bool(on)
        if on:
            self._install_hooks()
            self._pending = [set(mem) for _, _, mem in self.buckets]
            self._launched = [False] * len(self.buckets)

    _overlap_armed = False

    def _finish_overlap(self):
        """Buckets whose parameters did not all report (an unused parameter) are exchanged now; then the compute stream waits
        for the communication stream."""
        for b in range(len(self.buckets) - 1, -1, -1):
            if not self._launched[b]:
                self._launch_bucket(b)
        self._overlap_armed = False
        torch.cuda.current_stream().wait_stream(self._comm_stream)

    def _allreduce(self):
        """Un-overlapped exchange (fallback, and the CPU/gloo path): bucketed SUM all-reduce of the trainable ranges."""
        if self.world == 1:
            return
        g = self.flat.flat_g
        for rs, re_ in self.flat.ranges:
            for s in range(rs, re_, self.bucket_elems):
                torch.distributed.all_reduce(g[s:min(s + self.bucket_elems, re_)], group=self.pg)

    # -- one eager step ----------------------------------------------------------------------------
    def _prepare(self, x: torch.Tensor, mask: torch.Tensor):
        """reference-style inputs (fp32 NCHW image, fp32/uint8 {0,1} NCHW mask) -> (x*mask in compute dtype NHWC, HoleMask)"""
        n, c, h, w = x.shape
        # the 3-channel image travels as an 8-channel-padded NHWC buffer: 16-byte pixels feed the row-packed
        # tensor-core stem and the tail's second gather source directly
        buf = torch.empty((n, (c + 7) // 8 * 8, h, w), dtype=self.dtype, device=x.device, memory_format=CL).zero_()
        xin = buf[:, :c]
        xin.copy_(x * mask.to(x.dtype))                                                # Dataloader.py:131
        # masks of the reference's data path are one plane repeated over RGB (Dataloader.py:128-129); outside a graph capture
        # that promise is checked (one device sync), inside a capture it was checked by the eager warm-up steps
        if not torch.cuda.is_current_stream_capturing() and mask.shape[1] > 1:
            if not bool((mask == mask[:, :1]).all()):
                raise ValueError("TrainStep expects a channel-uniform hole mask (one plane repeated over the input channels)")
        return xin, HoleMask.from_dense(mask, channel_uniform=True)

    def _fwd_bwd(self, x, mask, overlap=False):
        self.flat.flat_g.zero_()
        for sk in self.flat.sinks:
            sk.used = False
        ops.bump_weight_epoch()
        self._arm_overlap(overlap)
        try:
            with self._scope:
                self._sync_cache_modes()
                ops.prefetch_weights(self._caches)     # operand re-layout of all trainable layers runs ahead on its own stream
                loss = self._forward_loss(x, mask)
                loss.backward()
        finally:
            if overlap:
                self._finish_overlap()
        return loss.detach()

    def _forward_loss(self, x, mask):
        """Forward + scalar loss of one step (SURVEY 8d benchmark loss: out.abs().mean())."""
        xin, hm = self._prepare(x, mask)
        return ops.l1_mean(self.net((xin, hm)))

    def _update(self, first_step: bool):
        """One SGD launch per trainable range (the whole arena unless some slots are frozen): frozen slots keep their
        parameters and momentum bitwise."""
        fp = self.flat
        if self.lr_schedule is None:
            for s, e in fp.ranges:
                ops.sgd_step(fp.flat_p[s:e], fp.flat_g[s:e], fp.flat_m[s:e], self.lr, self.momentum, self.wd, self.nesterov,
                             first_step, grad_scale=self.grad_scale)
            return
        s = self.lr_schedule
        ops.lr_cyclic(self._lr_iter, self._lr32, self._lr64, s.base_lr, s.max_lr, s.step_size, CyclicLR.MODES[s.mode], s.gamma)
        for a, e in fp.ranges:
            ops.sgd_step_dev(fp.flat_p[a:e], fp.flat_g[a:e], fp.flat_m[a:e], self._lr32, self.momentum, self.wd, self.nesterov,
                             grad_scale=self.grad_scale)

    def _step(self, x, mask, first_step: bool, overlap=None):
        overlap = self.overlap if overlap is None else overlap
        loss = self._fwd_bwd(x, mask, overlap=overlap)
        if self.world > 1 and not overlap:
            self._allreduce()
        self._update(first_step)
        return loss

    # -- public -------------------------------------------------------------------------------------
    def warmup_and_capture(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None, eager_warmup=2):
        """Run eager warm-up steps (also counts this library's launches per step), then capture the step."""
        for _ in range(eager_warmup):
            before = _lib.launch_count()
            self._step(x, mask, self.first)
            self.first = False
            self.launches_per_step = _lib.launch_count() - before
        torch.cuda.synchronize()
        self.overlap_active = self.overlap
        if not self.use_graph:
            return
        self.static_x = x.clone()
        self.static_m = mask.clone() if mask is not None else None
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._step(self.static_x, self.static_m, False)
        torch.cuda.current_stream().wait_stream(side)
        self._sync_cache_modes()        # caches the step above created (eager_warmup=0) take their mode before the capture
        torch.cuda.synchronize()
        graph = None
        if self.world == 1 or self.overlap:
            # one graph for the whole step.  Data parallel: the bucketed NCCL all-reduces are captured with it, on the
            # communication stream, each ordered after the kernels that complete its bucket -- they overlap the rest of backward
            try:
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    self.static_loss = self._step(self.static_x, self.static_m, False)
            except Exception as exc:  # noqa: BLE001 -- a collective that cannot be captured: fall back to the split scheme
                if self.world == 1:
                    raise
                print(f"[engine] capturing the overlapped all-reduce failed ({type(exc).__name__}: {exc}); "
                      "falling back to graph(forward+backward) | eager all-reduce | graph(SGD)", flush=True)
                graph = None
                self.overlap = self.overlap_active = False
                self._overlap_armed = False
                torch.cuda.synchronize()
        if graph is None:
            # data parallel fallback: the NCCL all-reduce stays OUTSIDE the captured graphs (graph A = forward+backward,
            # eager bucketed all-reduce of the gradient arena, graph B = fused SGD): no collective is captured
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self.static_loss = self._fwd_bwd(self.static_x, self.static_m)
            self.graph_update = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph_update):
                self._update(False)
        self.graph = graph
        # The captured kernels hold raw pointers to the per-layer operand buffers (ops.Operands): keep them alive for as long
        # as the graph exists.  An eager forward after capture (validation) misses the cache -- the optimiser bumps the
        # weight epoch -- and, with the in-place refresh off, replaces the cache's record with new buffers; without this list
        # the old ones would be freed under the graph.  (Each replay refreshes the captured buffers itself.)
        self._captured_operands = [c.current for c in self._caches if c.current is not None]
        torch.cuda.synchronize()

    def step(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x, mask already on the device.  Returns the (device) loss of this step."""
        if self.graph is not None:
            if x.data_ptr() != self.static_x.data_ptr():
                self.static_x.copy_(x, non_blocking=True)
            if mask is not None and mask.data_ptr() != self.static_m.data_ptr():
                self.static_m.copy_(mask, non_blocking=True)
            self.graph.replay()
            if self.graph_update is not None:
                self._allreduce()
                self.graph_update.replay()
            ops.bump_weight_epoch()             # the replay updated the parameters and running statistics in place
            return self.static_loss
        loss = self._step(x, mask, self.first)
        self.first = False
        return loss

    # -- checkpoints ----------------------------------------------------------------------------------
    def _arena_views(self, arena):
        """Per trainable parameter (FlatParams order), its slice of `arena` with the parameter's logical shape."""
        return [_flat_view(arena, o, p.data) for p, o in zip(self.flat.params, self.flat.offsets)]

    def state_dict(self) -> dict:
        """The training state as CPU tensors (for torch.save; loads on any machine):

          * "model": `net.state_dict()` -- the reference's keys, BatchNorm buffers included;
          * "optimizer": in torch.optim.SGD's state_dict format over the trainable parameters (FlatParams order:
            `[p for p in net.parameters() if p.requires_grad]`), each momentum buffer in its parameter's logical shape;
            `param_groups[0]["lr"]` is the current rate (`last_lr` with a schedule).  With `retrainable` it lists all of
            `net.parameters()` instead, and every slot, frozen or not, carries its buffer, so that it loads at either stage;
          * "last_batch_iteration" (with a schedule): the value that continues the reference's CyclicLR;
          * "batcher_rng" (steps fed by a GPU batcher): the batcher's device generator state.

        Data parallel: save rank 0's (its BatchNorm running statistics are the ones that count, see _sync_replicas)."""
        def cpu(t):
            return t.detach().to("cpu", copy=True)
        sched = self.lr_schedule is not None
        group = {"lr": float(self._lr64) if sched else float(self.lr), "momentum": self.momentum, "dampening": 0,
                 "weight_decay": self.wd, "nesterov": bool(self.nesterov), "maximize": False, "foreach": None,
                 "differentiable": False, "fused": None, "params": list(range(len(self.flat.params)))}
        index = list(range(len(self.flat.params)))
        if self.retrainable:
            pos = {id(p): j for j, p in enumerate(self.net.parameters())}
            group["params"] = list(range(len(pos)))
            index = [pos[id(p)] for p in self.flat.params]
        state = {}
        if self.momentum != 0:
            state = {j: {"momentum_buffer": cpu(m)} for j, m in zip(index, self._arena_views(self.flat.flat_m))}
        sd = {"model": OrderedDict((k, cpu(v)) for k, v in self.net.state_dict().items()),
              "optimizer": {"state": state, "param_groups": [group]}}
        if sched:
            sd["last_batch_iteration"] = self.iteration - 1
        batcher = getattr(self, "batcher", None)
        if batcher is not None:
            sd["batcher_rng"] = cpu(batcher.rng)
        return sd

    def _momentum_buffers(self, opt) -> list:
        """The momentum buffer of every slot (None: zeros) from a torch.optim.SGD-format state dict, whose one parameter group
        lists the slots, the trainable parameters or all of `net.parameters()`.  Only a frozen parameter without a slot may not
        carry state (with `retrainable`, a frozen slot keeps its buffer)."""
        groups = opt.get("param_groups")
        if not isinstance(groups, (list, tuple)) or len(groups) != 1:
            raise ValueError("load_state_dict: the optimizer state must have exactly one parameter group")
        g = groups[0]
        for key, have, want in (("momentum", float(g.get("momentum", 0.0)), float(self.momentum)),
                                ("nesterov", bool(g.get("nesterov", False)), bool(self.nesterov)),
                                ("dampening", float(g.get("dampening", 0.0)), 0.0),
                                ("maximize", bool(g.get("maximize", False)), False)):
            if have != want:
                raise ValueError(f"load_state_dict: the checkpoint's {key} is {have}, this step's {want}: its momentum buffers "
                                 "would mean something else")
        params = self.flat.params
        every = list(self.net.parameters())
        trainable = [p for p in params if p.requires_grad]
        ids = list(g.get("params", []))
        if len(ids) == len(params):
            order = params
        elif len(ids) == len(every):
            order = every
        elif len(ids) == len(trainable):    # a checkpoint of a step without `retrainable` at the current stage
            order = trainable
        else:
            raise ValueError(f"load_state_dict: the optimizer state lists {len(ids)} parameters; this network has {len(params)} "
                             f"trainable of {len(every)}")
        pos = {id(p): i for i, p in enumerate(params)}
        state = opt.get("state", {})
        bufs = [None] * len(params)
        for j, (pid, p) in enumerate(zip(ids, order)):
            buf = state.get(pid, {}).get("momentum_buffer")
            if buf is None:
                continue
            if id(p) not in pos:
                raise ValueError(f"load_state_dict: optimizer parameter {j} is frozen here but carries a momentum buffer")
            if tuple(buf.shape) != tuple(p.shape):
                raise ValueError(f"load_state_dict: optimizer parameter {j}: momentum buffer of shape {tuple(buf.shape)}, "
                                 f"parameter of shape {tuple(p.shape)}")
            bufs[pos[id(p)]] = buf
        return bufs

    def load_state_dict(self, state_dict: dict):
        """Restore a `state_dict()` (or a checkpoint of the reference modules: their state_dict as "model" and a
        torch.optim.SGD state_dict as "optimizer") IN PLACE: parameters and momentum into their arenas, module buffers
        (`num_batches_tracked` included), the schedule counter (from "last_batch_iteration"; without it, the schedule's own
        start) and the batcher's generator (when saved).  A missing momentum buffer means zeros.  The captured graph keeps
        replaying, now from the loaded state: capture first, then load (the warm-up of `warmup_and_capture()` takes real
        updates, which the load overwrites).

        The learning rate and weight decay stay this step's own; a momentum, nesterov, dampening or maximize that differs
        from it, or a parameter count or shape mismatch, raises ValueError before anything is written.  Data parallel: rank
        0's loaded state is then broadcast to every rank."""
        if "model" not in state_dict or "optimizer" not in state_dict:
            raise ValueError("load_state_dict: needs 'model' and 'optimizer' entries (net.load_state_dict loads weights alone)")
        model = state_dict["model"]
        own = self.net.state_dict()
        if set(model) != set(own):
            missing, extra = sorted(set(own) - set(model)), sorted(set(model) - set(own))
            raise ValueError(f"load_state_dict: model keys differ: missing {missing[:5]}, unexpected {extra[:5]}")
        for k, v in own.items():
            if tuple(model[k].shape) != tuple(v.shape):
                raise ValueError(f"load_state_dict: {k} has shape {tuple(model[k].shape)}, the network's {tuple(v.shape)}")
        bufs = self._momentum_buffers(state_dict["optimizer"])
        it = None
        if self.lr_schedule is not None:
            it = int(state_dict.get("last_batch_iteration", self.lr_schedule.last_batch_iteration)) + 1
            if it < 0:
                raise ValueError("load_state_dict: last_batch_iteration must be >= -1")
        batcher, rng = getattr(self, "batcher", None), state_dict.get("batcher_rng")
        if batcher is not None and rng is not None and tuple(rng.shape) != tuple(batcher.rng.shape):
            raise ValueError(f"load_state_dict: batcher_rng has shape {tuple(rng.shape)}, expected {tuple(batcher.rng.shape)}")
        with torch.no_grad():
            for k, v in own.items():
                v.copy_(model[k])
            for view, buf in zip(self._arena_views(self.flat.flat_m), bufs):
                view.zero_() if buf is None else view.copy_(buf)
            if it is not None:
                self._lr_iter.fill_(it)
                self._lr64.fill_(self.lr_schedule.rate(it))
            if batcher is not None and rng is not None:
                batcher.rng.copy_(rng)
        self.first = False          # the constant-rate path must read the restored momentum on its next update
        ops.bump_weight_epoch()
        if self.pg is not None:
            self._sync_replicas(momentum=True)
        self._sync_cache_modes(refresh_frozen=True)     # frozen layers' operands are not refreshed by the step itself

    def close(self):
        """Destroy the captured graphs (the step falls back to eager mode).  REQUIRED before
        `torch.distributed.destroy_process_group()` when the all-reduce was captured (`overlap_active`): NCCL keeps a reference
        per graph that holds captured collectives and its communicator teardown waits until those graphs are gone -- with the
        graphs alive the process hangs at exit (measured: the 2-GPU bench printed its line and never returned)."""
        if self.graph is not None or self.graph_update is not None:
            torch.cuda.synchronize()
            self.graph = None
            self.graph_update = None
            self._captured_operands = None
            import gc
            gc.collect()
            torch.cuda.synchronize()


class _BatcherStep:
    """`warmup_and_capture()` and `step(params=None)` of a training step whose step begins with a GPU batcher's `prepare()`
    (data.InpaintBatcher, data.SegBatcher): the captured graph draws the parameters and prepares the batch on the device.  Per
    step the host only decodes, calls ``batcher.stage(samples)`` and ``step()``.

    ``step(params)`` with explicit parameters needs ``use_graph=False`` (the graph holds the device sampler)."""

    def warmup_and_capture(self, eager_warmup=2):
        super().warmup_and_capture(torch.empty(0, device=self.batcher.device), None, eager_warmup=eager_warmup)

    def step(self, params=None) -> torch.Tensor:
        """One step on the staged batch.  Returns the (device) loss."""
        if self.graph is None:
            self._params = params
            try:
                loss = self._step(None, None, self.first)
            finally:
                self._params = None
            self.first = False
            return loss
        if params is not None:
            raise ValueError("explicit parameters need use_graph=False: the captured step draws its own")
        self.batcher.activate()
        self.graph.replay()
        self.batcher.release()
        if self.graph_update is not None:
            self._allreduce()
            self.graph_update.replay()
        ops.bump_weight_epoch()                 # the replay updated the parameters and running statistics in place
        return self.static_loss


class InpaintTrainStep(_BatcherStep, TrainStep):
    """TrainStep whose step begins with the GPU data path (data.InpaintBatcher.prepare): the captured graph samples the crop
    boxes, grayscale draws and strokes, resizes, masks and dilates on the device and then runs the training step on the result.
    Per step the host only decodes, calls ``batcher.stage(samples)`` and ``step()``.

    ``step(params)`` with explicit parameters needs ``use_graph=False`` (the graph holds the device sampler)."""

    def __init__(self, net: torch.nn.Module, batcher, **kwargs):
        super().__init__(net, compute_dtype=batcher.dtype, **kwargs)
        self.batcher = batcher
        self._params = None

    def _forward_loss(self, x, mask):
        xin, hm, _ = self.batcher.prepare(self._params)
        return ops.l1_mean(self.net((xin, hm)))


class InpaintLossTrainStep(InpaintTrainStep):
    """InpaintTrainStep trained on the reference's InpaintingLoss (loss.py:185-225) instead of the benchmark's L1 stand-in:
    the batcher's clean image is both `raw_input` (where the mask is valid they agree) and `origin`.  The loss runs inside the
    same captured graph.  The extractor's frozen parameters stay out of the gradient arena; its operand buffers are laid out
    once (keyed on the weights, not the step's weight epoch, so they are not refreshed every step) and kept alive with the
    graph's captured operands.  `last_terms` holds the five unweighted terms of the last step (device fp32 [5]:
    valid, hole, tv, perceptual, style)."""

    def __init__(self, net: torch.nn.Module, batcher, extractor, feature_range=3, **kwargs):
        from .loss import InpaintingLoss
        super().__init__(net, batcher, **kwargs)
        self.criterion = InpaintingLoss(extractor, feature_range)
        self._caches += [c for _, _, c in ops.operand_caches(extractor)]     # frozen: pinned with the graph, never prefetched

    @property
    def last_terms(self):
        return self.criterion.last_terms

    def _forward_loss(self, x, mask):
        xin, hm, clean = self.batcher.prepare(self._params)
        return self.criterion(clean, hm, self.net((xin, hm)), clean)


class SegTrainStep(TrainStep):
    """The same step for the dense segmentation networks (models/text_segmentation.py: `net(x)`, no masks): BASELINE.json
    configs[1] (TextSegament, batch 8) and configs[3] (XceptionTextSegment, batch 16, bf16).  `mask` is ignored."""

    def _forward_loss(self, x, mask=None):
        n, c, h, w = x.shape
        buf = torch.empty((n, (c + 7) // 8 * 8, h, w), dtype=self.dtype, device=x.device, memory_format=CL).zero_()
        xin = buf[:, :c]
        xin.copy_(x)
        return ops.l1_mean(self.net(xin))


class SegLossTrainStep(_BatcherStep, SegTrainStep):
    """SegTrainStep trained on the reference's data and losses: the step begins with the GPU segmentation data path
    (data.SegBatcher.prepare: crop, resize, ColorJitter, ToTensor on the device) and ends in ``criterion(net(x), target)``
    (loss.BinaryFocalLoss or loss.SoftBootstrapCrossEntropy with a reduced output), all in the one captured graph.  The
    logits reach the loss as the network returns them, the [n, 1, h, w] view of a channel-padded NHWC buffer."""

    def __init__(self, net: torch.nn.Module, batcher, criterion, **kwargs):
        super().__init__(net, compute_dtype=batcher.dtype, **kwargs)
        self.batcher = batcher
        self.criterion = criterion
        self._params = None

    def _forward_loss(self, x, mask=None):
        xin, target = self.batcher.prepare(self._params)
        return self.criterion(self.net(xin), target)


class InferStep:
    """Graph-captured inference of the partial-conv U-Nets: ``run(x, mask)`` with the reference's inputs (fp32 NCHW image and
    {0, 1} hole mask, prepared like TrainStep._prepare) returns the output as a static fp32 NCHW buffer that the next call
    overwrites.  The net runs in eval mode under no_grad, with the mask chain on its own stream and every eval-mode BatchNorm +
    activation that directly follows a convolution applied in that convolution's epilogue (an inference ops.StepScope).  The
    first call for an input shape runs the forward eagerly (operand caches, BatchNorm coefficients, counters), then captures it
    in one CUDA graph; later calls copy the inputs in and replay.

    Counters (from the eager warm-up): `launches_per_run` (this library's kernels per forward), `fused_sites` / `unfused_sites`
    (BatchNorm/activation passes applied in a convolution epilogue / still run on their own).

    Weights: a change of the weight epoch since capture (``load_state_dict`` and the initialisers bump it) makes the next run()
    rewrite the captured operand buffers in place (ops.OperandCache.refresh) and the BatchNorm coefficients before it replays;
    call refresh() after a mutation that does not bump the epoch."""

    def __init__(self, net: torch.nn.Module, compute_dtype=torch.bfloat16):
        self.net = net.eval()
        self.dtype = compute_dtype
        self._bns = [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
        self._scope = ops.StepScope(next(net.parameters()).device, training=False)
        self._graphs = {}
        self._captured_operands = []          # (cache, ops.Operands) of every captured convolution
        self._epoch = None
        self.launches_per_run = 0
        self.fused_sites = self.unfused_sites = 0

    _prepare = TrainStep._prepare

    def _forward(self, x, mask):
        xin, hm = self._prepare(x, mask)
        return self.net((xin, hm))

    def _key(self, x, mask):
        return tuple(x.shape), x.dtype, (tuple(mask.shape), mask.dtype) if mask is not None else None

    def _inputs(self, x, mask):
        return (x, mask)

    def _run_forward(self, *inputs):
        with self._scope, torch.no_grad():
            return self._forward(*inputs)

    def _check_markers(self):
        from .models.BaseModels import B200BNAct
        stale = [name for name, m in self.net.named_modules() if isinstance(m, B200BNAct) and "_pcb_fused_out" in m.__dict__]
        if stale:
            raise _lib.PcbError(f"fused convolution outputs were never consumed by their BatchNorm: {stale}")

    def _refresh_coefficients(self):
        for bn in self._bns:
            if not bn.training and bn.running_mean is not None and bn.weight is not None and bn.bias is not None:
                ops.bn_eval_coefficients(bn)

    def _capture(self, inputs):
        for _ in range(2):                    # eager warm-up: operand caches, coefficients, counters
            before = _lib.launch_count()
            out = self._run_forward(*inputs)
            self.launches_per_run = _lib.launch_count() - before
            self.fused_sites, self.unfused_sites = self._scope.fused_sites, self._scope.unfused_sites
            self._check_markers()
        torch.cuda.synchronize()
        static_in = tuple(t.clone() if t is not None else None for t in inputs)
        static_out = self._static_out(out)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._into(static_out, self._run_forward(*static_in))
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._into(static_out, self._run_forward(*static_in))
        self._check_markers()
        # the captured kernels hold raw pointers to the operand buffers current at capture: keep them (and what rewrites them)
        self._captured_operands += [(c, c.current) for _, _, c in ops.operand_caches(self.net) if c.current is not None]
        torch.cuda.synchronize()
        return graph, static_in, static_out

    def _static_out(self, out):
        """The buffer run() returns for this shape: a fp32 copy of the forward's output (a subclass whose forward writes a buffer
        of its own returns that buffer, and nothing is copied)."""
        return torch.empty(tuple(out.shape), dtype=torch.float32, device=out.device)

    @staticmethod
    def _into(static_out, out):
        if out is not static_out:
            static_out.copy_(out)

    def refresh(self):
        """Rewrite the captured operand buffers and BatchNorm coefficients from the current parameters and buffers."""
        ops.bump_weight_epoch()
        self._refresh()

    def _refresh(self):
        for cache, rec in self._captured_operands:
            cache.refresh(rec)
        self._refresh_coefficients()
        self._epoch = ops._WEIGHT_EPOCH

    def run(self, *inputs) -> torch.Tensor:
        key = self._key(*inputs)
        entry = self._graphs.get(key)
        if entry is None:
            if self._epoch is not None and self._epoch != ops._WEIGHT_EPOCH:
                self._refresh()
            entry = self._graphs[key] = self._capture(self._inputs(*inputs))
            self._epoch = ops._WEIGHT_EPOCH
        elif self._epoch != ops._WEIGHT_EPOCH:
            self._refresh()
        graph, static_in, static_out = entry
        for dst, src in zip(static_in, self._inputs(*inputs)):
            if dst is not None and src.data_ptr() != dst.data_ptr():
                dst.copy_(src, non_blocking=True)
        graph.replay()
        return static_out


class SegInferStep(InferStep):
    """InferStep for the segmentation networks (models/text_segmentation.py): ``run(x)``, fp32 NCHW image; returns the logits
    [n, 1, h, w] as a static fp32 NCHW buffer.  The demo's mask is ``ops.text_mask_postprocess(out, border_pad, out_hw)``."""

    def _forward(self, x):
        n, c, h, w = x.shape
        buf = torch.empty((n, (c + 7) // 8 * 8, h, w), dtype=self.dtype, device=x.device, memory_format=CL).zero_()
        xin = buf[:, :c]
        xin.copy_(x)
        return self.net(xin)

    def _key(self, x):
        return tuple(x.shape), x.dtype

    def _inputs(self, x):
        return (x,)


# the segmentation demo's Normalize (Examples/demo_segmentation.py:59-62), the input convention of the published checkpoint
DEMO_MEAN_STD = ((0.4935, 0.4563, 0.4544), (0.3769, 0.3615, 0.3566))


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


class _TextRemovalNets(torch.nn.Module):
    """Both networks of a TextRemovalStep under one module, so InferStep's BatchNorm list, operand caches, fused-output markers
    and weight refresh cover them together."""

    def __init__(self, seg_net, fill_net):
        super().__init__()
        self.seg = seg_net
        self.fill = fill_net


class TextRemovalStep(InferStep):
    """Text removal from pages in one CUDA graph per page shape, the pipeline the reference's README describes (detect the text
    and make a mask, white it out, inpaint the hole), each stage as the reference's own code defines it (DESIGN 5.2):

      1. ``Normalize(mean, std)`` of the page and zero padding on the right and bottom to multiples of 8 (EvaluateSet);
      2. the segmentation network's logits (eval mode, fused BatchNorm + activation epilogues);
      3. the demo's text mask: ``sigmoid > 0.5``, 3x3 max-pool, unpad (ops.text_mask_postprocess);
      4. the holes the U-Nets were trained on: the mask as a {0, 255} image, ``> 0.4 * 255``, ``cv2.dilate`` 10x10;
      5. ``valid = 1 - hole`` and ``page * valid``, padded on the right and bottom to multiples of ``2 ** len(fill_net.decoder)``
         (the padding is hole);
      6. the U-Net's fill (eval mode, fused epilogues, the mask chain on its own stream);
      7. the composite ``valid * page + (1 - valid) * fill`` cropped to the page, not clamped.

    `seg_net`: TextSegament or XceptionTextSegment; `fill_net`: ImageFillOrigin, ImageFillOriginV2 or ImageFill, on the same
    CUDA device.  `normalize`: (mean, std) of step 1, the demo's by default; None skips it.

    `seg_resize`: None segments the page at the size it is given.  An int is EvaluateSet's `resize` (600 in the segmentation
    demo, the scale the published checkpoint is used at): steps 1-3 then run on the page as EvaluateSet prepares it -- resized
    with Pillow's bicubic so its long side is about `seg_resize` (ops.evaluate_set_geometry, ops.page_resize_bicubic),
    normalized and padded on one side to `seg_resize` -- and step 3 brings the mask back to the page's size (EvaluateSet's
    resize_mask).  Steps 4-7 run at the page's own resolution either way.

    `region_hulls`: None leaves the step as above.  A number is the segmentation demo's area threshold (500 in its call): the
    graph then also draws the demo's ``_contour`` image from the step's own text mask and page (ops.text_region_hulls: the
    convex hull of every outer text contour with contourArea above the threshold, filled in RGB (50, 128, 30) on the page's
    bytes), so with ``seg_resize=600`` one run() gives both of the demo's images and the text-removed page.

    ``run(page)`` takes fp32 NCHW pages [n, 3, h, w] in [0, 1] (``to_tensor`` of the RGB page) and returns the composite as a
    static fp32 NCHW buffer that the next call overwrites.  The same call leaves static buffers of its stages:
    `text_mask` (uint8 [n, 1, h, w], 1 = text: the demo's mask), `valid` (uint8 [n, hu, wu], 1 = kept), `last_resized` (the
    resized fp32 page, None without `seg_resize`), `last_seg_input` (the segmentation network's input), `last_logits` and
    `last_fill` (the two networks' raw outputs), and `text_regions` (uint8 [n, h, w, 3], the demo's region image; None without
    `region_hulls`).  Counters and weight reloads as InferStep: ``load_state_dict`` on either network
    is picked up by the next run()."""

    def __init__(self, seg_net: torch.nn.Module, fill_net: torch.nn.Module, normalize=DEMO_MEAN_STD, compute_dtype=torch.bfloat16,
                 seg_resize=None, region_hulls=None):
        from .models.image_inpainting import ImageFill, ImageFillOrigin, ImageFillOriginV2
        from .models.text_segmentation import TextSegament, XceptionTextSegment
        if not isinstance(seg_net, (TextSegament, XceptionTextSegment)):
            raise TypeError(f"TextRemovalStep: seg_net must be a TextSegament or XceptionTextSegment, got {type(seg_net).__name__}")
        if not isinstance(fill_net, (ImageFillOrigin, ImageFillOriginV2, ImageFill)):
            raise TypeError(f"TextRemovalStep: fill_net must be an ImageFillOrigin, ImageFillOriginV2 or ImageFill, got "
                            f"{type(fill_net).__name__}")
        if compute_dtype not in (torch.bfloat16, torch.float32):
            raise ValueError("TextRemovalStep: compute_dtype must be torch.bfloat16 or torch.float32")
        devs = {t.device for net in (seg_net, fill_net) for t in list(net.parameters()) + list(net.buffers())}
        if len(devs) != 1 or next(iter(devs)).type != "cuda":
            raise ValueError(f"TextRemovalStep: both networks must be on one CUDA device, found {sorted(str(d) for d in devs)}")
        self.device = next(iter(devs))
        self.normalize = None
        if normalize is not None:
            mean, std = (tuple(float(v) for v in t) for t in normalize)
            if len(mean) != 3 or len(std) != 3:
                raise ValueError("TextRemovalStep: normalize takes (mean, std) with three values each")
            self.normalize = (mean, std)
        self.seg_resize = None
        if seg_resize is not None:
            if isinstance(seg_resize, bool) or not isinstance(seg_resize, int) or seg_resize <= 0 or seg_resize % 8:
                raise ValueError(f"TextRemovalStep: seg_resize must be None or a positive multiple of 8, got {seg_resize!r}")
            self.seg_resize = seg_resize
        self.region_hulls = None
        if region_hulls is not None:
            if isinstance(region_hulls, bool) or not isinstance(region_hulls, (int, float)) \
                    or not float("-inf") < float(region_hulls) < float("inf"):
                raise ValueError(f"TextRemovalStep: region_hulls must be None or a finite area threshold, got {region_hulls!r}")
            self.region_hulls = region_hulls
        super().__init__(_TextRemovalNets(seg_net, fill_net), compute_dtype)
        self.multiple = 2 ** len(fill_net.decoder)        # one nearest x2 per decoder stage
        self._outs = {}                                   # page shape -> the composite buffer run() returns
        self._products = {}                               # page shape -> the stage buffers of its graph (_PRODUCTS)
        self._cur = None
        self.text_mask = self.valid = self.last_resized = self.last_seg_input = self.last_logits = self.last_fill = None
        self.text_regions = None

    _PRODUCTS = ("text_mask", "valid", "last_resized", "last_seg_input", "last_logits", "last_fill", "text_regions")

    def _seg_geometry(self, h: int, w: int):
        """((rh, rw), border_pad): the size the page is segmented at and the padding to the segmentation grid."""
        if self.seg_resize is None:
            return (h, w), (0, _round_up(w, 8) - w, 0, _round_up(h, 8) - h)
        return ops.evaluate_set_geometry(h, w, self.seg_resize)

    def padded_sizes(self, h: int, w: int):
        """((hs, ws), (hu, wu)): the segmentation and U-Net grids of an h x w page."""
        (rh, rw), (_, right, _, bottom) = self._seg_geometry(h, w)
        return (rh + bottom, rw + right), (_round_up(h, self.multiple), _round_up(w, self.multiple))

    def _forward(self, page):
        n, _, h, w = page.shape
        (rh, rw), pad = self._seg_geometry(h, w)
        (hs, ws), (hu, wu) = self.padded_sizes(h, w)
        resized = ops.page_resize_bicubic(page, rh, rw) if self.seg_resize is not None else None
        x = ops.removal_seg_input(page if resized is None else resized, self.normalize, hs, ws, self.dtype)
        logits = self.net.seg(x)
        text_mask = ops.text_mask_postprocess(logits, pad, (h, w))
        corrupted, valid = ops.removal_holes(text_mask, page, hu, wu, self.dtype)
        fill = self.net.fill((corrupted, HoleMask.from_plane(valid, 3)))
        key = self._key(page)
        out = self._outs.get(key)
        if out is None:                                   # the first eager warm-up: never inside a capture
            out = self._outs[key] = torch.empty((n, 3, h, w), dtype=torch.float32, device=page.device)
        ops.removal_composite(fill, page, valid, out=out)
        regions = ops.text_region_hulls(text_mask, page, self.region_hulls) if self.region_hulls is not None else None
        self._cur = (text_mask, valid, resized, x, logits, fill, regions)
        return out

    def _static_out(self, out):
        return out                                        # the composite is written straight into the returned buffer

    def _key(self, page):
        return tuple(page.shape), page.dtype

    def _inputs(self, page):
        return (page,)

    def _capture(self, inputs):
        entry = super()._capture(inputs)
        self._products[self._key(*inputs)] = self._cur   # the captured forward's buffers, rewritten by every replay
        self._cur = None
        return entry

    def run(self, page: torch.Tensor) -> torch.Tensor:
        """Remove the text from a batch of pages (fp32 NCHW [n, 3, h, w]).  Returns the static fp32 NCHW composite."""
        ops._check_page(page, "TextRemovalStep.run", contiguous=False)
        if page.device != self.device:
            raise _lib.PcbError(f"TextRemovalStep.run: the page is on {page.device}, the networks on {self.device}")
        self._seg_geometry(*page.shape[2:])              # refuses a page seg_resize cannot take before anything is launched
        out = super().run(page.contiguous())
        for name, t in zip(self._PRODUCTS, self._products[self._key(page)]):
            setattr(self, name, t)
        return out


class _BatcherEvalStep(InferStep):
    """Held-out evaluation on a GPU batcher in one CUDA graph: `batcher.prepare()`, the eval-mode forward with InferStep's fused
    BatchNorm + activation epilogues and whatever the subclass's `_forward` adds, captured on the first call.  Per batch the host
    decodes, calls ``batcher.stage(samples)`` and ``run()``, which returns the network output as a static fp32 NCHW buffer that
    the next call overwrites.  ``batcher.reseed(seed)`` before a validation pass makes every pass draw the same crops;
    `warmup_and_capture()` leaves the generator (and the tensors `_kept_by_warmup` names) where it found them.

    Sharing the network with a (captured) TrainStep: run() evaluates the parameters and BatchNorm running statistics as they are
    at the call.  Every TrainStep step bumps the weight epoch, and the first run() after a change rewrites this step's operand
    buffers and BatchNorm coefficients once (InferStep's refresh).  The forward runs on operand caches of its own, swapped in for
    the call, so it never writes a buffer that the training graph reads, and it keeps every buffer its graph captured alive.
    run() leaves `net.training` as it found it.  Give it a batcher of its own: the training step's batcher buffers are the
    training graph's inputs."""

    def __init__(self, net: torch.nn.Module, batcher, compute_dtype=None, extra_modules=()):
        if compute_dtype is not None and compute_dtype != batcher.dtype:
            raise ValueError(f"compute_dtype {compute_dtype} differs from the batcher's {batcher.dtype}")
        training = net.training
        super().__init__(net, compute_dtype=batcher.dtype)
        net.train(training)
        self.batcher = batcher
        self._own = [(m, name, ops.OperandCache(c.frozen, c.derive)) for m, name, c in ops.operand_caches(net, *extra_modules)]
        self.last_loss = None

    @contextlib.contextmanager
    def _own_state(self):
        """Eval mode and this step's own operand caches for the duration of a call; the modules' own are restored after."""
        training = self.net.training
        saved = [(m, name, vars(m)[name]) for m, name, _ in self._own]
        for m, name, own in self._own:
            vars(m)[name] = own
        self.net.eval()
        try:
            yield
        finally:
            self.net.train(training)
            for m, name, cache in saved:
                vars(m)[name] = cache

    def _keep_loss(self, loss):
        if self.last_loss is None:
            self.last_loss = torch.zeros((), dtype=torch.float32, device=loss.device)
        self.last_loss.copy_(loss)

    def _key(self):
        return ()

    def _inputs(self):
        return ()

    def _kept_by_warmup(self):
        """The device state the warm-up's eager forwards advance and `warmup_and_capture()` restores."""
        return [self.batcher.rng]

    def warmup_and_capture(self):
        """Run the eager warm-up and capture the graph on the staged batch (the first run() does this when not called)."""
        kept = self._kept_by_warmup()
        saved = [t.clone() for t in kept]
        self._run()
        for t, v in zip(kept, saved):
            t.copy_(v)

    def _run(self) -> torch.Tensor:
        self.batcher.activate()
        with self._own_state():
            out = super().run()
        self.batcher.release()
        return out

    def run(self) -> torch.Tensor:
        """Evaluate the staged batch.  Returns the static fp32 NCHW output."""
        return self._run()


class InpaintEvalStep(_BatcherEvalStep):
    """Held-out evaluation of an inpainting U-Net in one CUDA graph (see _BatcherEvalStep): `batcher.prepare()`
    (data.InpaintBatcher or data.InpaintPairBatcher: the device draws the crops and strokes), the eval-mode forward with
    InferStep's fused BatchNorm + activation epilogues and mask-chain stream, and, with an `extractor` (loss.VggExtractor), the
    reference's InpaintingLoss forward without a backward.

    ``run()`` returns the output as a static fp32 NCHW buffer that the next call overwrites; `last_loss` (device fp32 scalar) and
    `last_terms` (device fp32 [5]: valid, hole, tv, perceptual, style, unweighted) hold the loss of that batch (None without an
    extractor).  ``batcher.reseed(seed)`` before a validation pass makes every pass draw the same crops and strokes."""

    def __init__(self, net: torch.nn.Module, batcher, extractor=None, feature_range=3, compute_dtype=None):
        super().__init__(net, batcher, compute_dtype=compute_dtype, extra_modules=() if extractor is None else (extractor,))
        self.criterion = None
        if extractor is not None:
            from .loss import InpaintingLoss
            self.criterion = InpaintingLoss(extractor, feature_range)

    @property
    def last_terms(self):
        return self.criterion.last_terms if self.criterion is not None else None

    def _forward(self):
        xin, hm, clean = self.batcher.prepare()
        out = self.net((xin, hm))
        if self.criterion is not None:
            self._keep_loss(self.criterion(clean, hm, out, clean))
        return out


class SegEvalStep(_BatcherEvalStep):
    """Held-out evaluation of a segmentation network (TextSegament, XceptionTextSegment) in one CUDA graph (see
    _BatcherEvalStep): `batcher.prepare()` (data.SegBatcher), the eval-mode forward with the fused BatchNorm + activation
    epilogues, the optional loss forward (`criterion`: loss.BinaryFocalLoss or loss.SoftBootstrapCrossEntropy with a reduced
    output; `last_loss` is its device fp32 scalar) and `score.update(logits, target)` (metrics.PixelAveragePrecision), which
    reads the logits in place as the network returns them.

    ``run()`` returns the logits [n, 1, h, w] as a static fp32 NCHW buffer that the next call overwrites.  A validation pass:
    ``reset()`` (and ``batcher.reseed(seed)`` to repeat the draws), then per batch ``batcher.stage(samples)`` and ``run()``,
    then ``score.average_precision()`` and ``score.counts``.  The capture's eager warm-up leaves the score as it found it, and a
    first run() without `warmup_and_capture()` captures first, so every run() counts its batch exactly once.

    The criterion is copied: the evaluation graph reduces its loss through a workspace of its own, never the one a training
    step captured."""

    def __init__(self, net: torch.nn.Module, batcher, criterion=None, compute_dtype=None):
        super().__init__(net, batcher, compute_dtype=compute_dtype)
        from .metrics import PixelAveragePrecision
        self.criterion = None
        if criterion is not None:
            self.criterion = copy.copy(criterion)
            self.criterion.__dict__.pop("_pcb_ws", None)
        self.score = PixelAveragePrecision(batcher.device)

    def reset(self):
        """Start a pass: zero the score."""
        self.score.reset()

    def _kept_by_warmup(self):
        return [self.batcher.rng, self.score.hist, self.score.counts_tensor]

    def _forward(self):
        x, target = self.batcher.prepare()
        out = self.net(x)
        if self.criterion is not None:
            self._keep_loss(self.criterion(out, target))
        self.score.update(out, target)
        return out

    def run(self) -> torch.Tensor:
        """Evaluate the staged batch and add it to the score.  Returns the static fp32 NCHW logits."""
        if not self._graphs:
            self.warmup_and_capture()
        return self._run()
