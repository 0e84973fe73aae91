"""The training step of train.py:117-352 around the icafusion_b200 model: optimiser groups, DDP wrap, GradScaler, one step,
and gradient accumulation over train.py's nominal batch of 64.

This is the caller side of the hot path (SURVEY.md section 8e): what the reference's ``train_rgb_ir`` does between building
the model and ``ema.update`` -- minus data loading, logging, checkpoints and evaluation.  The model's forward and backward are
the autograd nodes of ``icafusion_b200.autograd`` (our kernels); the optimiser, the GradScaler and DistributedDataParallel
are torch's, exactly the objects train.py constructs, so the one exchange step of the data-parallel path is DDP's bucketed
NCCL all-reduce of the gradients (481 MB fp32 for yolov5l), overlapped with the rest of the backward pass.

Two defects of the reference's multi-GPU mode are repaired here, outside the model code (SURVEY.md section 3):
  * 30 DMFF parameters per model never receive a gradient (``ln_input``, ``ln_output``, the block-level ``mlp`` and ``LN1``
    of every CrossTransformerBlock: common.py:701-702,716-721,724) while train.py:233 builds DDP with
    ``find_unused_parameters=False`` -> DDP raises in the second iteration.  ``freeze_dead_parameters`` takes them out of the
    graph (``requires_grad_(False)``) before the wrap; they stay in the state_dict.
  * train.py:583-588 only calls ``train_rgb_ir`` on rank 0; ``TrainStep`` is constructed and called on every rank.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .common import CrossTransformerBlock
from .loss import ComputeLoss

HYP_SCRATCH = dict(lr0=0.01, momentum=0.937, weight_decay=0.0005, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0,
                   fl_gamma=0.0)      # data/hyp.scratch.yaml (the keys the step reads)


def dead_parameters(model: nn.Module) -> List[str]:
    """Names of the parameters the reference's forward never touches (they get no gradient in the reference either)."""
    names = []
    for mod_name, m in model.named_modules():
        if isinstance(m, CrossTransformerBlock):
            for sub in ("ln_input", "ln_output", "mlp", "LN1"):
                for k, _ in getattr(m, sub).named_parameters():
                    names.append(f"{mod_name}.{sub}.{k}" if mod_name else f"{sub}.{k}")
    return names


def freeze_dead_parameters(model: nn.Module) -> List[str]:
    names = dead_parameters(model)
    params = dict(model.named_parameters())
    for k in names:
        params[k].requires_grad_(False)
    return names


def param_groups(model: nn.Module):
    """train.py:124-131: (BatchNorm weights [no decay], other weights [decay], biases), trainable parameters only.  A model
    converted to nn.SyncBatchNorm beforehand gets the groups of the unconverted one (the reference builds its groups before
    converting, train.py:124-131 then 196)."""
    pg0, pg1, pg2 = [], [], []
    for _, v in model.named_modules():
        if hasattr(v, "bias") and isinstance(v.bias, nn.Parameter) and v.bias.requires_grad:
            pg2.append(v.bias)
        if isinstance(v, (nn.BatchNorm2d, nn.SyncBatchNorm)):
            if v.weight.requires_grad:
                pg0.append(v.weight)
        elif hasattr(v, "weight") and isinstance(v.weight, nn.Parameter) and v.weight.requires_grad:
            pg1.append(v.weight)
    # (like the reference, parameters that are neither .weight nor .bias -- pos_emb, LearnableWeights.w1/w2 -- join no group;
    #  LearnableCoefficient.bias lands in the bias group)
    return pg0, pg1, pg2


class ModelEMA:
    """utils/torch_utils.py:278-330: exponential moving average of every floating state_dict entry, decay ramped by the update
    count.  Same attributes (`ema`, `updates`, `decay`) and the same `update(model)`; the per-tensor Python loop of the
    reference (two kernels per tensor, ~1 300 launches for yolov5l) is two multi-tensor launches here."""

    def __init__(self, model: nn.Module, decay: float = 0.9999, updates: int = 0):
        import math
        from copy import deepcopy
        src = model.module if hasattr(model, "module") else model
        packs = {id(m): {k: m.__dict__.pop(k) for k in [k for k in m.__dict__ if k.startswith("_icaf_")]} for m in src.modules()}
        try:
            self.ema = deepcopy(src).eval()              # (packed-filter caches and stream pools are not part of the model)
        finally:
            for m in src.modules():
                m.__dict__.update(packs[id(m)])
        self.updates = updates
        self.decay = lambda x: decay * (1 - math.exp(-x / 2000))
        for p in self.ema.parameters():
            p.requires_grad_(False)

    def update(self, model: nn.Module) -> None:
        with torch.no_grad():
            self.updates += 1
            d = self.decay(self.updates)
            msd = (model.module if hasattr(model, "module") else model).state_dict()
            dst, src = [], []
            for k, v in self.ema.state_dict().items():
                if v.dtype.is_floating_point:
                    dst.append(v)
                    src.append(msd[k].detach())
            torch._foreach_mul_(dst, d)
            torch._foreach_add_(dst, src, alpha=1.0 - d)


class TrainStep:
    """model -> (optional DDP) -> loss -> scaled backward -> optimiser step, per call (train.py:334-352).

    Gradient accumulation (train.py:123-125, 314-320, 346-352): the reference steps the optimiser once per nominal batch of
    64 images, every ``accumulate`` batches.  ``__call__(..., optimizer_step=False)`` runs forward, loss and the scaled
    backward and leaves the gradients in ``.grad`` for the next call to add to; a train.py-shaped loop reads

        step(rgb, ir, targets, optimizer_step=(ni % step.accumulate_at(ni, nw) == 0))

    and calls ``step.zero_grad()`` at the start of each epoch (train.py:291).  Under DDP every backward all-reduces, as in the
    reference (no ``no_sync``): the bucket views accumulate the per-micro-batch averages.

    adam (train.py --adam): ``optim.Adam(pg0, lr=lr0, betas=(momentum, 0.999))`` instead of nesterov SGD, same three groups.

    sync_bn (train.py --sync-bn): with world_size > 1, every BatchNorm2d is converted to nn.SyncBatchNorm after the optimiser
    groups are built and before the DDP wrap (train.py:195-198), so BatchNorm normalises over the batch of all ranks.  At
    world size 1 the model is left as it is.  A model the caller converted beforehand trains synchronised as well."""

    def __init__(self, model: nn.Module, hyp: Optional[Dict[str, float]] = None, total_batch_size: int = 64, world_size: int = 1,
                 local_rank: Optional[int] = None, imgsz: int = 640, amp_scale: bool = True, ema: bool = False, sync_bn: bool = False,
                 adam: bool = False):
        hyp = dict(HYP_SCRATCH if hyp is None else hyp)
        det = model.model[-1]
        nl, nc = det.nl, det.nc
        nbs = 64
        accumulate = max(round(nbs / total_batch_size), 1)
        hyp["weight_decay"] *= total_batch_size * accumulate / nbs                    # train.py:121
        self.nbs, self.total_batch_size, self.accumulate = nbs, total_batch_size, accumulate
        self.dead = freeze_dead_parameters(model)
        pg0, pg1, pg2 = param_groups(model)
        if adam:
            self.optimizer = torch.optim.Adam(pg0, lr=hyp["lr0"], betas=(hyp["momentum"], 0.999))            # train.py:133-134
        else:
            self.optimizer = torch.optim.SGD(pg0, lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)  # train.py:136
        self.optimizer.add_param_group({"params": pg1, "weight_decay": hyp["weight_decay"]})
        self.optimizer.add_param_group({"params": pg2})
        hyp["box"] *= 3.0 / nl                                                        # train.py:238-240
        hyp["cls"] *= nc / 80.0 * 3.0 / nl
        hyp["obj"] *= (imgsz / 640) ** 2 * 3.0 / nl
        model.nc, model.hyp, model.gr = nc, hyp, 1.0                                  # train.py:242-244
        if sync_bn and world_size > 1:
            model = nn.SyncBatchNorm.convert_sync_batchnorm(model)                     # train.py:195-198
        self.raw_model = model
        self.world_size = world_size
        if world_size > 1:
            from torch.nn.parallel import DistributedDataParallel as DDP
            model = DDP(model, device_ids=None if local_rank is None else [local_rank], output_device=local_rank,   # train.py:233
                        find_unused_parameters=False,
                        gradient_as_bucket_view=True)              # .grad aliases the all-reduce buckets: no copy in / out
        self.model = model
        self.scaler = torch.amp.GradScaler("cuda", enabled=amp_scale and torch.cuda.is_available())    # train.py:282
        self.compute_loss = ComputeLoss(self.raw_model)                               # train.py:284
        self.hyp = hyp
        self.ema = ModelEMA(self.raw_model) if ema else None                          # train.py:154 (rank 0 / single GPU in the reference)

    def accumulate_at(self, ni: int, nw: int) -> int:
        """Batches per optimiser step at integrated batch ``ni`` with ``nw`` warm-up batches: train.py:317's ramp from 1 to
        64 / total_batch_size during warm-up, ``accumulate`` (train.py:124) after it."""
        if ni <= nw:
            return int(max(1, np.interp(ni, [0, nw], [1, self.nbs / self.total_batch_size]).round()))
        return self.accumulate

    def __call__(self, rgb: torch.Tensor, ir: torch.Tensor, targets: torch.Tensor, optimizer_step: bool = True):
        """rgb / ir: (B,3,H,W) uint8 (scaled by 1/255 inside the stem staging, train.py:297-298) or float images on the device;
        targets (nt, 6).  optimizer_step=False: only add this batch's scaled gradients to ``.grad`` (train.py:346 with
        ``ni % accumulate != 0``).  Returns (loss, loss_items) of this rank."""
        pred = self.model(rgb, ir)                                                    # train.py:336
        loss, items = self.compute_loss(pred, targets)                                # train.py:337
        if self.world_size > 1:
            loss = loss * self.world_size                                             # train.py:339
        self.scaler.scale(loss).backward()                                            # train.py:344
        if optimizer_step:
            self.scaler.step(self.optimizer)                                          # train.py:347-350
            self.scaler.update()
            self.zero_grad()
            if self.ema is not None:
                self.ema.update(self.raw_model)                                       # train.py:351-352
        return loss.detach(), items

    def zero_grad(self) -> None:
        """optimizer.zero_grad() of train.py:350, extended to the 18 trainable parameters no optimiser group holds (pos_emb_*,
        LearnableWeights.w1/w2): the reference never clears their .grad, which then grows by one gradient per step."""
        self.raw_model.zero_grad(set_to_none=True)


class GraphedTrainStep:
    """The same step with forward + loss + scaled backward (+ DDP's bucketed all-reduce) captured ONCE as a CUDA graph and
    replayed per batch: the ~3000 kernel launches of a yolov5l step cost the host more time than the GPU needs to run them.
    Static shapes: (B,3,H,W) uint8 batches and at most `max_targets` label rows (unused rows carry image index -1, which
    build_targets rejects).  The optimiser step and GradScaler.update stay eager (train.py:348-350; GradScaler reads its
    inf flag on the host).  Dropout masks: the kernels add a device-side step counter to their seeds (icaf_set_seed_offset),
    incremented inside the graph, so every replay draws new masks.

    Gradient accumulation: the graph above (the "fresh" one) writes the gradients into the static ``.grad`` tensors.  The
    first call with ``optimizer_step=False`` captures a second, "accumulating" graph on the same inputs and memory pool while
    ``.grad`` is defined, so autograd adds into those tensors in place.  The fresh graph serves the first micro-batch after
    construction, an optimiser step or ``zero_grad()``; the accumulating one every other micro-batch.  A run that steps on
    every call never captures it.

    DDP (world_size > 1): construct the TrainStep inside ``torch.cuda.stream(side)`` and set TORCH_NCCL_ASYNC_ERROR_HANDLING=0
    before init_process_group, as torch's CUDA-graph notes require; 11 eager iterations run before the capture."""

    def __init__(self, ts: TrainStep, B: int, H: int, W: int, max_targets: int, device, warmup: Optional[int] = None):
        from .autograd import sync_group
        for m in ts.raw_model.modules():           # SyncBatchNorm exchanges are captured like DDP's all-reduces: over NCCL only
            g = sync_group(m)
            if g is not None and torch.distributed.get_backend(g) != "nccl":
                raise ValueError(f"GraphedTrainStep: synchronised BatchNorm needs an NCCL process group to be captured, "
                                 f"got {torch.distributed.get_backend(g)}")
        self.ts = ts
        dev = torch.device(device)
        self.rgb = torch.zeros(B, 3, H, W, dtype=torch.uint8, device=dev)
        self.ir = torch.zeros_like(self.rgb)
        self.tg = torch.zeros(max_targets, 6, dtype=torch.float32, device=dev)
        self.tg[:, 0] = -1.0
        self.seed_ctr = torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.check(_lib.lib().icaf_set_seed_offset(self.seed_ctr.data_ptr()), "icaf_set_seed_offset")
        self.max_targets = max_targets
        warmup = (11 if ts.world_size > 1 else 3) if warmup is None else warmup
        # the warm-up iterations are real steps on an all-zero batch: snapshot everything they touch and put it back afterwards
        saved = {k: v.detach().clone() for k, v in ts.raw_model.state_dict().items()}
        saved_scaler = ts.scaler.state_dict()
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(warmup):                      # real steps on the zero batch: allocator, cuBLAS-free lazy inits, DDP buckets
                self.seed_ctr += 1
                ts(self.rgb, self.ir, self.tg)
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        with torch.no_grad():
            for k, v in ts.raw_model.state_dict().items():
                v.copy_(saved[k])                        # in place: the graph will be captured on these very tensors
            for st in ts.optimizer.state.values():   # == the state before the first step: SGD seeds its momentum buffer with
                for v in st.values():                # the gradient; Adam starts from step 0 and zero moments
                    if torch.is_tensor(v):
                        v.zero_()
        if saved_scaler:
            ts.scaler.load_state_dict(saved_scaler)
        self.seed_ctr.zero_()
        ts.zero_grad()
        self.graph = torch.cuda.CUDAGraph()
        self.loss, self.items = self._capture(self.graph)
        self.acc_graph = None                            # the accumulating graph, captured on first use
        self.fresh = True                                # the next replay starts a new accumulation window

    def _capture(self, graph, pool=None):
        ts = self.ts
        with torch.cuda.graph(graph, pool=pool):
            self.seed_ctr += 1
            pred = ts.model(self.rgb, self.ir)
            loss, items = ts.compute_loss(pred, self.tg)
            if ts.world_size > 1:
                loss = loss * ts.world_size
            ts.scaler.scale(loss).backward()
        return loss, items

    def __call__(self, rgb: torch.Tensor, ir: torch.Tensor, targets: torch.Tensor, optimizer_step: bool = True):
        """As TrainStep.__call__; optimizer_step=False adds this batch's gradients to the static ``.grad`` tensors."""
        nt = int(targets.shape[0])
        if nt > self.max_targets:
            raise ValueError(f"GraphedTrainStep: {nt} label rows, captured for at most {self.max_targets}")
        self.rgb.copy_(rgb, non_blocking=True)
        self.ir.copy_(ir, non_blocking=True)
        self.tg[:nt].copy_(targets, non_blocking=True)
        if nt < self.max_targets:
            self.tg[nt:, 0] = -1.0
        if self.fresh:
            self.graph.replay()
            loss, items = self.loss, self.items
        else:
            if self.acc_graph is None:                   # .grad holds this window's gradients: the capture adds into them
                self.acc_graph = torch.cuda.CUDAGraph()
                self.acc_loss, self.acc_items = self._capture(self.acc_graph, pool=self.graph.pool())
            self.acc_graph.replay()
            loss, items = self.acc_loss, self.acc_items
        self.fresh = optimizer_step
        if optimizer_step:
            self.ts.scaler.step(self.ts.optimizer)        # gradients live in static buffers the next fresh replay overwrites
            self.ts.scaler.update()
            if self.ts.ema is not None:
                self.ts.ema.update(self.ts.raw_model)
        return loss.detach(), items

    def zero_grad(self) -> None:
        """Start a new accumulation window (train.py:291): the next call replays the fresh graph, which overwrites ``.grad``.
        The gradient tensors stay allocated, because both graphs write them in place."""
        self.fresh = True

    def close(self) -> None:
        _lib.lib().icaf_set_seed_offset(None)
