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
from .common import CrossTransformerBlock, TransformerFusionBlock
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


def set_dmff_stream_dtype(model: nn.Module, fp32: bool) -> None:
    """Train every DMFF block of `model` with fp32 token streams (fp32) or fp16 ones: TransformerFusionBlock.stream_dtype."""
    for m in model.modules():
        if isinstance(m, TransformerFusionBlock):
            m.stream_dtype = torch.float32 if fp32 else torch.float16


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
    world size 1 the model is left as it is.  A model the caller converted beforehand trains synchronised as well.

    dmff_fp32: True gives every TransformerFusionBlock fp32 token streams and stream gradients (stream_dtype): the dtype
    each DMFF node has in the reference's autocast step, with fp16 GEMM operands.  False gives them fp16 streams; None (the
    default) keeps each block's stream_dtype as it is (fp16 unless the caller set it).  The precision of the whole step's
    one-element DMFF gradients is measured, per model, in DESIGN.md section 4.6."""

    def __init__(self, model: nn.Module, hyp: Optional[Dict[str, float]] = None, total_batch_size: int = 64, world_size: int = 1,
                 local_rank: Optional[int] = None, imgsz: int = 640, amp_scale: bool = True, ema: bool = False, sync_bn: bool = False,
                 adam: bool = False, dmff_fp32: Optional[bool] = None):
        hyp = dict(HYP_SCRATCH if hyp is None else hyp)
        if dmff_fp32 is not None:
            set_dmff_stream_dtype(model, dmff_fp32)
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


def adam_bias_corrections(beta1: float, beta2: float, steps: int) -> np.ndarray:
    """float64 (steps, 2): row s = (1 - beta1 ** s, (1 - beta2 ** s) ** 0.5), the Python expressions torch's Adam evaluates on
    the host for a tensor at step s (_multi_tensor_adam, non-capturable branch).  Row 0 is never read."""
    out = np.empty((steps, 2), dtype=np.float64)
    for s in range(steps):
        out[s, 0] = 1 - beta1 ** float(s)
        out[s, 1] = (1 - beta2 ** float(s)) ** 0.5
    return out


class DeviceOptimizerStep:
    """``scaler.step(optimizer); scaler.update(); ema.update(model)`` of train.py:347-352 as a fixed list of our kernels that
    reads nothing back to the host, so it can be captured into a CUDA graph: unscale with the inf check into a device flag,
    nesterov SGD or Adam over each parameter group (skipped on the device when the flag is set), the scale update (which
    clears the flag) and the EMA update.  The kernels work on torch's own tensors -- parameters, ``.grad``, the optimiser's
    state, GradScaler's ``_scale`` / ``_growth_tracker``, the EMA model's state -- so ``optimizer.state_dict()``,
    ``scaler.state_dict()`` and ``ema.ema`` stay what the eager path would have made of them.

    The tables hold the addresses of those tensors: every group parameter needs its ``.grad`` before construction, and none
    of them may be reallocated afterwards.  Missing optimiser state is created as torch's first step would see it (a zero
    momentum buffer gives buf = d; Adam's moments start at zero); Adam's ``step`` tensors move to the device.

    Per-step scalars -- each group's lr, momentum / betas, weight decay and eps, and the EMA decay -- are read from
    ``param_groups`` and ``ema.updates`` by :meth:`stage` and staged through a ring of pinned slots; each slot is reused only
    once the copy out of it has completed (one CUDA event per slot).  GradScaler's growth factor, backoff factor and interval
    are read at construction.

    Adam's bias corrections come from a per-group table of rows 0 .. BIAS_STEPS - 1; when the number of stepping calls
    reaches its size, :meth:`stage` reallocates it at twice the size and the launches must be captured again (a graph
    capture synchronises the device: the one host wait of this path, once per doubling)."""

    RING = 4
    BIAS_STEPS = 65536          # rows of Adam's bias-correction table (train.py's 300 epochs of KAIST take ~42 000 steps);
                                # it doubles when the step count reaches it

    def __init__(self, optimizer, scaler, ema, model: nn.Module, device):
        from . import ops
        self.optimizer, self.scaler, self.ema = optimizer, scaler, ema
        dev = torch.device(device)
        self.adam = isinstance(optimizer, torch.optim.Adam)
        if not self.adam and not isinstance(optimizer, torch.optim.SGD):
            raise ValueError(f"DeviceOptimizerStep: SGD or Adam, got {type(optimizer).__name__}")
        rows, ranges = [], {}
        for gi, group in enumerate(optimizer.param_groups):
            if group.get("maximize") or group.get("differentiable"):
                raise ValueError("DeviceOptimizerStep: maximize / differentiable are not supported")
            if self.adam and (group["amsgrad"] or group.get("decoupled_weight_decay")):
                raise ValueError("DeviceOptimizerStep: Adam without amsgrad or decoupled weight decay only")
            if not self.adam and (not group["nesterov"] or group["dampening"] != 0):
                raise ValueError("DeviceOptimizerStep: SGD with nesterov=True and dampening=0 only (train.py:136)")
            lo = len(rows)
            for p in group["params"]:
                if p.grad is None:
                    raise ValueError("DeviceOptimizerStep: every group parameter needs its .grad (run a backward first)")
                st = optimizer.state[p]
                if self.adam:
                    step = st.get("step")
                    st["step"] = torch.zeros((), dtype=torch.float32, device=dev) if step is None else \
                        torch.as_tensor(step, dtype=torch.float32).to(dev)
                    for k in ("exp_avg", "exp_avg_sq"):
                        if st.get(k) is None:
                            st[k] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    rows.append((p, p.grad, st["exp_avg"], st["exp_avg_sq"], st["step"]))
                else:
                    if st.get("momentum_buffer") is None:
                        st["momentum_buffer"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    rows.append((p, p.grad, st["momentum_buffer"], None, None))
            ranges[gi] = (lo, len(rows))
        self.groups = [gi for gi, (lo, hi) in ranges.items() if hi > lo]
        self.table = ops.OptimTable(rows, dev, ranges)
        self.ema_table = None
        if ema is not None:
            msd = model.state_dict()
            self.ema_table = ops.OptimTable([(v, msd[k], None, None, None) for k, v in ema.ema.state_dict().items()
                                             if v.dtype.is_floating_point], dev)
        self.scaled = scaler.is_enabled()
        if self.scaled and scaler._scale is None:
            raise ValueError("DeviceOptimizerStep: GradScaler has no scale tensor yet (call scaler.scale() once first)")
        G = len(optimizer.param_groups)
        self.found_inf = torch.zeros(1, dtype=torch.float32, device=dev)
        self.scalars = torch.zeros(1 + G, _lib.OPTIM_HYPER, dtype=torch.float64, device=dev)   # row 0: EMA decay; 1 + g: group g
        self.hyper = self.scalars[1:]
        pinned = not ops.dry_running()
        self.slots = torch.zeros(self.RING, 1 + G, _lib.OPTIM_HYPER, dtype=torch.float64, pin_memory=pinned)
        self.slots_np = self.slots.numpy()
        self.events = [None] * self.RING
        self.slot = 0
        self.device = dev
        self.bias_corr = None
        if self.adam:           # rows for every step the kernels can reach before the table next grows
            self.max_step = 0 if ops.dry_running() or not rows else int(torch.stack([r[4] for r in rows]).max())
            self._bias_corr_rows(self.BIAS_STEPS)

    def _bias_corr_rows(self, steps: int) -> None:
        from . import ops
        self.betas = [tuple(map(float, g["betas"])) for g in self.optimizer.param_groups]
        rows = {b: adam_bias_corrections(*b, steps) for b in set(self.betas)}
        host = torch.from_numpy(np.stack([rows[b] for b in self.betas]))
        host = host if ops.dry_running() else host.pin_memory()
        if self.bias_corr is not None and self.bias_corr.shape[1] == steps:
            self.bias_corr.copy_(host, non_blocking=True)       # same address: captured launches keep reading it
        else:
            self.bias_corr = host.to(self.device, non_blocking=True)

    def enqueue(self) -> None:
        """The step's launches on the current stream (what a CUDA graph captures)."""
        from . import ops
        sc = self.scaler
        if self.scaled:
            ops.amp_unscale(self.table, sc._scale, self.found_inf)
        for gi in self.groups:
            if self.adam:
                ops.adam_step(self.table, gi, self.hyper, self.bias_corr, self.found_inf)
            else:
                ops.sgd_step(self.table, gi, self.hyper, self.found_inf)
        if self.scaled:
            ops.amp_update_scale(sc._scale, sc._growth_tracker, self.found_inf, sc._growth_factor, sc._backoff_factor,
                                 sc._growth_interval)
        if self.ema_table is not None:
            ops.ema_update(self.ema_table, self.scalars[0])

    def stage(self) -> bool:
        """Host side of one step, before its launches run: copy this step's scalars to the device (ModelEMA's update count
        advances here, as ``ema.update`` advances it).  Returns True when Adam's bias-correction table was reallocated to
        cover more steps: launches enqueued (or captured) before then must be enqueued again."""
        k = self.slot
        if self.events[k] is None:
            self.events[k] = torch.cuda.Event()
        elif not self.events[k].query():             # the GPU is a whole ring behind: wait for this slot's last copy
            self.events[k].synchronize()
        s = self.slots_np[k]
        for gi, g in enumerate(self.optimizer.param_groups):
            row = s[1 + gi]
            row[0], row[2] = g["lr"], g["weight_decay"]
            if self.adam:
                row[1], row[3] = g["betas"]
                row[4] = g["eps"]
            else:
                row[1] = g["momentum"]
        if self.ema is not None:
            self.ema.updates += 1
            s[0, 0] = self.ema.decay(self.ema.updates)
        grew = False
        if self.adam:
            self.max_step += 1
            betas = [tuple(map(float, g["betas"])) for g in self.optimizer.param_groups]
            steps = self.bias_corr.shape[1]
            if self.max_step >= steps or betas != self.betas:
                grew = self.max_step >= steps
                self._bias_corr_rows(2 * steps if grew else steps)
        self.scalars.copy_(self.slots[k], non_blocking=True)
        self.events[k].record()
        self.slot = (k + 1) % self.RING
        self.optimizer._opt_called = True            # what LRScheduler.step checks for "scheduler before optimizer"
        return grew


class GraphedTrainStep:
    """The same step with forward + loss + scaled backward (+ DDP's bucketed all-reduce) captured ONCE as a CUDA graph and
    replayed per batch: the ~3000 kernel launches of a yolov5l step cost the host more time than the GPU needs to run them.
    Static shapes: (B,3,H,W) uint8 batches and at most `max_targets` label rows (unused rows carry image index -1, which
    build_targets rejects).  Dropout masks: the kernels add a device-side step counter to their seeds (icaf_set_seed_offset),
    incremented inside the graph, so every replay draws new masks.

    The optimiser step (train.py:347-352: scaler.step, scaler.update, zero_grad, ema.update) is a third, small graph on the
    same pool, replayed after the backward of every stepping call: :class:`DeviceOptimizerStep`'s unscale, SGD or Adam gated
    on the device-side inf flag, scale update and EMA update.  A call reads nothing back and never calls
    ``optimizer.step()``, so the host can prepare the next batch while the GPU trains.  (With Adam, the call that outgrows
    the bias-correction table -- the 65 536th stepping call, then every doubling -- captures the step graph again, which
    synchronises the device once.)  Each call stages the groups' current
    lr / momentum (train.py's warm-up and LambdaLR write them between calls) and the EMA decay; ``optimizer.state_dict()``,
    ``scaler.state_dict()`` and ``ema`` hold what the eager TrainStep would have after the same calls.  Under DDP every rank
    steps on the same all-reduced gradients, so the ranks take the same skip decisions without an exchange.

    Gradient accumulation: the graph above (the "fresh" one) writes the gradients into the static ``.grad`` tensors.  The
    first call with ``optimizer_step=False`` captures a second, "accumulating" graph on the same inputs and memory pool while
    ``.grad`` is defined, so autograd adds into those tensors in place.  The fresh graph serves the first micro-batch after
    construction, an optimiser step or ``zero_grad()``; the accumulating one every other micro-batch.  A run that steps on
    every call never captures it.

    DDP (world_size > 1): construct the TrainStep inside ``torch.cuda.stream(side)`` and set TORCH_NCCL_ASYNC_ERROR_HANDLING=0
    before init_process_group, as torch's CUDA-graph notes require; 11 eager iterations run before the capture.

    dmff_fp32: as TrainStep's, set on the model before the capture; None keeps what the TrainStep set."""

    def __init__(self, ts: TrainStep, B: int, H: int, W: int, max_targets: int, device, warmup: Optional[int] = None,
                 dmff_fp32: Optional[bool] = None):
        from .autograd import sync_group
        if dmff_fp32 is not None:
            set_dmff_stream_dtype(ts.raw_model, dmff_fp32)
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
        if ts.ema is not None:
            saved_ema = ({k: v.detach().clone() for k, v in ts.ema.ema.state_dict().items()}, ts.ema.updates)
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
            if ts.ema is not None:
                for k, v in ts.ema.ema.state_dict().items():
                    v.copy_(saved_ema[0][k])
                ts.ema.updates = saved_ema[1]
        if saved_scaler:
            ts.scaler.load_state_dict(saved_scaler)
        self.seed_ctr.zero_()
        ts.zero_grad()
        self.graph = torch.cuda.CUDAGraph()
        self.loss, self.items = self._capture(self.graph)
        self.opt = DeviceOptimizerStep(ts.optimizer, ts.scaler, ts.ema, ts.raw_model, dev)    # on the graph's static .grad
        self.step_graph = self._capture_step()
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

    def _capture_step(self):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=self.graph.pool()):
            self.opt.enqueue()
        return graph

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
        if optimizer_step:                               # the next fresh replay overwrites the static gradients (zero_grad)
            if self.opt.stage():
                self.step_graph = self._capture_step()
            self.step_graph.replay()
        return loss.detach(), items

    def zero_grad(self) -> None:
        """Start a new accumulation window (train.py:291): the next call replays the fresh graph, which overwrites ``.grad``.
        The gradient tensors stay allocated, because both graphs write them in place."""
        self.fresh = True

    def close(self) -> None:
        _lib.lib().icaf_set_seed_offset(None)
