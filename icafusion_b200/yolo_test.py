"""Two-stream model builder: the ``Model`` / ``Detect`` / ``parse_model`` surface of the reference's
models/yolo_test.py, built on the icafusion_b200 operator classes.

``Model(cfg, ch=3, nc=None)`` accepts the reference's YAML row format (``[from, number, module, args]``) or a
stock name; ``model(rgb, ir)`` returns what the reference returns (eval: ``(z, logits, [x0,x1,x2])``).
The walk over the layer list follows Model.forward_once (yolo_test.py:136-163) -- ``f == -4`` routes the IR
image -- but runs on NHWC tensors and issues the RGB and IR streams as *grouped* launches (one kernel, two
filter banks), since both streams have identical geometry.
"""
from __future__ import annotations

import logging
import math
from copy import deepcopy
from typing import List, NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import ops
from .cfg import load_cfg
from .common import (C3, SPPF, Bottleneck, Concat, Conv, TransformerFusionBlock, Upsample, to_nchw, to_nhwc)
from .ops import ACT_NONE

logger = logging.getLogger(__name__)

_MODULES = {"Conv": Conv, "C3": C3, "SPPF": SPPF, "Bottleneck": Bottleneck, "Concat": Concat,
            "nn.Upsample": Upsample, "Upsample": Upsample, "TransformerFusionBlock": TransformerFusionBlock}


def make_divisible(x, divisor):
    """reference: utils/general.py:234-236"""
    return math.ceil(x / divisor) * divisor


class Detect(nn.Module):
    """Detection head (reference: models/yolo_test.py:26-70): per level a 1x1 Conv2d to na*(nc+5) channels,
    reshaped to (B,na,ny,nx,no); in eval additionally sigmoid + grid/anchor decode, concatenated over levels."""
    stride = None
    export = False

    def __init__(self, nc=80, anchors=(), ch=()):
        super().__init__()
        self.nc = nc
        self.no = nc + 5
        self.nl = len(anchors)
        self.na = len(anchors[0]) // 2
        self.grid = [torch.zeros(1)] * self.nl
        a = torch.tensor(anchors).float().view(self.nl, -1, 2)
        self.register_buffer("anchors", a)
        self.register_buffer("anchor_grid", a.clone().view(self.nl, 1, -1, 1, 1, 2))
        self.m = nn.ModuleList(nn.Conv2d(x, self.no * self.na, 1) for x in ch)

    def _packed(self, i):
        conv = self.m[i]
        key = (conv.weight.data_ptr(), conv.weight._version, conv.bias.data_ptr(), conv.bias._version)
        cache = self.__dict__.setdefault("_icaf_pack", {})
        if i not in cache or cache[i][0] != key:
            cache[i] = (key, ops.pack_conv_weight(conv.weight, conv.bias, 1, 0, ACT_NONE))
        return cache[i][1]

    def alloc_outputs(self, B: int, level_hw, device):
        """(z, logits, row offsets) for levels of spatial sizes level_hw = [(ny, nx), ...]."""
        rows = [self.na * ny * nx for ny, nx in level_hw]
        total = sum(rows)
        z = torch.empty(B, total, self.no, dtype=torch.float16, device=device)
        logits = torch.empty(B, total, self.no - 5, dtype=torch.float16, device=device)
        offs = [sum(rows[:i]) for i in range(len(rows))]
        return z, logits, offs

    def run_level(self, i: int, v: torch.Tensor, z, logits, off: int):
        """One detection level: 1x1 conv (yolo_test.py:49) + decode (:50-63) into rows [off, off+na*ny*nx) of z/logits."""
        if self.training:
            raise NotImplementedError("Detect.run_level is the inference path (decode); in train() call Detect.forward / autograd.detect")
        ag = self.anchor_grid
        key = (ag.data_ptr(), ag._version, ag.device)
        cache = self.__dict__.get("_icaf_anchor_px")
        if cache is None or cache[0] != key:       # host copy of anchor_grid (pixels); re-read when the buffer changes
            cache = (key, ag.detach().float().cpu().view(self.nl, -1).tolist())
            self.__dict__["_icaf_anchor_px"] = cache
        anchor_px = cache[1]
        p = ops.conv2d([v], [self._packed(i)])[0]
        return ops.detect_decode(p, self.na, self.no, z, logits, off, float(self.stride[i]), anchor_px[i])

    def run(self, vs: List[torch.Tensor]):
        """vs: NHWC maps of the nl levels."""
        z, logits, offs = self.alloc_outputs(vs[0].shape[0], [(v.shape[1], v.shape[2]) for v in vs], vs[0].device)
        xs = [self.run_level(i, v, z, logits, offs[i]) for i, v in enumerate(vs)]
        return z, logits, xs

    def forward(self, x):
        if self.training:                                  # yolo_test.py:49-51: the raw maps only
            from . import autograd
            return autograd.detect(self, [to_nhwc(t) for t in x])
        z, logits, xs = self.run([to_nhwc(t) for t in x])
        for i in range(self.nl):
            x[i] = xs[i]                 # the reference overwrites its input list in place (yolo_test.py:49-51)
        return z, logits, x


def check_anchor_order(m: "Detect") -> None:
    """Anchor areas must grow with the stride; flip the levels if the YAML lists them the other way round
    (reference: utils/autoanchor.py:12-20, called from Model.__init__, yolo_test.py:106)."""
    if m.anchor_grid.device.type == "meta":       # shape-only construction (torch.device("meta")): nothing to compare
        return
    a = m.anchor_grid.prod(-1).view(-1)
    if (a[-1] - a[0]).sign() != (m.stride[-1] - m.stride[0]).sign():
        m.anchors[:] = m.anchors.flip(0)
        m.anchor_grid[:] = m.anchor_grid.flip(0)


def fuse_conv_and_bn(conv: nn.Conv2d, bn: nn.BatchNorm2d) -> nn.Conv2d:
    """Fold an eval-mode BatchNorm into the preceding bias-free convolution
    (same result as the reference's utils/torch_utils.py:182-202)."""
    fused = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding,
                      groups=conv.groups, bias=True).requires_grad_(False).to(conv.weight.device, conv.weight.dtype)
    with torch.no_grad():
        scale = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).to(conv.weight.dtype)
        fused.weight.copy_(conv.weight * scale.view(-1, 1, 1, 1))
        b = conv.bias if conv.bias is not None else torch.zeros_like(bn.running_mean)
        fused.bias.copy_((b - bn.running_mean) * scale + bn.bias)
    return fused


def parse_model(d: dict, ch: List[int]):
    """Build the layer list from YAML rows (reference: models/yolo_test.py:216-302; the subset of module
    types the Transfusion configurations use)."""
    anchors, nc, gd, gw = d["anchors"], d["nc"], d["depth_multiple"], d["width_multiple"]
    na = (len(anchors[0]) // 2) if isinstance(anchors, list) else anchors
    no = na * (nc + 5)
    layers, save, c2 = [], [], ch[-1]
    for i, (f, n, m, args) in enumerate(d["backbone"] + d["head"]):
        name = m if isinstance(m, str) else m.__name__
        if name == "Detect":
            cls = Detect
        elif name in _MODULES:
            cls = _MODULES[name]
        else:
            raise NotImplementedError(f"parse_model: module '{name}' is outside the ICAFusion hot path built here")
        args = [nc if a == "nc" else anchors if a == "anchors" else (None if a == "None" else a) for a in args]
        n = max(round(n * gd), 1) if n > 1 else n
        if cls in (Conv, C3, SPPF, Bottleneck):
            c1 = 3 if (cls is Conv and args[0] == 64) else ch[f]      # yolo_test.py:242-246: both stems take an image
            c2 = args[0]
            if c2 != no:
                c2 = make_divisible(c2 * gw, 8)
            args = [c1, c2, *args[1:]]
            if cls is C3:
                args.insert(2, n)
                n = 1
        elif cls is Concat:
            c2 = sum(ch[x] for x in f)
        elif cls is Detect:
            args.append([ch[x] for x in f])
            if isinstance(args[1], int):
                args[1] = [list(range(args[1] * 2))] * len(f)
        elif cls is TransformerFusionBlock:
            c2 = ch[f[0]]
            args = [c2, *args[1:]]
        else:   # Upsample
            c2 = ch[f]
        m_ = nn.Sequential(*[cls(*args) for _ in range(n)]) if n > 1 else cls(*args)
        t = f"{cls.__module__}.{cls.__name__}"
        np_ = sum(x.numel() for x in m_.parameters())
        m_.i, m_.f, m_.type, m_.np = i, f, t, np_
        logger.info("%3s%18s%3s%10.0f  %-40s%-30s" % (i, f, n, np_, t, args))
        save.extend(x % i for x in ([f] if isinstance(f, int) else f) if x != -1)
        layers.append(m_)
        if i == 0:
            ch = []
        ch.append(c2)
    return nn.Sequential(*layers), sorted(save)


class LayerPlan(NamedTuple):
    """What the inference and training layer walks need to know about the layer list, derived from it once.

    ir_start:  index of the IR stream's first layer (the one layer with from == -4) when the IR stream mirrors the RGB
               stream layer by layer, so that layers k and ir_start + k run as one grouped launch; else None.
    srcs:      per layer, the indices of the layers it reads (-1 and other relative indices resolved); () for a layer
               fed an image (the RGB stem, or from == -4: the IR stem).
    ch:        per layer, its output channels (None for Detect).
    stride:    per layer, the input image's size over its output's (Conv strides, Upsample x2).
    dst:       per layer, (Concat layer, channel offset) when the layer writes its output straight into that slice of
               the Concat's buffer (see plan_layers), else None.
    side_dmff: the DMFF blocks whose inputs all lie in the two backbones: they may run on a side stream."""
    ir_start: Optional[int]
    srcs: Tuple[Tuple[int, ...], ...]
    ch: Tuple[Optional[int], ...]
    stride: Tuple[Optional[int], ...]
    dst: Tuple[Optional[Tuple[int, int]], ...]
    side_dmff: Tuple[int, ...]


def plan_layers(layers) -> LayerPlan:
    """The LayerPlan of a parsed layer list.  Concat elimination (`dst`): every tensor that feeds a Concat layer is produced
    directly inside that layer's output buffer (all kernels take channel-slice views), so the Concat itself launches
    nothing.  A producer feeding two concats keeps the first and is copied for the rest; the two streams' layers, which run
    as grouped launches, are never producers."""
    layers = list(layers)
    starts = [m.i for m in layers if m.f == -4]
    ir = starts[0] if len(starts) == 1 and 2 * starts[0] <= len(layers) else None

    def sig(m):
        return (type(m), [tuple(p.shape) for p in m.parameters()])
    for k in range(ir or 0):                      # the IR stream must mirror the RGB stream layer by layer
        a, b = layers[k], layers[ir + k]
        if sig(a) != sig(b) or (k > 0 and (a.f != -1 or b.f != -1)):
            ir = None
            break
    paired = 2 * ir if ir is not None else 0
    n = len(layers)
    srcs, ch, stride, dst = [()] * n, [None] * n, [None] * n, [None] * n
    for m in layers:
        i = m.i
        if i > 0 and m.f != -4:
            srcs[i] = tuple(j % i for j in ([m.f] if isinstance(m.f, int) else m.f))
        s_in = stride[srcs[i][0]] if srcs[i] else 1
        stride[i] = (s_in * m.conv.stride[0] if isinstance(m, Conv) else s_in // 2 if isinstance(m, nn.Upsample) else
                     None if isinstance(m, Detect) else s_in)
        if isinstance(m, Conv):
            ch[i] = m.conv.out_channels
        elif isinstance(m, C3):
            ch[i] = m.cv3.conv.out_channels
        elif isinstance(m, SPPF):
            ch[i] = m.cv2.conv.out_channels
        elif isinstance(m, TransformerFusionBlock):
            ch[i] = m.n_embd
        elif isinstance(m, nn.Upsample):
            ch[i] = ch[srcs[i][0]]
        elif isinstance(m, Concat):
            if m.d == 1 and not isinstance(m.f, int) and \
                    all(ch[j] and j >= paired and dst[j] is None and not isinstance(layers[j], (Concat, Detect)) for j in srcs[i]):
                off = 0
                for j in srcs[i]:
                    dst[j] = (i, off)
                    off += ch[j]
            ch[i] = sum(ch[j] for j in srcs[i])
    side_dmff = tuple(m.i for m in layers[paired:] if isinstance(m, TransformerFusionBlock) and not isinstance(m.f, int)
                      and all(j < paired for j in srcs[m.i]))
    return LayerPlan(ir, tuple(srcs), tuple(ch), tuple(stride), tuple(dst), side_dmff)


class Model(nn.Module):
    """reference: models/yolo_test.py:73-213"""

    def __init__(self, cfg="yolov5s_Transfusion_kaist", ch=3, nc=None, anchors=None):
        super().__init__()
        self.yaml = load_cfg(cfg)
        ch = self.yaml["ch"] = self.yaml.get("ch", ch)
        if nc and nc != self.yaml["nc"]:
            logger.info(f"Overriding model.yaml nc={self.yaml['nc']} with nc={nc}")
            self.yaml["nc"] = nc
        if anchors:
            self.yaml["anchors"] = round(anchors)
        self.model, self.save = parse_model(deepcopy(self.yaml), ch=[ch])
        self.names = [str(i) for i in range(self.yaml["nc"])]
        m = self.model[-1]
        if isinstance(m, Detect):
            m.stride = torch.Tensor([8.0, 16.0, 32.0])              # yolo_test.py:104 (hard-coded in the reference)
            m.anchors /= m.stride.view(-1, 1, 1)
            check_anchor_order(m)
            self.stride = m.stride
        for mod in self.modules():                                    # utils/torch_utils.py:144-154
            if type(mod) is nn.BatchNorm2d:
                mod.eps = 1e-3
                mod.momentum = 0.03
        self._plan = plan_layers(self.model)

    def _layer_plan(self) -> LayerPlan:
        if "_plan" not in self.__dict__:          # an unpickled checkpoint (models/experimental.py:118) never ran __init__
            self._plan = plan_layers(self.model)
        return self._plan

    @property
    def _ir_start(self):
        """Index of the IR stream's first layer, or None when the two streams do not pair up (see plan_layers)."""
        return self._layer_plan().ir_start

    def forward(self, x, x2, augment=False, profile=False):
        if augment:
            raise NotImplementedError("augmented (multi-scale / flip) inference is outside the hot path built here")
        if tuple(x.shape) != tuple(x2.shape):
            raise ValueError(f"RGB and IR batches must share one shape, got {tuple(x.shape)} and {tuple(x2.shape)}")
        smax = int(self.stride.max()) if hasattr(self, "stride") else 32
        if x.dim() != 4 or x.shape[2] % smax or x.shape[3] % smax:
            # the reference fails at torch.cat for such inputs (models/common.py:321); here the concat buffers are planned
            # from the stride pyramid, so reject up front
            raise ValueError(f"image height and width must be multiples of the maximum stride {smax}, got {tuple(x.shape)}")
        return self.forward_once(x, x2, profile)

    def forward_once(self, x, x2, profile=False):
        if self.training:                           # train.py:336: the list of raw Detect maps, with an autograd graph
            from . import autograd
            return autograd.model_forward(self, x, x2)
        z, logits, xs = self._forward_nhwc(x, x2)
        return z, logits, xs

    @staticmethod
    def _run_layer(ms, xs, out=None):
        """Run one layer, ms = [m], on the NHWC maps xs of its sources; or the twin layers ms = [rgb, ir] of the two
        streams, one map each, as grouped launches.  `out`: the view a single layer writes into.  Returns one map per
        module.  (Detect runs level by level in the walk.)"""
        m, outs = ms[0], None if out is None else [out]
        if isinstance(m, Conv):
            return Conv.run(ms, xs, outs)
        if isinstance(m, C3):
            return C3.run(ms, xs, outs)
        if isinstance(m, SPPF):
            return SPPF.run(ms, xs, outs)
        if isinstance(m, nn.Upsample):             # ours, or torch's own class inside an unpickled reference checkpoint
            if m.mode != "nearest" or m.scale_factor is None or float(m.scale_factor) != 2.0:
                raise NotImplementedError("Upsample: only nearest x2 is supported")
            return [ops.upsample2x(xs[0], out)]
        if isinstance(m, Concat):
            return [Concat.run(xs)]
        if isinstance(m, TransformerFusionBlock):
            return [m.run(xs[0], xs[1], out)]
        raise NotImplementedError(type(m).__name__)

    def _stage(self, img, stem):
        """Image staging for the stem layer `stem` (a Conv taking the 3-channel image)."""
        if img.dim() != 4 or img.shape[1] != 3:
            raise ValueError(f"expected (B,3,H,W) images, got {tuple(img.shape)}")
        if not ops.on_device(img):
            raise RuntimeError("icafusion_b200 runs on CUDA tensors only (no CPU fallback)")
        if isinstance(stem, Conv) and stem.conv.in_channels == 3:
            return stem.stage_image(img)
        if img.dtype not in (torch.float16, torch.float32, torch.uint8):
            img = img.float()
        return ops.pack_image(img, 1.0 / 255.0 if img.dtype == torch.uint8 else 1.0)

    def _side_streams(self, device, n: int):
        pool = self.__dict__.setdefault("_icaf_streams", {})
        lst = pool.setdefault(device, [])
        while len(lst) < n:
            lst.append(torch.cuda.Stream(device))
        return lst

    def _forward_nhwc(self, rgb, ir):
        """Layer walk with branch-level concurrency: the RGB/IR streams run as grouped launches on the current stream;
        a side-stream DMFF block is forked as soon as both of its inputs exist (P3 and P4 fusion overlap the rest of the
        backbone; the last block feeds the head directly and stays in order), every Detect level but the last is forked as
        soon as its input exists; consumers join before they read, and the end of the walk joins whatever is left."""
        plan = self._layer_plan()
        if not (ops.on_device(rgb) and ops.on_device(ir)):     # before any stream lookup: torch rejects a CPU device there
            raise RuntimeError("icafusion_b200 runs on CUDA tensors only (no CPU fallback)")
        layers = list(self.model)
        y: List = [None] * len(layers)
        dev = rgb.device
        B, H, W = rgb.shape[0], rgb.shape[2], rgb.shape[3]
        dry = ops.dry_running()                   # shape-only walk on meta tensors (no streams, nothing launched)
        main = None if dry else torch.cuda.current_stream(dev)
        forked = {}                               # layer index (or Detect level) -> side stream its result is produced on
        n_side = 0
        concurrent = self.__dict__.get("_icaf_concurrent", True) and not dry

        def fork(key):
            nonlocal n_side
            st = self._side_streams(dev, n_side + 1)[n_side]
            n_side += 1
            st.wait_stream(main)
            forked[key] = st
            return torch.cuda.stream(st)

        def join(keys):
            for k in keys:
                st = forked.pop(k, None)
                if st is not None:
                    main.wait_stream(st)

        cats = {}                                 # concat layer index -> its output buffer, allocated by its first producer

        def dest(i):
            """The slice of its Concat's buffer layer i writes into (or None); allocated on the main stream."""
            if plan.dst[i] is None:
                return None
            c, off = plan.dst[i]
            if c not in cats:
                s = plan.stride[i]
                cats[c] = torch.empty(B, H // s, W // s, plan.ch[c], dtype=torch.float16, device=dev)
            return cats[c][..., off:off + plan.ch[i]]

        arena = self.__dict__.get("_icaf_arena")
        if concurrent and arena is not None and arena.numel() * 2 <= (96 << 20):
            # the whole packed filter set fits the 126 MB L2: stream it in once, concurrently with the first layers
            with fork("prefetch"):
                ops.prefetch_l2(arena)
        ir_first = next((m for m in layers if m.f == -4), layers[0])
        images = self._stage(rgb, layers[0]), self._stage(ir, ir_first)
        side_dmff = plan.side_dmff[:-1] if concurrent else ()
        s = plan.ir_start or 0
        for k in range(s):                        # both streams, one grouped launch per operator
            y[k], y[s + k] = self._run_layer([layers[k], layers[s + k]], [y[k - 1], y[s + k - 1]] if k else images)
            for i in side_dmff:
                if y[i] is None and all(y[j] is not None for j in plan.srcs[i]):
                    out = dest(i)
                    with fork(i):
                        y[i] = self._run_layer([layers[i]], [y[j] for j in plan.srcs[i]], out)[0]

        det = layers[-1] if isinstance(layers[-1], Detect) else None
        det_srcs = plan.srcs[-1] if det is not None else ()
        det_early = det_srcs[:-1] if concurrent else ()     # forked as their input appears; the last level closes the forward
        det_out = None                            # (z, logits, row offsets, level maps)

        def det_outputs():
            nonlocal det_out
            if det_out is None:
                z, logits, offs = det.alloc_outputs(B, [(H // plan.stride[j], W // plan.stride[j]) for j in det_srcs], dev)
                det_out = (z, logits, offs, [None] * len(det_srcs))
            return det_out

        for m in layers[2 * s:]:
            i = m.i
            if y[i] is not None:                  # a DMFF block forked during the streams
                continue
            join(plan.srcs[i])
            if m is det:
                z, logits, offs, maps = det_outputs()
                for lvl, j in enumerate(det_srcs):
                    if maps[lvl] is None:
                        maps[lvl] = m.run_level(lvl, y[j], z, logits, offs[lvl])
                y[i] = (z, logits, maps)
            elif isinstance(m, Concat) and i in cats:
                y[i] = cats[i]                    # every source already wrote its slice
            else:
                xs = [y[j] for j in plan.srcs[i]] if plan.srcs[i] else [images[1] if m.f == -4 else images[0]]
                y[i] = self._run_layer([m], xs, dest(i))[0]
            if i in det_early:
                z, logits, offs, maps = det_outputs()
                lvl = det_srcs.index(i)
                with fork(("det", lvl)):
                    maps[lvl] = det.run_level(lvl, y[i], z, logits, offs[lvl])
        join(list(forked))                        # nothing may outlive the forward on a side stream
        return y[-1]

    def consolidate_weights(self, rgb, ir):
        """Run one forward on (rgb, ir), collect every packed filter it touches and move them into one contiguous arena
        (enables the per-step L2 prefetch).  Call again after the parameters change (re-packing creates new tensors)."""
        with ops.trace_weights() as tr:
            self._forward_nhwc(rgb, ir)
        self.__dict__["_icaf_arena"] = ops.consolidate_weights(tr.items)
        return self.__dict__["_icaf_arena"]

    def fuse(self):
        """Fold every Conv's BatchNorm (reference: models/yolo_test.py:182-190)."""
        for m in self.model.modules():
            if type(m) is Conv and hasattr(m, "bn"):
                m.conv = fuse_conv_and_bn(m.conv, m.bn)
                delattr(m, "bn")
                m.forward = m.fuseforward
                m.__dict__.pop("_icaf_pack", None)
        return self

    def info(self, verbose=False, img_size=640):
        n_p = sum(x.numel() for x in self.parameters())
        logger.info(f"Model Summary: {len(list(self.modules()))} layers, {n_p} parameters")
