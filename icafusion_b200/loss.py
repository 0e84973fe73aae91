"""Detection loss with the reference's name and call signature (utils/loss.py:325-463), forward on the device.

``ComputeLoss(model)(p, targets)`` returns ``(loss * batch_size, cat(lbox, lobj, lcls, lrk))`` like the reference.  This is
the use test.py:132-133 (validation loss) and train.py:338-344 (training loss + backward) make of it: when a prediction
requires grad the returned loss carries an autograd node whose backward launches icaf_compute_loss_bwd.  Target assignment,
CIoU, both BCE terms, the reductions and their gradients run as kernels of libicaf_b200 (csrc/loss.cu) with no host sync.
``hyp['fl_gamma'] > 0`` wraps both BCE terms in the reference's FocalLoss (alpha 0.25, loss.py:37-64, 341-344) on the device.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import torch

from . import _lib, ops


def smooth_BCE(eps: float = 0.1):
    """reference: utils/loss.py:15-17"""
    return 1.0 - 0.5 * eps, 0.5 * eps


class ComputeLoss:
    def __init__(self, model, autobalance: bool = False):
        if autobalance:
            raise NotImplementedError("ComputeLoss: autobalance needs a host read per level and step; not built")
        m = model.module if hasattr(model, "module") else model
        h = m.hyp                                            # train.py:229 attaches the hyper-parameter dict to the model
        det = m.model[-1]
        self.na, self.nc, self.nl = det.na, det.nc, det.nl
        self.anchors = det.anchors.detach().float().cpu().reshape(-1).tolist()      # grid units, (nl, na, 2)
        cp, cn = smooth_BCE(eps=h.get("label_smoothing", 0.0))
        balance = {3: [4.0, 1.0, 0.4]}.get(det.nl, [4.0, 1.0, 0.25, 0.06, 0.02])    # loss.py:346
        self.hyp = _lib.LossHyp(float(h["box"]), float(h["obj"]), float(h["cls"]), float(h["cls_pw"]), float(h["obj_pw"]),
                                float(h["anchor_t"]), float(h.get("fl_gamma", 0.0)), float(getattr(m, "gr", 1.0)), cp, cn,
                                (C.c_float * 5)(*(balance + [0.0] * 5)[:5]))

    # -- one launch group, forward or backward ----------------------------------------------------
    def _layout(self, p: Sequence[torch.Tensor]):
        """-> (p_ld, tensors whose data_ptr is the level's base).  p_ld = 0: (B, na, ny, nx, no) contiguous; otherwise every
        level is a permuted view of the head's own NHWC map (B, ny, nx, na*no [+ pad]) with pixel pitch p_ld."""
        B, na, ny, nx, no = p[0].shape
        if all(t.is_contiguous() for t in p):
            return 0, list(p)
        ld = p[0].stride(3)
        for t in p:
            _, _, ny, nx, _ = t.shape
            if t.stride() != (ny * nx * ld, no, nx * ld, ld, 1):
                return 0, [t.contiguous() for t in p]
        return ld, list(p)

    def _launch(self, ps, p_ld, tg, out=None, ws=None, grad_out=None, dps=None):
        nl = len(ps)
        B, na, _, _, no = ps[0].shape
        dev, dt = ps[0].device, ps[0].dtype
        nt = int(tg.shape[0])
        ny = (C.c_int * nl)(*[t.shape[2] for t in ps])
        nx = (C.c_int * nl)(*[t.shape[3] for t in ps])
        if ws is None:
            need = int(_lib.lib().icaf_loss_workspace_bytes(B, na, nt, ny, nx, nl, no if self.with_backward else 0))
            ws = torch.empty((need + 7) // 8, dtype=torch.int64, device=dev)
        ptrs = (C.c_void_p * nl)(*[t.data_ptr() for t in ps])
        anch = (C.c_float * len(self.anchors))(*self.anchors)
        head = (ptrs, 1 if dt == torch.float32 else 0, p_ld, ny, nx, nl, B, na, no, ops._ptr(tg if nt else None), nt, anch, C.byref(self.hyp))
        work = {"bytes": float(sum(t.numel() * t.element_size() for t in ps))}
        if grad_out is None:
            ops._call("icaf_compute_loss_fwd", _lib.lib().icaf_compute_loss_fwd, head + (ops._ptr(out), ops._ptr(ws), C.c_size_t(ws.numel() * 8)), work)
        else:
            dptrs = (C.c_void_p * nl)(*[t.data_ptr() for t in dps])
            ops._call("icaf_compute_loss_bwd", _lib.lib().icaf_compute_loss_bwd,
                      head + (ops._ptr(grad_out), dptrs, ops._ptr(ws), C.c_size_t(ws.numel() * 8)), work)
        return ws

    def __call__(self, p: Sequence[torch.Tensor], targets: torch.Tensor):
        nl = len(p)
        if nl != self.nl:
            raise ValueError(f"ComputeLoss: {nl} prediction levels, Detect has {self.nl}")
        dev = p[0].device
        if not ops.on_device(p[0]):
            raise RuntimeError("icafusion_b200 runs on CUDA tensors only (no CPU fallback)")
        dt = p[0].dtype
        if dt not in (torch.float16, torch.float32) or any(t.dtype != dt for t in p):
            raise ValueError("ComputeLoss: predictions must all be fp16 or all fp32")
        B, na, _, _, no = p[0].shape
        if na != self.na or no != self.nc + 5:
            raise ValueError(f"ComputeLoss: predictions are (B, {na}, ny, nx, {no}), Detect has na={self.na}, nc={self.nc}")
        tg = targets.detach().to(dev, torch.float32).contiguous()
        self.with_backward = torch.is_grad_enabled() and any(t.requires_grad for t in p)
        out = _LossFn.apply(self, tg, *p)
        return out[0:1], out[1:5].detach()


class _LossFn(torch.autograd.Function):
    """loss.py:325-398 forward and its backward (train.py:344 starts here) as two launch groups of csrc/loss.cu."""

    @staticmethod
    def forward(ctx, crit: ComputeLoss, tg: torch.Tensor, *p):
        p_ld, ps = crit._layout([t.detach() for t in p])
        out = torch.empty(5, dtype=torch.float32, device=tg.device)
        ws = crit._launch(ps, p_ld, tg, out=out)
        ctx.crit, ctx.p_ld, ctx.tg, ctx.ws, ctx.ps = crit, p_ld, tg, ws, ps
        ctx.with_backward = crit.with_backward
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.with_backward:
            raise RuntimeError("ComputeLoss: the forward ran without a backward workspace")
        crit, ps, p_ld = ctx.crit, ctx.ps, ctx.p_ld
        g = grad_out.detach().to(torch.float32).contiguous()            # d / d out[0] is the first element
        if p_ld:      # gradient in the head map's own memory; pad channels (pitch > na*no) must read as zero downstream
            dps = []
            for t in ps:
                B, na, ny, nx, no = t.shape
                buf = torch.zeros(B, ny, nx, p_ld, dtype=t.dtype, device=t.device) if p_ld > na * no else \
                    torch.empty(B, ny, nx, p_ld, dtype=t.dtype, device=t.device)
                dps.append(buf.as_strided(t.shape, t.stride()))
        else:
            dps = [torch.empty_like(t) for t in ps]
        crit._launch(ps, p_ld, ctx.tg, ws=ctx.ws, grad_out=g, dps=dps)
        return (None, None) + tuple(dps)
