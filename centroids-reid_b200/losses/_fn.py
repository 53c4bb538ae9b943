"""torch.autograd bridges to the fused forward+backward C-ABI loss kernels.

Every C entry point computes the loss value AND the gradient of that value in one enqueue;
the autograd.Function stores the gradient and scales it by grad_output in backward().
"""
from __future__ import annotations

import ctypes as C

import torch

from .. import _native as N


def _i32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.int32).contiguous()


def _u8(t):
    return None if t is None else t.detach().to(torch.uint8).contiguous()


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().float().contiguous()


_CONTRACT = {1: "a label is outside [0, num_classes)", 2: "labels are not constant inside a block of K rows (the batch is "
             "not pid-major)", 3: "the same label appears in two blocks of K rows"}


def raise_if_poisoned(value: torch.Tensor, what: str):
    """The loss kernels report a violated input contract as a NaN with a payload (no host synchronisation inside the
    step); this reads ONE float back and turns it into the exception the reference's asserts would raise."""
    v = value.detach().reshape(-1)[:1].float()
    if bool(torch.isnan(v)):
        code = int(v.view(torch.int32).item()) & 0x3FFFFF
        if code in _CONTRACT:
            raise ValueError(f"{what}: {_CONTRACT[code]} (datasets/bases.py:346-406 batch contract; "
                             "losses/center_loss.py:32 label range)")
        raise FloatingPointError(f"{what}: the loss is NaN (non-finite features?)")


class TripletFn(torch.autograd.Function):
    """losses/triplet_loss.py:139-173 (euclidean, MarginRankingLoss) -> loss, dist_ap, dist_an."""

    @staticmethod
    def forward(ctx, feats, labels, mask, margin, soft=False, cosine=False):
        N.require_cuda(feats, labels)
        f = _f32(feats)
        n, d = f.shape
        L = N.lib()
        dev = f.device
        loss = torch.empty(1, device=dev)
        ap = torch.empty(n, device=dev)
        an = torch.empty(n, device=dev)
        grad = torch.empty_like(f)
        ws_bytes = L.ctl_triplet_workspace_bytes(n, d)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        lab, m = _i32(labels), _u8(mask)
        with torch.cuda.device(dev):
            N.check(L.ctl_triplet_step_ex(f.data_ptr(), n, d, lab.data_ptr(), N.ptr(m), float(margin or 0.0), int(soft),
                                          int(cosine), loss.data_ptr(), ap.data_ptr(), an.data_ptr(), grad.data_ptr(),
                                          ws.data_ptr(), ws_bytes, N.stream_ptr()))
        ctx.save_for_backward(grad)
        ctx.in_dtype = feats.dtype
        ctx.mark_non_differentiable(ap, an)
        return loss[0], ap, an

    @staticmethod
    def backward(ctx, g_loss, g_ap, g_an):
        (grad,) = ctx.saved_tensors
        return (grad * g_loss).to(ctx.in_dtype), None, None, None, None, None


class CenterLossFn(torch.autograd.Function):
    """losses/center_loss.py:26-45."""

    @staticmethod
    def forward(ctx, x, centers, labels):
        N.require_cuda(x, centers, labels)
        xf, cf = _f32(x), _f32(centers)
        b, d = xf.shape
        c = cf.shape[0]
        L = N.lib()
        dev = xf.device
        loss = torch.empty(1, device=dev)
        dx = torch.empty_like(xf)
        dc = torch.empty_like(cf)
        ws_bytes = 4 * (b * 4 + 256) + 1024
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        lab = _i32(labels)
        with torch.cuda.device(dev):
            N.check(L.ctl_center_loss_step(xf.data_ptr(), b, d, lab.data_ptr(), cf.data_ptr(), c, loss.data_ptr(),
                                           dx.data_ptr(), dc.data_ptr(), ws.data_ptr(), ws_bytes, N.stream_ptr()))
        ctx.save_for_backward(dx, dc)
        ctx.in_dtype = x.dtype
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        dx, dc = ctx.saved_tensors
        return (dx * g).to(ctx.in_dtype), dc * g, None


class XentSmoothFn(torch.autograd.Function):
    """losses/triplet_loss.py:194-205."""

    @staticmethod
    def forward(ctx, logits, targets, epsilon):
        N.require_cuda(logits, targets)
        z = _f32(logits)
        b, c = z.shape
        L = N.lib()
        dev = z.device
        loss = torch.empty(1, device=dev)
        dz = torch.empty_like(z)
        ws_bytes = b * 4 + 512
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        t = _i32(targets)
        with torch.cuda.device(dev):
            N.check(L.ctl_xent_smooth_step(z.data_ptr(), b, c, t.data_ptr(), float(epsilon), loss.data_ptr(),
                                           dz.data_ptr(), ws.data_ptr(), ws_bytes, N.stream_ptr()))
        ctx.save_for_backward(dz)
        ctx.in_dtype = logits.dtype
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dz,) = ctx.saved_tensors
        return (dz * g).to(ctx.in_dtype), None, None


def _fused_step(ctx, n_out, workspace_bytes, step, feats, centers, bn_weight, fc_weight, bn_bias, run_mean, run_var,
                labels, is_real, cfg):
    """Shared forward of the fused loss steps (ctl_loss_step, ctl_base_loss_step): one enqueue fills out[n_out] and the
    gradients of out[0], which are saved for backward."""
    N.require_cuda(feats, centers, bn_weight, fc_weight, labels, is_real)
    f, c, bw, fw = _f32(feats), _f32(centers), _f32(bn_weight), _f32(fc_weight)
    bb = _f32(bn_bias)
    dev = f.device
    out = torch.zeros(n_out, device=dev)
    d_f, d_c, d_bw, d_fw = torch.empty_like(f), torch.empty_like(c), torch.empty_like(bw), torch.empty_like(fw)
    ws_bytes = workspace_bytes(C.byref(cfg))
    if ws_bytes == 0:
        N.check(-1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    lab, real = _i32(labels), _u8(is_real)
    with torch.cuda.device(dev):
        N.check(step(C.byref(cfg), f.data_ptr(), lab.data_ptr(), real.data_ptr(), c.data_ptr(), bw.data_ptr(),
                     bb.data_ptr(), N.ptr(run_mean), N.ptr(run_var), fw.data_ptr(), out.data_ptr(), d_f.data_ptr(),
                     d_c.data_ptr(), d_bw.data_ptr(), d_fw.data_ptr(), ws.data_ptr(), ws_bytes, N.stream_ptr()))
    ctx.save_for_backward(d_f, d_c, d_bw, d_fw)
    ctx.in_dtype = feats.dtype
    parts = out.detach()
    ctx.mark_non_differentiable(parts)
    return out[0], parts


class CTLStepFn(torch.autograd.Function):
    """Everything between the trunk and manual_backward in CTLModel.training_step
    (train_ctl_model.py:54-152): returns (total, parts[8]) with gradients w.r.t.
    (features, centers, bn.weight, fc_query.weight)."""

    @staticmethod
    def forward(ctx, feats, centers, bn_weight, fc_weight, bn_bias, run_mean, run_var, labels, is_real, cfg):
        L = N.lib()
        return _fused_step(ctx, 8, L.ctl_loss_workspace_bytes, L.ctl_loss_step, feats, centers, bn_weight, fc_weight,
                           bn_bias, run_mean, run_var, labels, is_real, cfg)

    @staticmethod
    def backward(ctx, g_total, g_parts):
        d_f, d_c, d_bw, d_fw = ctx.saved_tensors
        return ((d_f * g_total).to(ctx.in_dtype), d_c * g_total, d_bw * g_total, d_fw * g_total,
                None, None, None, None, None, None)


class BaseStepFn(CTLStepFn):
    """Everything between the trunk and manual_backward in the base model's training_step
    (train_base_model.py:57-75): returns (total, parts[6] = total, xent, triplet, center, dist_ap, dist_an) with
    gradients w.r.t. (features, centers, bn.weight, fc_query.weight); `cfg` is an N.BaseLossConfig.  Unlike the CTL step,
    every row enters the center loss and the head; `is_real` only masks the triplet anchors."""

    @staticmethod
    def forward(ctx, feats, centers, bn_weight, fc_weight, bn_bias, run_mean, run_var, labels, is_real, cfg):
        L = N.lib()
        return _fused_step(ctx, 6, L.ctl_base_loss_workspace_bytes, L.ctl_base_loss_step, feats, centers, bn_weight,
                           fc_weight, bn_bias, run_mean, run_var, labels, is_real, cfg)
