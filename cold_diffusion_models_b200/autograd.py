"""torch.autograd bridge: lets `loss.backward()` (Trainer.train, DB:1190-1196) drive the engine's
backward schedule.  The Function's gradient w.r.t. parameters is written by the kernels directly into the
flat gradient buffer whose views are the parameters' `.grad`, so nothing is returned to autograd for them.
The gradient w.r.t. the input `x` is returned when `x` requires it; frozen parameters (requires_grad=False)
get no gradient and cost no weight-gradient launch.
The Functions of the degradations D(x, t) below give `GaussianDiffusion.degrade` of every package its backward."""
import ctypes as C

import torch
from torch.autograd.function import once_differentiable

from ._lib import call, ptr, stream


def check_first_order(dout, what):
    """the engine's backward is not itself differentiable: refuse create_graph=True instead of returning a gradient
    whose own derivative would be wrong"""
    if dout.requires_grad:
        raise RuntimeError("%s: the engine backward is first order only; create_graph=True (second derivatives) is not "
                           "supported" % what)


def trainable_names(named_params, needs_input_grad):
    """names of the parameters that require a gradient, from the Function's needs_input_grad (parameters are inputs 3..)"""
    return [n for (n, _), need in zip(named_params, needs_input_grad[3:]) if need]


class UnetFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, unet, x, time, *params):
        eng = unet.engine
        save = {}
        out = eng.forward(x, time, save=save)
        ctx.unet = unet
        ctx.save = save
        ctx.nparams = len(params)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        check_first_order(dout, "Unet backward")
        eng = ctx.unet.engine
        eng.attach_grads()
        need_dx = ctx.needs_input_grad[1]
        dx = eng.backward(ctx.save, dout, need_dx=need_dx,
                          trainable=trainable_names(ctx.unet.named_parameters(), ctx.needs_input_grad))
        ctx.save = None
        return (None, dx if need_dx else None, None) + (None,) * ctx.nparams


# ==========================================================================================================================
# Degradations D(x, t) (`GaussianDiffusion.degrade` of every package).  Each forward launches the kernel `q_sample` launches,
# so the values are q_sample's bit for bit; each backward is the adjoint of that linear map, first order only.
# ==========================================================================================================================
def wants_grad(*xs):
    return torch.is_grad_enabled() and any(x is not None and x.requires_grad for x in xs)


def refuse_grad(what, *xs):
    """`what` has no usable derivative: raise when a gradient of it is requested (the forward alone stays allowed)"""
    if wants_grad(*xs):
        raise RuntimeError("degrade: %s is not differentiable; call it under torch.no_grad() or on inputs that do not "
                           "require grad" % what)


class BlurDegrade(torch.autograd.Function):
    """out = A_{t_b} x A_{t_b}^T per plane (cd_blur_apply); dx = A^T g A (cd_blur_apply_adjoint).  t: int64 (B,) or None
    (t_scalar for every sample).  quantize must be 0 when x requires grad (see refuse_grad)."""

    @staticmethod
    def forward(ctx, x, ops, t, t_scalar, T, collapse, quantize):
        B, Cc, S, _ = x.shape
        out = torch.empty_like(x)
        call('cd_blur_apply', ptr(x), ptr(out), ptr(ops), ptr(t), int(t_scalar), B, Cc, S, T, int(collapse), int(quantize), stream())
        ctx.args = (ops, t, int(t_scalar), T, int(collapse))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        check_first_order(dout, "degrade backward")
        ops, t, t_scalar, T, collapse = ctx.args
        g = dout.contiguous()
        B, Cc, S, _ = g.shape
        dx = torch.empty_like(g)
        call('cd_blur_apply_adjoint', ptr(g), ptr(dx), ptr(ops), ptr(t), t_scalar, B, Cc, S, T, collapse, stream())
        return dx, None, None, None, None, None, None


class MaskDegrade(torch.autograd.Function):
    """out = x * M[t_b] in each sample's window (cd_mask_apply); the product is self-adjoint: dx = g * M[t_b]"""

    @staticmethod
    def forward(ctx, x, masks, t, rx, ry, quantize):
        B, Cc, S, _ = x.shape
        out = torch.empty_like(x)
        call('cd_mask_apply', ptr(x), ptr(out), ptr(masks), ptr(t), 0, ptr(rx), ptr(ry), B, Cc, S, masks.shape[-1], int(quantize),
             stream())
        ctx.args = (masks, t, rx, ry)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        check_first_order(dout, "degrade backward")
        masks, t, rx, ry = ctx.args
        g = dout.contiguous()
        B, Cc, S, _ = g.shape
        dx = torch.empty_like(g)
        call('cd_mask_apply', ptr(g), ptr(dx), ptr(masks), ptr(t), 0, ptr(rx), ptr(ry), B, Cc, S, masks.shape[-1], 0, stream())
        return dx, None, None, None, None, None


class LerpDegrade(torch.autograd.Function):
    """out = wa[w] x1 + wb[w] x2 with per-sample scalars (per_pixel = 0: cd_noise_lerp, w = t_b) or per-pixel tables
    (per_pixel = 1: cd_fade_lerp, w = (t_b, pixel)); both gradients come from one cd_lerp2_adjoint pass"""

    @staticmethod
    def forward(ctx, x1, x2, t, t_scalar, wa, wb, per_pixel):
        B, Cc, H, W = x1.shape
        out = torch.empty_like(x1)
        if per_pixel:
            call('cd_fade_lerp', ptr(x1), ptr(x2), ptr(t), int(t_scalar), ptr(wa), ptr(wb), B, Cc, H * W, ptr(out), stream())
        else:
            call('cd_noise_lerp', ptr(x1), ptr(x2), ptr(t), int(t_scalar), ptr(wa), ptr(wb), C.c_int64(x1[0].numel()),
                 C.c_int64(x1.numel()), ptr(out), stream())
        ctx.args = (t, int(t_scalar), wa, wb, int(per_pixel))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        check_first_order(dout, "degrade backward")
        t, t_scalar, wa, wb, per_pixel = ctx.args
        g = dout.contiguous()
        B, Cc, H, W = g.shape
        g1 = torch.empty_like(g) if ctx.needs_input_grad[0] else None
        g2 = torch.empty_like(g) if ctx.needs_input_grad[1] else None
        if g1 is not None or g2 is not None:
            call('cd_lerp2_adjoint', ptr(g), ptr(t), t_scalar, ptr(wa), ptr(wb), B, Cc, C.c_int64(H * W), per_pixel, ptr(g1), ptr(g2),
                 stream())
        return g1, g2, None, None, None, None, None


class ChanmixDegrade(torch.autograd.Function):
    """out = M[t_b] x per pixel (cd_chanmix mode 0); dx = M[t_b]^T g through the same kernel with the transposed table"""

    @staticmethod
    def forward(ctx, x, mats, mats_t, t):
        B, Cc, H, W = x.shape
        out = torch.empty_like(x)
        call('cd_chanmix', ptr(None), ptr(x), ptr(out), ptr(mats), ptr(t), ptr(None), 0, 0, B, Cc, C.c_int64(H * W), 0, stream())
        ctx.args = (mats_t, t)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        check_first_order(dout, "degrade backward")
        mats_t, t = ctx.args
        g = dout.contiguous()
        B, Cc, H, W = g.shape
        dx = torch.empty_like(g)
        call('cd_chanmix', ptr(None), ptr(g), ptr(dx), ptr(mats_t), ptr(t), ptr(None), 0, 0, B, Cc, C.c_int64(H * W), 0, stream())
        return dx, None, None, None
