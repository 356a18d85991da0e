"""torch.autograd bridge: lets `loss.backward()` (Trainer.train, DB:1190-1196) drive the engine's
backward schedule.  The Function's gradient w.r.t. parameters is written by the kernels directly into the
flat gradient buffer whose views are the parameters' `.grad`, so nothing is returned to autograd for them.
The gradient w.r.t. the input `x` is returned when `x` requires it; frozen parameters (requires_grad=False)
get no gradient and cost no weight-gradient launch."""
import torch
from torch.autograd.function import once_differentiable


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
