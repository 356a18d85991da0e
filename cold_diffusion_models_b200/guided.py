"""Guided restoration: `GaussianDiffusion.restore(y, s, weight=..., steps=...)` of the packages whose degradation is linear in
the image (deblurring, resolution, defading, decolorization without Lab).

Algorithm 2 started at an observation y = D_s(x) instead of at a degraded sample, with reconstruction guidance: every step
pulls x0_hat = R(x_hi, hi - 1) towards agreeing with y under the observation operator D_s,

    g    = d/dx_hi  1/2 sum || D_s(x0_hat) - y ||^2  = J_R^T D_s^T (D_s x0_hat - y)
    x_lo = x_hi - D(x0_hat, hi) + D(x0_hat, lo) - weight g      ('x0_step_down')
    x_lo = D(x0_hat, lo) - weight g                             ('default')

over the levels of strided.reverse_levels(s, steps).  The package supplies two callables backed by fused kernels:
`guide_grad(x0_hat)` = D_s^T (D_s x0_hat - y) in image space, and `step(x_hi, x0_hat, g, hi, lo)`, the routine's update with
"- weight g" in its epilogue (g None: the unguided update of `sample`, the same kernel).  J_R^T is the network's input-only
backward.  weight = 0 runs no backward: the network takes its inference path (and its CUDA-graph replay when enabled), and
the result is `sample(img=x, t=s, steps=steps)`'s final image bit for bit when y = D_s(x)."""
import math
import numbers

import torch


def check_arguments(package, y, s, weight, T, shape):
    """ValueError naming the argument: y a (B, C, S, S) fp32 tensor of the package's shape, s an int in 1..T, weight a finite
    float >= 0"""
    if not torch.is_tensor(y) or y.dim() != 4 or tuple(y.shape[1:]) != tuple(shape) or y.dtype != torch.float32:
        raise ValueError("%s: restore needs y of shape (B, %s) and dtype float32, got %s" % (
            package, ', '.join(map(str, shape)), (tuple(y.shape), y.dtype) if torch.is_tensor(y) else type(y).__name__))
    if isinstance(s, bool) or not isinstance(s, numbers.Integral) or not 1 <= int(s) <= T:
        raise ValueError("%s: restore needs an integer level 1 <= s <= T = %d, got %r" % (package, T, s))
    if isinstance(weight, bool) or not isinstance(weight, numbers.Real) or not math.isfinite(float(weight)) or float(weight) < 0:
        raise ValueError("%s: restore needs a finite guidance weight >= 0, got %r" % (package, weight))


def refuse_restore(package, what):
    raise ValueError("%s: restore is not defined for %s" % (package, what))


def restore_loop(net, y, levels, weight, guide_grad, step):
    """x_{tau_0} = y, then one guided step per pair of levels -> x_0.  The network's parameters are frozen for the loop (their
    requires_grad restored afterwards, also when the loop raises), so the input-only backward writes no parameter .grad."""
    B = y.shape[0]
    img = y
    if weight == 0:
        with torch.no_grad():
            for hi, lo in zip(levels, levels[1:]):
                x0 = net(img, torch.full((B,), hi - 1, dtype=torch.long, device=y.device))
                img = step(img, x0, None, hi, lo)
        return img
    params = list(net.parameters())
    saved = [p.requires_grad for p in params]
    try:
        for p in params:
            p.requires_grad_(False)
        for hi, lo in zip(levels, levels[1:]):
            x = img.detach().requires_grad_()
            with torch.enable_grad():
                x0 = net(x, torch.full((B,), hi - 1, dtype=torch.long, device=y.device))
            x0 = x0.contiguous()
            g, = torch.autograd.grad(x0, x, guide_grad(x0.detach()))
            with torch.no_grad():
                img = step(img, x0.detach(), g.contiguous(), hi, lo)
    finally:
        for p, r in zip(params, saved):
            p.requires_grad_(r)
    return img
