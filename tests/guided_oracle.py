"""TEST INFRASTRUCTURE: the numpy statements of the guided-restoration entry points (include/colddiff.h: cd_*_guide_grad,
cd_*_guided_step / cd_chanmix_guided) that install_emulator() adds to tests/abi_emulator.py's `call`, and the float64
restatement of `GaussianDiffusion.restore` built from a network, the oracles' degradations (tests/strided_oracle.py) and torch
autograd -- never imported by the product.

The restatement: x_{tau_0} = y, then for (hi, lo) over strided levels
    x0 = R(x_hi, hi - 1),  g = d/dx_hi 1/2 ||D_s(x0) - y||^2,  x_lo = update(x_hi, x0, hi, lo) - weight g.
`guide_on='x0'` differentiates with respect to x0 instead of x_hi (J_R left out): the control of the GPU test."""
import numpy as np
import torch

import strided_oracle as SO

F64 = torch.float64


def guided_reverse(net, y, s, K, update, D_obs, weight, batch, guide_on='x_hi'):
    """-> x_0 of the guided loop in the dtype of y (float64 for the restatements); update(img, x0, hi, lo) as in strided_oracle,
    D_obs(x) = D_s(x) of the package"""
    lv = SO.levels(s, K)
    img = y
    for hi, lo in zip(lv, lv[1:]):
        x = img.detach().requires_grad_()
        with torch.enable_grad():
            x0 = net(x, torch.full((batch,), hi - 1, dtype=torch.long, device=y.device))
            loss = 0.5 * ((D_obs(x0) - y) ** 2).sum()
            g, = torch.autograd.grad(loss, x if guide_on == 'x_hi' else x0)
        img = update(img.detach(), x0.detach(), hi, lo) - weight * g
    return img.detach()


# ---- numpy statements of the entry points, fp32 results as the kernels store them ------------------------------------------
def _planes(addr, B, Cc, S):
    from abi_emulator import _arr
    return _arr(addr, (B, Cc, S, S), (Cc * S * S, S * S, S, 1))


def cd_blur_guide_grad(x0, y, out, work, ops_, idx, B, Cc, S, T, stream):
    from abi_emulator import _arr
    assert S <= 128 or _v(work), "cd_blur_guide_grad: S > 128 needs a workspace"
    X, Y = _planes(x0, B, Cc, S).astype(np.float64), _planes(y, B, Cc, S).astype(np.float64)
    if idx < 0:
        r = X - Y
    else:
        A = _arr(ops_, (T, S, S), (S * S, S, 1)).astype(np.float64)[idx]
        r = np.einsum('ji,bcjk,kl->bcil', A, np.einsum('ij,bcjk,lk->bcil', A, X, A) - Y, A)
    _planes(out, B, Cc, S)[:] = r.astype(np.float32)
    return 0


def _axpy(out, g, weight, shape, strides):
    from abi_emulator import _arr
    if _v(g):
        O = _arr(out, shape, strides)
        O[:] = (O.astype(np.float64) - np.float64(_v(weight)) * _arr(g, shape, strides).astype(np.float64)).astype(np.float32)


def cd_blur_guided_step(xt, xhat, g, weight, out, ops_, t_hi, t_lo, B, Cc, S, T, stream):
    import abi_emulator as E
    if _v(xt):
        E.cd_blur_step_down(xt, xhat, out, ops_, t_hi, t_lo, B, Cc, S, T, 0, stream)
    else:
        E.cd_blur_apply(xhat, out, ops_, None, t_lo, B, Cc, S, T, 0, 0, stream)
    _axpy(out, g, weight, (B, Cc, S, S), (Cc * S * S, S * S, S, 1))
    return 0


def cd_mask_guide_grad(x0, y, out, masks, idx, rx, ry, B, Cc, S, MS, stream):
    import abi_emulator as E
    m = E._mask_windows(masks, [idx] * B, rx, ry, B, S, MS, max(idx + 1, 1)).astype(np.float64)
    X, Y = _planes(x0, B, Cc, S).astype(np.float64), _planes(y, B, Cc, S).astype(np.float64)
    _planes(out, B, Cc, S)[:] = (m * (m * X - Y)).astype(np.float32)
    return 0


def cd_mask_guided_step(xt, xhat, g, weight, out, masks, idx_hi, idx_lo, rx, ry, B, Cc, S, MS, stream):
    import abi_emulator as E
    if _v(xt):
        E.cd_mask_step_down(xt, xhat, out, masks, idx_hi, idx_lo, rx, ry, B, Cc, S, MS, stream)
    else:
        E.cd_mask_apply(xhat, out, masks, None, idx_lo, rx, ry, B, Cc, S, MS, 0, stream)
    _axpy(out, g, weight, (B, Cc, S, S), (Cc * S * S, S * S, S, 1))
    return 0


def cd_chanmix_guide_grad(x0, y, out, mats, t, off, B, Cc, HW, stream):
    from abi_emulator import _arr, _i64
    HW = _v(HW)
    idx = _i64(t, B) + off
    M = _arr(mats, (max(int(idx.max()) + 1, 1), Cc, Cc), (Cc * Cc, Cc, 1)).astype(np.float64)
    shp, st = (B, Cc, HW), (Cc * HW, HW, 1)
    X, Y, O = _arr(x0, shp, st).astype(np.float64), _arr(y, shp, st).astype(np.float64), _arr(out, shp, st)
    for b in range(B):
        O[b] = (X[b] - Y[b] if idx[b] < 0 else M[idx[b]].T @ (M[idx[b]] @ X[b] - Y[b])).astype(np.float32)
    return 0


def cd_chanmix_guided(xt, xsrc, g, weight, out, mats, t_hi, t_lo, hi_off, lo_off, B, Cc, HW, mode, stream):
    import abi_emulator as E
    E.cd_chanmix(xt, xsrc, out, mats, t_hi, t_lo, hi_off, lo_off, B, Cc, HW, mode, stream)
    _axpy(out, g, weight, (B, Cc, _v(HW)), (Cc * _v(HW), _v(HW), 1))
    return 0


def _v(a):
    from abi_emulator import _v as v
    return v(a)


ENTRY_POINTS = (cd_blur_guide_grad, cd_blur_guided_step, cd_mask_guide_grad, cd_mask_guided_step, cd_chanmix_guide_grad,
                cd_chanmix_guided)


def install_emulator():
    """route the guided-restoration entry points of tests/abi_emulator.py's `call` to the statements above"""
    import abi_emulator
    for fn in ENTRY_POINTS:
        abi_emulator._TABLE[fn.__name__] = fn
