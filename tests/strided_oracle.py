"""TEST INFRASTRUCTURE: float64 restatements of the strided reverse loops of `sample(..., steps=K)`, written from the oracles'
degradations (oracle/*.py), and the numpy statements of the two strided entry points (cd_noise_step_to, cd_fade_step_to)
that install_emulator() adds to tests/abi_emulator.py's `call` -- never imported by the product.

Every loop is the same: x0_hat = R(x, hi - 1), then the routine's update from level hi to level lo over the levels
t = tau_0 > ... > tau_K = 0, tau_i = round(t (K - i) / K).  D(x, n) below is n forward steps of the oracle's degradation.
`lo_of` replaces the lower level the update goes to, and `table_shift` the row the cosine schedule is read at: the controls of
the GPU test use them to state the two mistakes a strided loop can make (stepping to hi - 1 instead of lo; reading sqrt_ac at
s instead of s - 1), which must NOT match the package."""
import numpy as np
import torch

F64 = torch.float64


def levels(t, K):
    return [(2 * t * (K - i) + K) // (2 * K) for i in range(K + 1)]


def reverse(net, img, t, K, update, batch, lo_of=None):
    """-> (direct_recons, img) of the strided loop; update(img, x0_hat, hi, lo)"""
    lv = levels(t, K)
    direct = None
    for hi, lo in zip(lv, lv[1:]):
        x = net(img, torch.full((batch,), hi - 1, dtype=torch.long, device=img.device))
        if direct is None:
            direct = x
        img = update(img, x, hi, lo if lo_of is None else lo_of(hi, lo))
    return direct, img


def cold_update(D, routine):
    """Algorithm 1 ('default': x_s = D(x0_hat, s)) or 2 ('x0_step_down': x_s = x_t - D(x0_hat, t) + D(x0_hat, s))"""
    if routine == 'default':
        return lambda img, x, hi, lo: D(x, lo)
    assert routine == 'x0_step_down'
    return lambda img, x, hi, lo: img - D(x, hi) + D(x, lo)


# ---- the degradations D(x, n) of each package, in float64 ----------------------------------------------------------------
def deblur_D(o):
    """deblur_oracle.DeblurOracle with its taps in float64 (no `discrete`)"""
    o.kernels2d = [k.to(F64) for k in o.kernels2d]
    return lambda x, n: o._cum(x, n)


def resolution_D(o):
    def D(x, n):
        for i in range(n):
            x = o.func(i, x)
        return x
    return D


def defading_D(o, rx=None, ry=None):
    o.fade_kernels = o.fade_kernels.to(F64)

    def D(x, n):
        for i in range(n):
            x = o._kern(i, rx, ry).to(x.device) * x
        return x
    return D


def snow_D(fp):
    """snow_oracle DecolorFP / SnowFP: D(og, n) applies steps 0 .. n-1 with og = the prediction (n <= 0: og itself)"""
    def D(x, n):
        y = x
        for i in range(n):
            y = fp.forward(y, i, og=x)
        return y
    return D


def snow_update(D, routine):
    """the snow package's one-step update indexes D one step lower than Algorithm 1 / 2 (SN:195-245): 'default' x_s =
    D(x0_hat, s - 1), 'x0_step_down' x_s = x_t - D(x0_hat, t - 1) + D(x0_hat, s - 1)"""
    if routine == 'default':
        return lambda img, x, hi, lo: D(x, lo - 1)
    return lambda img, x, hi, lo: img - D(x, hi - 1) + D(x, lo - 1)


def noise_update(sa, sb, fixed_x2=None, table_shift=-1):
    """cosine-schedule step (denoising / demixing 'ddim' when fixed_x2 is None): x2 = (x_t - a_t x0_hat) / b_t,
    x_s = x_t - (a_t x0_hat + b_t x2) + (a_s x0_hat + b_s x2), x_s = x0_hat at s = 0; a_n = sqrt_ac[n - 1]"""
    sa, sb = sa.to(F64), sb.to(F64)

    def update(img, x, hi, lo):
        a1, b1 = sa[hi - 1], sb[hi - 1]
        x2 = (img - a1 * x) / b1 if fixed_x2 is None else fixed_x2
        xs = x if lo == 0 else sa[lo + table_shift] * x + sb[lo + table_shift] * x2
        return img - (a1 * x + b1 * x2) + xs
    return update


def fade_update(alphas, one_minus, x2):
    """per-pixel fade step of defading-generation: x_s = x_t - (al_t x0_hat + om_t x2) + (al_s x0_hat + om_s x2)"""
    al, om = alphas.to(F64), one_minus.to(F64)

    def update(img, x, hi, lo):
        xs = x if lo == 0 else al[lo - 1].to(x.device) * x + om[lo - 1].to(x.device) * x2
        return img - (al[hi - 1].to(x.device) * x + om[hi - 1].to(x.device) * x2) + xs
    return update


# ---- numpy statements of the strided entry points (include/colddiff.h), fp32 as the kernels compute ----------------------
def cd_noise_step_to(img, x1_bar, noise, mode, t, s, sa, sb, n, out, stream):
    from abi_emulator import _arr, _v
    assert 0 <= s < t
    n = _v(n)
    A, Bc = _arr(sa, (t,), (1,)), _arr(sb, (t,), (1,))
    im, xv = _arr(img, (n,), (1,)), _arr(x1_bar, (n,), (1,))
    a1, b1 = A[t - 1], Bc[t - 1]
    x2 = (im - a1 * xv) / b1 if mode == 0 else _arr(noise, (n,), (1,))
    xt_bar = a1 * xv + b1 * x2
    xs = A[s - 1] * xv + Bc[s - 1] * x2 if s != 0 else xv
    _arr(out, (n,), (1,))[:] = (im - xt_bar + xs).astype(np.float32)
    return 0


def cd_fade_step_to(img, x1_bar, x2, t, s, alphas, one_minus, B, Cc, HW, out, stream):
    from abi_emulator import _arr
    assert 0 <= s < t
    al, om = _arr(alphas, (t, HW), (HW, 1)), _arr(one_minus, (t, HW), (HW, 1))
    shp, st = (B, Cc, HW), (Cc * HW, HW, 1)
    im, xv, ev = _arr(img, shp, st), _arr(x1_bar, shp, st), _arr(x2, shp, st)
    xt_bar = al[t - 1] * xv + om[t - 1] * ev
    xs = al[s - 1] * xv + om[s - 1] * ev if s != 0 else xv
    _arr(out, shp, st)[:] = (im - xt_bar + xs).astype(np.float32)
    return 0


def install_emulator():
    """route cd_noise_step_to / cd_fade_step_to of tests/abi_emulator.py's `call` to the statements above"""
    import abi_emulator
    for fn in (cd_noise_step_to, cd_fade_step_to):
        abi_emulator._TABLE[fn.__name__] = fn
