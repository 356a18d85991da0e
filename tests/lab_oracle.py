"""TEST INFRASTRUCTURE for the Lab colour path (`to_lab=True`) of the snowification / decolor package; never imported by the product.

* kornia restatement: the four colour stages the reference's rgb2lab / lab2rgb import from kornia (diffusion/utils.py:6-7), which
  is absent here and un-pinned upstream -- parity is unpinned at these constants:
    sRGB -> linear   x > 0.04045 ? ((x + 0.055) / 1.055)^2.4 : x / 12.92
    linear -> sRGB   x > 0.0031308 ? 1.055 max(x, 0.0031308)^(1/2.4) - 0.055 : 12.92 x
    linear RGB <-> XYZ by the sRGB / D65 matrix _M_XYZ and its inverse _M_RGB.
  `install_kornia()` puts them where the reference imports them from, so its own Lab code runs on the CPU
  (tests/golden/gen_golden_lab.py).
* oracle (CPU, dtype-generic so the same code gives an fp64 run): `rgb2lab`, `lab2rgb` (diffusion/utils.py:113-222, "UT") and
  `DecolorLabFP`, the Lab decolorization step rgb2lab(M_i lab2rgb(x)) and total_forward (FP:189-218), usable with
  oracle/snow_oracle.py's SnowOracle.
* numpy statements of cd_lab_convert / cd_chanmix_lab with the C argument lists; `install_emulator()` adds them to
  tests/abi_emulator.py's dispatch table so the package's host logic runs on CPU tensors."""
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

_M_XYZ = ((0.412453, 0.357580, 0.180423), (0.212671, 0.715160, 0.072169), (0.019334, 0.119193, 0.950227))
_M_RGB = ((3.2404813432005266, -1.5371515162713185, -0.4985363261688878), (-0.9692549499965682, 1.8759900014898907, 0.0415559265582928),
          (0.0556466391351772, -0.2040413383665112, 1.0572251624579105))
_WHITE = (0.95047, 1.0, 1.08883)


# ---- kornia's colour stages -----------------------------------------------------------------------------------------------
def _mix3(M, x):
    c = [x[..., i, :, :] for i in range(3)]
    return torch.stack([M[r][0] * c[0] + M[r][1] * c[1] + M[r][2] * c[2] for r in range(3)], dim=-3)


def rgb_to_linear_rgb(image):
    return torch.where(image > 0.04045, torch.pow(((image + 0.055) / 1.055), 2.4), image / 12.92)


def linear_rgb_to_rgb(image):
    threshold = 0.0031308
    return torch.where(image > threshold, 1.055 * torch.pow(image.clamp(min=threshold), 1 / 2.4) - 0.055, 12.92 * image)


def rgb_to_xyz(image):
    return _mix3(_M_XYZ, image)


def xyz_to_rgb(image):
    return _mix3(_M_RGB, image)


def install_kornia():
    """kornia.color.rgb / kornia.color.xyz modules holding the restatement (call before the reference is imported)"""
    for name, fns in (('kornia', ()), ('kornia.color', ()), ('kornia.color.rgb', (linear_rgb_to_rgb, rgb_to_linear_rgb)),
                      ('kornia.color.xyz', (rgb_to_xyz, xyz_to_rgb))):
        m = sys.modules.get(name)
        if m is None:
            m = sys.modules[name] = types.ModuleType(name)
            m.__path__ = []
            if '.' in name:
                setattr(sys.modules[name.rsplit('.', 1)[0]], name.rsplit('.', 1)[1], m)
        for fn in fns:
            setattr(m, fn.__name__, fn)


# ---- oracle -----------------------------------------------------------------------------------------------------------------
def rgb2lab(image):
    """RGB in [-1, 1] -> Lab (UT:113-163)"""
    image = (image + 1) * 0.5
    xyz = rgb_to_xyz(rgb_to_linear_rgb(image))
    xyz = xyz / torch.tensor(_WHITE, dtype=xyz.dtype, device=xyz.device)[..., :, None, None]
    th = 0.008856
    f = torch.where(xyz > th, torch.pow(xyz.clamp(min=th), 1 / 3.0), 7.787 * xyz + 4.0 / 29.0)
    x, y, z = f[..., 0, :, :], f[..., 1, :, :], f[..., 2, :, :]
    return torch.stack([116.0 * y - 16.0, 500.0 * (x - y), 200.0 * (y - z)], dim=-3)


def lab2rgb(image, clip=True):
    """Lab -> 2 rgb - 1 (UT:166-222): fz clamped at 0, rgb clipped to [0, 1] when `clip`"""
    L, a, b = image[..., 0, :, :], image[..., 1, :, :], image[..., 2, :, :]
    fy = (L + 16.0) / 116.0
    fx = a / 500.0 + fy
    fz = (fy - b / 200.0).clamp(min=0.0)
    f = torch.stack([fx, fy, fz], dim=-3)
    xyz = torch.where(f > 0.2068966, torch.pow(f, 3.0), (f - 4.0 / 29.0) / 7.787)
    xyz = xyz * torch.tensor(_WHITE, dtype=xyz.dtype, device=xyz.device)[..., :, None, None]
    rgb = linear_rgb_to_rgb(xyz_to_rgb(xyz))
    if clip:
        rgb = rgb.clamp(0.0, 1.0)
    return 2.0 * rgb - 1


class DecolorLabFP:
    """the Lab decolorization forward process (FP:189-218): step i = rgb2lab(M_i lab2rgb(x)), M_i = f_i I + (1 - f_i)/C 11^T"""

    def __init__(self, factors, channels=3):
        eye, ones = torch.eye(channels), torch.ones((channels, channels)) / float(channels)
        self.w = [(f * eye + (1.0 - f) * ones)[:, :, None, None] for f in factors]

    def forward(self, x, i, og=None):
        return rgb2lab(F.conv2d(lab2rgb(x), self.w[i].to(x)))

    def total_forward(self, x):
        Cn = x.shape[1]
        w = (torch.ones((Cn, Cn), dtype=x.dtype, device=x.device) / float(Cn))[:, :, None, None]
        return rgb2lab(F.conv2d(lab2rgb(x), w))


# ---- numpy statements of the two entry points (fp32) ------------------------------------------------------------------------
_F = np.float32


def _rgb2lab_np(v):
    """[..., 3, P] RGB in [-1, 1] -> Lab"""
    v = (v + _F(1)) * _F(0.5)
    lin = np.where(v > _F(0.04045), np.power((v + _F(0.055)) / _F(1.055), _F(2.4)), v / _F(12.92))
    xyz = np.einsum('rc,...cp->...rp', np.array(_M_XYZ, np.float32), lin) / np.array(_WHITE, np.float32)[:, None]
    f = np.where(xyz > _F(0.008856), np.power(np.maximum(xyz, _F(0.008856)), _F(1 / 3.0)), _F(7.787) * xyz + _F(4.0 / 29.0))
    return np.stack([_F(116) * f[..., 1, :] - _F(16), _F(500) * (f[..., 0, :] - f[..., 1, :]), _F(200) * (f[..., 1, :] - f[..., 2, :])], -2)


def _lab2rgb_np(v, clip=True):
    """[..., 3, P] Lab -> 2 rgb - 1"""
    fy = (v[..., 0, :] + _F(16)) / _F(116)
    fx = v[..., 1, :] / _F(500) + fy
    fz = np.maximum(fy - v[..., 2, :] / _F(200), _F(0))
    f = np.stack([fx, fy, fz], -2)
    xyz = np.where(f > _F(0.2068966), f * f * f, (f - _F(4.0 / 29.0)) / _F(7.787)) * np.array(_WHITE, np.float32)[:, None]
    lin = np.einsum('rc,...cp->...rp', np.array(_M_RGB, np.float32), xyz)
    rgb = np.where(lin > _F(0.0031308), _F(1.055) * np.power(np.maximum(lin, _F(0.0031308)), _F(1 / 2.4)) - _F(0.055), _F(12.92) * lin)
    if clip:
        rgb = np.clip(rgb, _F(0), _F(1))
    return (_F(2) * rgb - _F(1)).astype(np.float32)


def cd_lab_convert(x, out, B, HW, to_lab, clip, stream):
    from abi_emulator import _arr, _v
    HW = _v(HW)
    shp, st = (B, 3, HW), (3 * HW, HW, 1)
    v = np.array(_arr(x, shp, st), dtype=np.float32)           # a copy: out may alias x
    _arr(out, shp, st)[:] = _rgb2lab_np(v) if to_lab else _lab2rgb_np(v, bool(clip))
    return 0


def cd_chanmix_lab(xt, xsrc, out, step_mats, t_hi, t_lo, hi_off, lo_off, B, HW, mode, stream):
    from abi_emulator import _arr, _i64, _v
    HW = _v(HW)
    th = _i64(t_hi, B) + hi_off
    tl = (_i64(t_lo, B) + lo_off) if mode else np.full(B, -1)
    T = int(max(th.max(), tl.max())) + 1
    M = _arr(step_mats, (max(T, 1), 3, 3), (9, 3, 1))
    shp, st = (B, 3, HW), (3 * HW, HW, 1)
    src = np.array(_arr(xsrc, shp, st), dtype=np.float32)
    res = np.empty((B, 3, HW), np.float32)
    for b in range(B):
        v, hi, lo = src[b], src[b], src[b]
        for i in range(max(th[b], tl[b]) + 1):
            v = _rgb2lab_np(np.einsum('rc,cp->rp', M[i], _lab2rgb_np(v)).astype(np.float32))
            hi = v if i == th[b] else hi
            lo = v if i == tl[b] else lo
        res[b] = _arr(xt, shp, st)[b] - hi + lo if mode else hi
    _arr(out, shp, st)[:] = res
    return 0


def install_emulator():
    """route cd_lab_convert / cd_chanmix_lab of tests/abi_emulator.py's `call` to the statements above"""
    import abi_emulator
    for fn in (cd_lab_convert, cd_chanmix_lab):
        abi_emulator._TABLE[fn.__name__] = fn
