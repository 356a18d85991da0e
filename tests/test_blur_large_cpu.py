"""cd_blur_apply / cd_blur_step_down above 128² (the row-strip kernels of csrc/degrade.cu), executed from their CUDA source
on the CPU (tests/simt_cpu: every CUDA thread a fiber, cp.async copies completing at once) and compared with float64
A X A^T in numpy; and the column-batched probe of the resolution package's step operators.

The operators include dense random matrices besides the (symmetric, for circular padding) blur operators, so that a
transposed A or a swapped index shows.  S = 132 leaves a partial strip, a partial ring chunk and a partial 128-column
slice; S = 256 is the first size users run.  The emulator takes about a second per strip product at S = 256, so the S = 256
cases run one plane of products each (about two minutes and a half for the file)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))

from cold_diffusion_models_b200 import resolution as R  # noqa: E402
from cold_diffusion_models_b200.degradation import build_blur_operators  # noqa: E402


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


@pytest.fixture(scope='module', params=['ascending', 'descending'])
def lib(request):
    """threads of a block resumed in ascending / descending order: a missing barrier shows under at least one of them"""
    import build
    lib = C.CDLL(build.build_all())
    lib.simt_set_reverse_order(int(request.param == 'descending'))
    yield lib
    lib.simt_set_reverse_order(0)


def operators(S, T, kind, seed=0):
    """[T][S][S] fp32: the cumulative Exponential_reflect blur operators, or dense random ones"""
    if kind == 'blur':
        return build_blur_operators('Exponential_reflect', T, 15, 0.3, S)[0].contiguous()
    g = torch.Generator().manual_seed(seed + S)
    return (torch.randn(T, S, S, generator=g) / np.sqrt(S)).contiguous()


def images(B, Cc, S, seed=1):
    return (torch.rand(B, Cc, S, S, generator=torch.Generator().manual_seed(seed)) * 2 - 1).contiguous()


def ref_apply(x, ops, idx):
    """float64 A_idx X A_idx^T per plane (idx < 0: X)"""
    X = x.double().numpy()
    if idx < 0:
        return X
    A = ops[idx].double().numpy()
    return np.einsum('ij,...jk,lk->...il', A, X, A)


def apply(lib, x, ops, t=None, t_scalar=0, collapse=0, quantize=0):
    B, Cc, S, _ = x.shape
    out = torch.full_like(x, float('nan'))
    rc = lib.cd_blur_apply(P(x), P(out), P(ops), P(t), t_scalar, B, Cc, S, ops.shape[0], collapse, quantize, C.c_void_p(0))
    assert rc == 0
    return out


def step_down(lib, xt, xhat, ops, t_hi, t_lo, collapse=0):
    B, Cc, S, _ = xt.shape
    out = torch.full_like(xt, float('nan'))
    rc = lib.cd_blur_step_down(P(xt), P(xhat), P(out), P(ops), t_hi, t_lo, B, Cc, S, ops.shape[0], collapse, C.c_void_p(0))
    assert rc == 0
    return out


def rel(got, want):
    want = np.asarray(want, dtype=np.float64)
    return float(np.abs(got.double().numpy() - want).max() / max(1e-30, np.abs(want).max()))


def quantize8(v):
    """DB:954-958 in fp32, the op order of the kernels"""
    q = (v.float() + 1.0) * 0.5
    q = q * 255.0
    q = torch.trunc(q) / 255.0
    return q * 2.0 - 1.0


@pytest.mark.parametrize('S,kind', [(132, 'blur'), (132, 'dense'), (256, 'dense')])
def test_apply_per_sample_t(lib, S, kind):
    T = 4
    ops = operators(S, T, kind)
    t = torch.tensor([2, -1, 0] if S < 256 else [-1, 2], dtype=torch.int64)
    x = images(len(t), 2 if S < 256 else 1, S)
    out = apply(lib, x, ops, t=t)
    for b in range(len(t)):
        assert rel(out[b], ref_apply(x[b], ops, int(t[b]))) < 2e-6, b
    assert torch.equal(out[t == -1], x[t == -1])                      # t = -1 copies the plane


@pytest.mark.parametrize('S', [132, 256])
def test_apply_scalar_index(lib, S):
    ops = operators(S, 3, 'dense')
    x = images(2, 3, S, seed=2) if S < 256 else images(1, 1, S, seed=2)
    assert rel(apply(lib, x, ops, t_scalar=2), ref_apply(x, ops, 2)) < 2e-6
    assert torch.equal(apply(lib, x, ops, t_scalar=-1), x)


@pytest.mark.parametrize('S', [132])
def test_apply_collapse_and_quantize(lib, S):
    """`discrete`: planes at t = T-1 become their mean (closed form w^T X w / S^2), the others are untouched by the option;
    the 8-bit truncation equals quantize8 of the unquantized result bit for bit"""
    T = 3
    ops = operators(S, T, 'blur')
    x = images(3, 2, S, seed=3)
    t = torch.tensor([T - 1, 1, -1], dtype=torch.int64)
    plain = apply(lib, x, ops, t=t)
    coll = apply(lib, x, ops, t=t, collapse=1)
    want = ref_apply(x[0], ops, T - 1).mean(axis=(1, 2))
    for c in range(2):
        assert float((coll[0, c] - coll[0, c, 0, 0]).abs().max()) == 0.0
        assert abs(float(coll[0, c, 0, 0]) - want[c]) < 2e-6 * max(1.0, abs(want[c]))
    assert torch.equal(coll[1:], plain[1:])
    assert rel(plain[0], ref_apply(x[0], ops, T - 1)) < 2e-6
    quant = apply(lib, x, ops, t=t, collapse=1, quantize=1)
    assert torch.equal(quant, quantize8(coll))


@pytest.mark.parametrize('S,hi,lo,collapse', [(132, 3, 2, 0), (132, 0, -1, 0), (132, 3, 2, 1), (132, 2, 1, 1), (256, 3, 2, 1),
                                               (256, 0, -1, 0)])
def test_step_down(lib, S, hi, lo, collapse):
    """out = xt - D(xhat, hi) + D(xhat, lo); with `discrete` only the high term collapses, and only at hi = T-1"""
    T = 4
    ops = operators(S, T, 'dense', seed=5)
    B, Cc = (2, 2) if S < 256 else (1, 1)
    xt, xh = images(B, Cc, S, seed=6), images(B, Cc, S, seed=7)
    out = step_down(lib, xt, xh, ops, hi, lo, collapse)
    Zhi = ref_apply(xh, ops, hi)
    if collapse and hi == T - 1:
        Zhi = np.broadcast_to(Zhi.mean(axis=(2, 3), keepdims=True), Zhi.shape)
    want = xt.double().numpy() - Zhi + ref_apply(xh, ops, lo)
    err = float(np.abs(out.double().numpy() - want).max())
    assert err < 4e-6 * np.abs(want).max(), err


@pytest.mark.parametrize('S', [132, 256])
def test_range_table_of_one_operator(lib, S):
    """T = 1 tables: the range operator of `sample_from_blur` and resolution's `transform_func`"""
    A = torch.from_numpy(R.step_matrix(S, 5, 'bicubic', True).astype(np.float32))[None].contiguous()
    x = images(1, 3 if S < 256 else 1, S, seed=8)
    assert rel(apply(lib, x, A, t_scalar=0), ref_apply(x, A, 0)) < 2e-6


def test_strip_dispatch_refuses_unsupported_sizes(lib):
    x = torch.zeros(1, 1, 516, 516)
    ops = torch.zeros(1, 516, 516)
    for S in (516, 130):
        xs, os_ = x[..., :S, :S].contiguous(), ops[:, :S, :S].contiguous()
        assert lib.cd_blur_apply(P(xs), P(xs.clone()), P(os_), P(None), 0, 1, 1, S, 1, 0, 0, C.c_void_p(0)) != 0
        assert lib.cd_blur_step_down(P(xs), P(xs), P(xs.clone()), P(os_), 0, -1, 1, 1, S, 1, 0, C.c_void_p(0)) != 0
        buf = C.create_string_buffer(512)
        lib.cd_last_error(buf, 512)
        assert b'image size %d unsupported' % S in buf.value


def _step_matrix_one_batch(S, dec_size, mode, do_blur):
    """the single-probe statement of step_matrix: all S columns in one S x S x S interpolate"""
    return R.step_matrix(S, dec_size, mode, do_blur, probe_columns=S)


@pytest.mark.parametrize('S', [32, 100, 128])
@pytest.mark.parametrize('dec,mode,blur', [(1, 'bicubic', False), (7, 'bilinear', True), (None, 'area', False),
                                          (3, 'bicubic', True)])
def test_step_matrix_batching_is_bit_identical_up_to_128(S, dec, mode, blur):
    dec = S // 2 if dec is None else dec
    want = _step_matrix_one_batch(S, dec, mode, blur)
    for cols in (128, 48, 1):
        assert np.array_equal(R.step_matrix(S, dec, mode, blur, probe_columns=cols), want), cols


@pytest.mark.parametrize('dec,mode,blur', [(1, 'bicubic', False), (37, 'bilinear', True), (128, 'area', False)])
def test_step_matrix_batching_at_256(dec, mode, blur):
    got = R.step_matrix(256, dec, mode, blur)
    want = _step_matrix_one_batch(256, dec, mode, blur)
    assert float(np.abs(got - want).max()) <= 1e-12
