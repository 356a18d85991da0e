"""The line-coalesced epilogue of the tensor-core convolution (csrc/conv_epilogue.cuh, cd_conv_tc_set_staged_epilogue; opt-in) executed from SOURCE on the CPU (tests/simt_cpu) inside a test kernel that feeds it like the epilogue warps of
conv_tc_kernel do, against a numpy statement of the row epilogue (acc + bias + resid -> out2 -> activation -> TF32 rounding -> out).
Covers the transposition through the per-warp shared-memory tile, the pixel shuffles, invalid pixels, every optional operand,
padded row strides and both thread orders.  The wgmma / TMA side of the kernel is not executable here: the `-m gpu` test is
tests/test_helpers_and_variants_gpu.py::test_conv_staged_epilogue_matches_the_row_epilogue."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'simt_cpu'))
import abi_emulator as E  # noqa: E402


@pytest.fixture(scope='module', params=[0, 1])
def lib(request):
    import build
    l = C.CDLL(build.build([os.path.join(HERE, 'simt_cpu', 'epilogue_test.cu')], tag='epilogue_test'))
    l.simt_set_reverse_order(request.param)
    yield l
    l.simt_set_reverse_order(0)


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


_erf = np.vectorize(math.erf)


def gelu(x):
    return 0.5 * x * (1.0 + _erf(x * 0.7071067811865476))


def gelu_grad(x):
    return 0.5 * (1.0 + _erf(x * 0.7071067811865476)) + x * 0.3989422804014327 * np.exp(-0.5 * x * x)


@pytest.mark.parametrize('BN,act,bias,resid,out2,rnd,pad', [(128, 0, True, True, True, 1, 8), (64, 1, True, False, False, 0, 0),
                                                            (256, 2, False, False, False, 1, 4), (32, 0, False, True, False, 0, 12),
                                                            (128, 1, False, True, True, 0, 0)])
def test_staged_epilogue_source_against_the_row_epilogue_statement(lib, BN, act, bias, resid, out2, rnd, pad):
    g = torch.Generator().manual_seed(BN + act)
    npix = 300                                             # output rows; the tile's 128 pixels land on a scattered subset
    ld = BN + pad
    acc = torch.randn(128, BN, generator=g)
    perm = torch.randperm(npix, generator=g)[:128].to(torch.int64)
    valid = (torch.rand(128, generator=g) > 0.2).to(torch.int32)
    valid[5] = 0
    pix = perm.clone()
    pix[valid == 0] = 10 ** 9                              # an invalid pixel's index is never dereferenced
    bias_t = torch.randn(BN, generator=g) if bias else None
    resid_t = torch.randn(npix, ld, generator=g) if resid else None
    aux_t = torch.randn(npix, ld, generator=g) if act == 2 else None
    out = torch.full((npix, ld), 7.0)
    out2_t = torch.full((npix, ld), 9.0) if out2 else None
    rc = lib.cd_test_epilogue_staged(P(acc), BN, P(pix), P(valid), P(out), ld, P(bias_t), P(resid_t), ld, act, rnd, P(out2_t), ld,
                                     P(aux_t), ld)
    assert rc == 0
    want, want2 = np.full((npix, ld), 7.0, np.float32), np.full((npix, ld), 9.0, np.float32)
    for m in range(128):
        if not valid[m]:
            continue
        r = int(perm[m])
        v = acc[m].numpy().copy()
        if bias:
            v = v + bias_t.numpy()
        if resid:
            v = v + resid_t[r, :BN].numpy()
        want2[r, :BN] = v
        if act == 1:
            v = gelu(v.astype(np.float64)).astype(np.float32)
        elif act == 2:
            v = (v * gelu_grad(aux_t[r, :BN].numpy().astype(np.float64)).astype(np.float32)).astype(np.float32)
        if rnd:
            v = E._tf32(v)
        want[r, :BN] = v
    got = out.numpy()
    tol = 0 if act == 0 else 2e-6                           # erff / __expf against double precision
    if rnd and act:
        tol = 2e-3                                          # a 1-ulp difference before the TF32 rounding can move the result by one TF32 ulp
    assert np.allclose(got, want, rtol=tol, atol=tol), np.abs(got - want).max()
    assert (got[:, BN:] == 7.0).all()                       # row padding untouched
    untouched = np.ones(npix, bool)
    untouched[perm[valid == 1].numpy()] = False
    assert (got[untouched] == 7.0).all()                    # rows of invalid / foreign pixels untouched
    if out2:
        assert np.array_equal(out2_t.numpy(), want2)
