"""The CUDA source of the GroupNorm and LayerNorm backwards with their parameter gradients switched off (dgamma = dbeta = NULL,
the frozen-parameter backward), and of the NHWC -> NCHW conversion with an addend (the input gradient), executed on the CPU
through tests/simt_cpu: the data gradients must be the same bits as with the parameter gradients on."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))

SPLIT_MIN_HW = 128 * 128
NULL = C.c_void_p(0)


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


@pytest.fixture(scope='module')
def lib():
    import build
    return C.CDLL(build.build_all())


# (B, HW, C, groups, cond, swish, pad): one CTA per image (HW <= 128 * 128) and the split-plane path above it
GN_CASES = [(2, 16 * 16, 64, 32, True, 1, 4), (1, 8 * 8, 96, 32, False, 0, 0),
            (2, SPLIT_MIN_HW + 1, 32, 32, True, 1, 4), (1, 128 * 130, 96, 32, False, 0, 0)]
GN_IDS = ['one-cta-cond', 'one-cta-C96', 'split-cond', 'split-C96']


@pytest.mark.parametrize('B,HW,Cc,groups,with_cond,swish,pad', GN_CASES, ids=GN_IDS)
def test_groupnorm_backward_without_parameter_gradients(lib, B, HW, Cc, groups, with_cond, swish, pad):
    g = torch.Generator().manual_seed(HW + Cc)
    ld = Cc + pad
    x, dy = torch.randn(B * HW, ld, generator=g), torch.randn(B * HW, ld, generator=g)
    cond = 0.5 * torch.randn(B, Cc, generator=g) if with_cond else None
    gamma, beta = 1 + 0.2 * torch.randn(Cc, generator=g), 0.1 * torch.randn(Cc, generator=g)
    runs = []
    for params in (True, False):
        dx = torch.full((B * HW, ld), 7.0)
        dgamma, dbeta = (torch.zeros(Cc), torch.zeros(Cc)) if params else (None, None)
        dcond = torch.full((B, Cc), 3.0) if with_cond else None
        assert lib.cd_groupnorm_bwd(P(x), ld, B, C.c_int64(HW), Cc, groups, P(cond), Cc, P(gamma), P(beta), C.c_float(1e-6), swish,
                                    P(dy), ld, P(dx), ld, P(dgamma), P(dbeta), P(dcond), Cc, NULL) == 0
        runs.append((dx, dcond, dgamma))
    (dx1, dc1, dg1), (dx0, dc0, _) = runs
    assert float(dg1.abs().sum()) > 0                                    # the reference run did form dgamma
    assert torch.equal(dx0, dx1)
    if with_cond:
        assert torch.equal(dc0, dc1)
    # one of the two alone is refused
    dx = torch.empty(B * HW, ld)
    assert lib.cd_groupnorm_bwd(P(x), ld, B, C.c_int64(HW), Cc, groups, P(cond), Cc, P(gamma), P(beta), C.c_float(1e-6), swish,
                                P(dy), ld, P(dx), ld, P(torch.zeros(Cc)), NULL, NULL, Cc, NULL) != 0


@pytest.mark.parametrize('npix,Cc,with_addend', [(300, 64, True), (200, 256, False), (129, 32, False)])
def test_layernorm_backward_without_parameter_gradients(lib, npix, Cc, with_addend):
    g = torch.Generator().manual_seed(npix + Cc)
    h, dy = torch.randn(npix, Cc, generator=g), torch.randn(npix, Cc, generator=g)
    mean = h.mean(1)
    rstd = torch.rsqrt(h.var(1, unbiased=False) + 1e-5)
    stats = torch.stack([mean, rstd], 1).contiguous()
    gam = 1 + 0.2 * torch.randn(Cc, generator=g)
    add = torch.randn(npix, Cc, generator=g) if with_addend else None
    outs = []
    for params in (True, False):
        dh = torch.full((npix, Cc), 7.0)
        dg, db = (torch.zeros(Cc), torch.zeros(Cc)) if params else (None, None)
        assert lib.cd_layernorm_bwd(P(dy), Cc, P(h), Cc, P(stats), P(gam), C.c_int64(npix), Cc, P(add), Cc, P(dh), Cc, P(dg), P(db),
                                    NULL) == 0
        outs.append((dh, dg))
    (dh1, dg1), (dh0, _) = outs
    assert float(dg1.abs().sum()) > 0
    assert torch.equal(dh0, dh1)


def test_nhwc_to_nchw_with_addend(lib):
    B, Cc, H, W, ld = 2, 3, 5, 6, 4
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, H, W, ld, generator=g)
    add = torch.randn(B, Cc, H, W, generator=g)
    out0, out1 = torch.empty(B, Cc, H, W), torch.empty(B, Cc, H, W)
    assert lib.cd_nhwc_to_nchw(P(x), ld, B, H, W, Cc, P(out0), NULL) == 0
    assert lib.cd_nhwc_to_nchw_add(P(x), ld, B, H, W, Cc, P(add), P(out1), NULL) == 0
    want = x[..., :Cc].permute(0, 3, 1, 2)
    assert torch.equal(out0, want)
    assert torch.equal(out1, want + add)
