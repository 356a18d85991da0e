"""The CUDA source of the one-CTA GroupNorm (planes of at most 128 x 128 pixels, one 512-thread CTA per image: every GroupNorm of
the `Model` at 32², 64² and 128²), executed on the CPU through tests/simt_cpu with the threads of a block resumed in ascending
and in descending order, against the float64 numpy statements of cd_groupnorm_fwd / cd_groupnorm_bwd in tests/abi_emulator.py.

The inputs carry means of 0, 10 and 100, in x or in the per-(image, channel) `cond` row: statistics formed as E[v²] - mean² in
fp32 lose about 1e-3 at a mean of 100 (E[v²] ~ 1e4 has an ulp of 1e-3; the variance is 2.25), whatever the plane size.  The
bounds are those of the split-plane path (tests/test_groupnorm_split_cpu.py), and the planes on either side of the 128²
threshold meet the same ones."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))
import abi_emulator as E  # noqa: E402

SPLIT_MIN_HW = 128 * 128


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


@pytest.fixture(scope='module', params=['ascending', 'descending'])
def lib(request):
    import build
    lib = C.CDLL(build.build_all())
    lib.order = int(request.param == 'descending')
    lib.simt_set_reverse_order(lib.order)
    yield lib
    lib.simt_set_reverse_order(0)


def rel_max(a, b):
    return float((a.double() - b.double()).abs().max()) / max(1.0, float(b.double().abs().max()))


def _inputs(B, HW, Cc, with_cond, pad, shift, shift_in, seed):
    """x = 1.5 randn (+ shift), cond = 0.5 randn (+ shift): shift_in names which of the two carries the mean"""
    g = torch.Generator().manual_seed(seed)
    ld = Cc + pad
    x = torch.randn(B * HW, ld, generator=g) * 1.5 + (shift if shift_in == 'x' else 0.0)
    cond = 0.5 * torch.randn(B, Cc, generator=g) + (shift if shift_in == 'cond' else 0.0) if with_cond else None
    return dict(x=x, dy=torch.randn(B * HW, ld, generator=g), cond=cond,
                gamma=1 + 0.2 * torch.randn(Cc, generator=g), beta=0.1 * torch.randn(Cc, generator=g)), ld


def _fwd(impl, d, ld, B, HW, Cc, groups, swish):
    y = torch.full((d['x'].shape[0], ld), 7.0)
    assert impl.cd_groupnorm_fwd(P(d['x']), ld, B, C.c_int64(HW), Cc, groups, P(d['cond']), Cc, P(d['gamma']), P(d['beta']),
                                 C.c_float(1e-6), swish, P(y), ld, C.c_void_p(0)) == 0
    return y


def _bwd(impl, d, ld, B, HW, Cc, groups, swish):
    o = dict(dx=torch.full((B * HW, ld), 7.0), dgamma=torch.full((Cc,), 0.5), dbeta=torch.full((Cc,), -0.25),
             dcond=torch.full((B, Cc), 3.0) if d['cond'] is not None else None)
    assert impl.cd_groupnorm_bwd(P(d['x']), ld, B, C.c_int64(HW), Cc, groups, P(d['cond']), Cc, P(d['gamma']), P(d['beta']),
                                 C.c_float(1e-6), swish, P(d['dy']), ld, P(o['dx']), ld, P(o['dgamma']), P(o['dbeta']),
                                 P(o['dcond']), Cc, C.c_void_p(0)) == 0
    return o


# (B, HW, C, groups, cond, swish, pad, shift, shift_in).  C = 128 / 256 at 64² / 32² are planes of the `Model`; C = 96 has 24
# channel quads (21 pixel lanes, 8 idle threads, quads that straddle groups of 3); C = 36 with 4 groups has 9 quads (56 pixel
# lanes, 8 idle threads); C = 2048 has one pixel lane per quad (the C / 4 <= 512 limit), so on a 128² plane each thread sums
# 16384 values; C = groups = 1536 has one channel per group; 9 pixels at C = 128 (16 pixel lanes) and 4² at C = 64 (32 pixel
# lanes) leave pixel lanes without a pixel
CASES = [(2, 64 * 64, 128, 32, True, 1, 0, 0.0, 'x'),
         (2, 64 * 64, 128, 32, True, 1, 4, 10.0, 'cond'),
         (2, 64 * 64, 128, 32, True, 0, 0, 100.0, 'x'),
         (2, 32 * 32, 256, 32, True, 1, 0, 100.0, 'cond'),
         (2, 256, 96, 32, False, 1, 4, 100.0, 'x'),
         (3, 64, 36, 4, True, 0, 8, 10.0, 'x'),
         (1, 64, 2048, 32, True, 1, 0, 100.0, 'cond'),
         (1, 128 * 128, 2048, 32, True, 1, 0, 100.0, 'x'),
         (2, 16, 1536, 1536, True, 1, 0, 10.0, 'cond'),
         (2, 9, 128, 32, True, 1, 0, 100.0, 'x'),
         (2, 16, 64, 32, False, 0, 4, 0.0, 'x')]
IDS = ['64sq-C128', '64sq-C128-mean10-cond-pad', '64sq-C128-mean100-noswish', '32sq-C256-mean100-cond', 'C96-mean100-pad',
       'C36-groups4-mean10', 'C2048-mean100-cond', '128sq-C2048-mean100', 'C1536-groups1536-mean10', '9px-C128-mean100',
       '4sq-C64-nocond']


def _check_forward(lib, B, HW, Cc, groups, with_cond, swish, pad, shift, shift_in):
    d, ld = _inputs(B, HW, Cc, with_cond, pad, shift, shift_in, seed=HW + Cc)
    got, want = (_fwd(impl, d, ld, B, HW, Cc, groups, swish) for impl in (lib, E))
    assert bool((got[:, Cc:] == 7.0).all())                             # row padding untouched
    # the fp32 mean of a group rounds at the ulp of |mean| (7.6e-6 at 100); measured at most 2.5e-7 at mean 0 and 3.1e-6 at
    # mean 100 (the E[v²] - mean² statistics: 1.3e-5 at mean 10, 1.9e-3 at mean 100)
    assert rel_max(got[:, :Cc], want[:, :Cc]) < (5e-6 if shift else 1e-6)


def _check_backward(lib, B, HW, Cc, groups, with_cond, swish, pad, shift, shift_in):
    d, ld = _inputs(B, HW, Cc, with_cond, pad, shift, shift_in, seed=2 * HW + Cc)
    got, want = (_bwd(impl, d, ld, B, HW, Cc, groups, swish) for impl in (lib, E))
    assert bool((got['dx'][:, Cc:] == 7.0).all())
    tol = 1e-5 if shift else 1e-6                                       # measured at most 4.9e-6 and 3.6e-7
    assert rel_max(got['dx'][:, :Cc], want['dx'][:, :Cc]) < tol
    # dgamma / dbeta accumulate onto what the buffers held
    assert rel_max(got['dgamma'], want['dgamma']) < tol
    assert rel_max(got['dbeta'], want['dbeta']) < tol
    if with_cond:
        # dcond = the pixel sum of dx, bounded against the size of the terms: measured at most 1.2e-7 of it on planes of 32² and
        # more.  With a large mean, the rounding of the fp32 group mean offsets xh the same way at every pixel, which planes of
        # few pixels do not average out: 1.4e-6 on 9 and 64 pixels at mean 100
        scale = float(want['dx'][:, :Cc].abs().sum(0).max())
        assert float((got['dcond'] - want['dcond']).abs().max()) < (5e-6 if shift and HW < 1024 else 2e-7) * scale


@pytest.mark.parametrize('B,HW,Cc,groups,with_cond,swish,pad,shift,shift_in', CASES, ids=IDS)
def test_one_cta_groupnorm_forward_source(lib, B, HW, Cc, groups, with_cond, swish, pad, shift, shift_in):
    _check_forward(lib, B, HW, Cc, groups, with_cond, swish, pad, shift, shift_in)


@pytest.mark.parametrize('B,HW,Cc,groups,with_cond,swish,pad,shift,shift_in', CASES, ids=IDS)
def test_one_cta_groupnorm_backward_source(lib, B, HW, Cc, groups, with_cond, swish, pad, shift, shift_in):
    _check_backward(lib, B, HW, Cc, groups, with_cond, swish, pad, shift, shift_in)


@pytest.mark.parametrize('HW', [SPLIT_MIN_HW, SPLIT_MIN_HW + 1], ids=['128sq-one-CTA', '128sq+1-split'])
def test_groupnorm_meets_the_same_bounds_on_both_sides_of_the_split_threshold(lib, HW):
    """128² is the largest plane one CTA normalises, 128² + 1 the smallest the split-plane path takes"""
    _check_forward(lib, 1, HW, 64, 32, True, 1, 0, 100.0, 'x')
    _check_backward(lib, 1, HW, 64, 32, True, 1, 0, 100.0, 'x')


@pytest.mark.parametrize('B,HW,Cc,groups,shift', [(2, 1000, 96, 32, 100.0), (2, 9, 128, 32, 0.0), (1, 64, 36, 4, 10.0)])
def test_one_cta_groupnorm_does_not_depend_on_thread_order(lib, B, HW, Cc, groups, shift):
    """every sum of the one-CTA kernels is added in a fixed order, so y, dx, dgamma, dbeta and dcond are bit-identical whichever
    order the threads of a block run in (shared-memory float atomics would make them differ, and differ run to run on the GPU)"""
    d, ld = _inputs(B, HW, Cc, True, 0, shift, 'x', seed=13)
    runs = []
    try:
        for order in (0, 1):
            lib.simt_set_reverse_order(order)
            o = _bwd(lib, d, ld, B, HW, Cc, groups, 1)
            runs.append([_fwd(lib, d, ld, B, HW, Cc, groups, 1)] + [o[k] for k in ('dx', 'dgamma', 'dbeta', 'dcond')])
    finally:
        lib.simt_set_reverse_order(lib.order)
    differ = [k for k, a, b in zip(('y', 'dx', 'dgamma', 'dbeta', 'dcond'), *runs) if not torch.equal(a, b)]
    assert not differ, differ
