"""The CUDA source of the split-plane GroupNorm (planes of more than 128 x 128 pixels: a (chunk x image) grid, Chan-merged
statistics, chunk sums added in a fixed order), executed on the CPU through tests/simt_cpu with the threads of a block resumed
in ascending and in descending order, against the float64 numpy statements of cd_groupnorm_fwd / cd_groupnorm_bwd in
tests/abi_emulator.py."""
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
    lib.simt_set_reverse_order(int(request.param == 'descending'))
    yield lib
    lib.simt_set_reverse_order(0)


def rel_max(a, b):
    return float((a.double() - b.double()).abs().max()) / max(1.0, float(b.double().abs().max()))


# (B, HW, C, groups, cond, swish, pad, shift): 16385 = one pixel above the threshold (a one-pixel last chunk); C = 96 has 24
# channel quads (21 pixel lanes, 8 idle threads, quads that straddle groups of 3) and a ragged last chunk; shift adds a
# large mean to the input
CASES = [(2, SPLIT_MIN_HW + 1, 32, 32, True, 1, 4, 0.0),
         (1, 128 * 130, 96, 32, False, 0, 0, 0.0),
         (2, 128 * 129, 64, 32, True, 1, 8, 100.0),
         (1, 128 * 129, 128, 32, False, 1, 0, 100.0)]
IDS = ['just-above-threshold', 'ragged-C96', 'large-mean-cond', 'large-mean-C128']


def _inputs(B, HW, Cc, with_cond, pad, shift, seed):
    g = torch.Generator().manual_seed(seed)
    ld = Cc + pad
    x = torch.randn(B * HW, ld, generator=g) * 1.5 + shift
    return dict(x=x, dy=torch.randn(B * HW, ld, generator=g),
                cond=0.5 * torch.randn(B, Cc, generator=g) if with_cond else None,
                gamma=1 + 0.2 * torch.randn(Cc, generator=g), beta=0.1 * torch.randn(Cc, generator=g)), ld


@pytest.mark.parametrize('B,HW,Cc,groups,with_cond,swish,pad,shift', CASES, ids=IDS)
def test_split_groupnorm_forward_source(lib, B, HW, Cc, groups, with_cond, swish, pad, shift):
    d, ld = _inputs(B, HW, Cc, with_cond, pad, shift, seed=HW + Cc)
    outs = []
    for impl in (lib.cd_groupnorm_fwd, E.cd_groupnorm_fwd):
        y = torch.full((B * HW, ld), 7.0)
        assert impl(P(d['x']), ld, B, C.c_int64(HW), Cc, groups, P(d['cond']), Cc, P(d['gamma']), P(d['beta']), C.c_float(1e-6),
                    swish, P(y), ld, C.c_void_p(0)) == 0
        outs.append(y)
    got, want = outs
    assert bool((got[:, Cc:] == 7.0).all())                             # row padding untouched
    # measured at most 1.7e-7 without the shift and 1.4e-6 with it (x - mean rounds at the ulp of |x| ~ 100, 7.6e-6)
    assert rel_max(got[:, :Cc], want[:, :Cc]) < (5e-6 if shift else 1e-6)


@pytest.mark.parametrize('B,HW,Cc,groups,with_cond,swish,pad,shift', CASES, ids=IDS)
def test_split_groupnorm_backward_source(lib, B, HW, Cc, groups, with_cond, swish, pad, shift):
    d, ld = _inputs(B, HW, Cc, with_cond, pad, shift, seed=2 * HW + Cc)
    res = []
    for impl in (lib.cd_groupnorm_bwd, E.cd_groupnorm_bwd):
        o = dict(dx=torch.full((B * HW, ld), 7.0), dgamma=torch.full((Cc,), 0.5), dbeta=torch.full((Cc,), -0.25),
                 dcond=torch.full((B, Cc), 3.0) if with_cond else None)
        assert impl(P(d['x']), ld, B, C.c_int64(HW), Cc, groups, P(d['cond']), Cc, P(d['gamma']), P(d['beta']), C.c_float(1e-6),
                    swish, P(d['dy']), ld, P(o['dx']), ld, P(o['dgamma']), P(o['dbeta']), P(o['dcond']), Cc, C.c_void_p(0)) == 0
        res.append(o)
    got, want = res
    assert bool((got['dx'][:, Cc:] == 7.0).all())
    tol = 1e-5 if shift else 1e-6                                       # measured at most 3.4e-6 and 3.6e-7
    assert rel_max(got['dx'][:, :Cc], want['dx'][:, :Cc]) < tol
    # dgamma / dbeta accumulate onto what the buffers held; sums over B * HW pixels
    assert rel_max(got['dgamma'], want['dgamma']) < tol
    assert rel_max(got['dbeta'], want['dbeta']) < tol
    if with_cond:
        # dcond = sum over the pixels of dx, exactly zero in real arithmetic (dx sums to zero over a group): the float64
        # statement gives round-off; bound it against the size of the terms
        scale = float(want['dx'][:, :Cc].abs().sum(0).max())
        assert float((got['dcond'] - want['dcond']).abs().max()) < 2e-7 * scale      # measured 4.7e-8


def test_split_groupnorm_does_not_depend_on_thread_order(lib):
    """every sum of the split path is added in a fixed order, so the results are bit-identical whichever order the threads of
    a block run in (shared- or global-memory float atomics would make them differ)"""
    B, HW, Cc, ld = 2, SPLIT_MIN_HW + 300, 64, 64
    d, _ = _inputs(B, HW, Cc, True, 0, 0.0, seed=11)
    runs = []
    try:
        for order in (0, 1):
            lib.simt_set_reverse_order(order)
            y, dx = torch.empty(B * HW, ld), torch.empty(B * HW, ld)
            dg, db, dc = torch.zeros(Cc), torch.zeros(Cc), torch.zeros(B, Cc)
            assert lib.cd_groupnorm_fwd(P(d['x']), ld, B, C.c_int64(HW), Cc, 32, P(d['cond']), Cc, P(d['gamma']), P(d['beta']),
                                        C.c_float(1e-6), 1, P(y), ld, C.c_void_p(0)) == 0
            assert lib.cd_groupnorm_bwd(P(d['x']), ld, B, C.c_int64(HW), Cc, 32, P(d['cond']), Cc, P(d['gamma']), P(d['beta']),
                                        C.c_float(1e-6), 1, P(d['dy']), ld, P(dx), ld, P(dg), P(db), P(dc), Cc, C.c_void_p(0)) == 0
            runs.append((y, dx, dg, db, dc))
    finally:
        lib.simt_set_reverse_order(0)
    assert all(torch.equal(a, b) for a, b in zip(*runs))
