"""`cd_dropout_seed_dev` (the dropout of a captured training step, its seed read from device memory) from the CUDA source,
executed on the CPU (tests/simt_cpu): for the same seed it gives cd_dropout's output bit for bit, and the numpy statement of
cd_dropout's mask in tests/abi_emulator.py for the seed value it reads."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))
import abi_emulator as E  # noqa: E402


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


@pytest.fixture(scope='module')
def m2lib():
    import build
    return C.CDLL(build.build_all())


@pytest.mark.parametrize('npix,Cc,pad,p,seed', [(37, 5, 3, 0.1, 0x1234567890ABCDEF), (1000, 64, 0, 0.5, 2 ** 62 - 1),
                                                 (256, 32, 4, 0.1, 7)])
def test_seed_from_memory_gives_the_mask_of_the_seed_by_value(m2lib, npix, Cc, pad, p, seed):
    ld = Cc + pad
    x = torch.randn(npix, ld, generator=torch.Generator().manual_seed(3))
    seed_mem = torch.tensor([seed], dtype=torch.int64)
    outs = {}
    for name, impl, s in (('by_value', m2lib.cd_dropout, C.c_uint64(seed)), ('from_memory', m2lib.cd_dropout_seed_dev, P(seed_mem)),
                          ('emulator', E.cd_dropout, C.c_uint64(seed))):
        y = torch.full((npix, ld), 9.0)
        assert impl(P(x), ld, C.c_int64(npix), Cc, C.c_float(p), s, P(y), ld, C.c_void_p(0)) == 0
        outs[name] = y
    assert torch.equal(outs['from_memory'], outs['by_value'])
    assert torch.equal(outs['emulator'], outs['by_value'])
    assert bool((outs['by_value'][:, Cc:] == 9.0).all())


def test_another_seed_gives_another_mask(m2lib):
    x = torch.ones(512, 32)
    ys = []
    for seed in (11, 12):
        y = torch.zeros_like(x)
        s = torch.tensor([seed], dtype=torch.int64)
        assert m2lib.cd_dropout_seed_dev(P(x), 32, C.c_int64(512), 32, C.c_float(0.3), P(s), P(y), 32, C.c_void_p(0)) == 0
        ys.append(y)
    assert not torch.equal(ys[0], ys[1])


def test_null_seed_pointer_is_refused(m2lib):
    x = torch.ones(4, 4)
    assert m2lib.cd_dropout_seed_dev(P(x), 4, C.c_int64(4), 4, C.c_float(0.1), C.c_void_p(0), P(x), 4, C.c_void_p(0)) != 0
