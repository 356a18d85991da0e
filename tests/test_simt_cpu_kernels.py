"""The CUDA SOURCE of SIMT kernels, executed on the CPU (tests/simt_cpu: the .cu file is compiled
by g++ against a shim <cuda_runtime.h>, every CUDA thread is a fiber, barriers and warp shuffles are scheduling points) and
compared with the numpy statement of the same entry point in tests/abi_emulator.py, which in turn is pinned to the reference
goldens by tests/test_model2_host_logic.py.  Catches indexing, reduction and launch-geometry mistakes in the kernels themselves;
says nothing about performance or about wgmma / TMA code (not executable this way)."""
import ctypes as C
import ctypes as ctypes_mod
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))
import abi_emulator as E  # noqa: E402


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


@pytest.fixture(scope='module', params=['ascending', 'descending'])
def m2lib(request):
    """threads of a block resumed in ascending / descending order: a missing barrier shows under at least one of them"""
    import build
    lib = C.CDLL(build.build_all())              # one CPU library for the whole module (a second g++ build costs ~20 s)
    lib.simt_set_reverse_order(int(request.param == 'descending'))
    yield lib
    lib.simt_set_reverse_order(0)


def both(lib, name, args_fn, outs):
    """run `name` from the CPU-compiled CUDA source and from the numpy emulator on identical inputs; `outs` lists the output
    tensors inside the dict args_fn() builds; returns [(cuda_src_result, emulator_result), ...]"""
    res = []
    for impl in (getattr(lib, name), getattr(E, name)):
        d, args = args_fn()
        rc = impl(*args)
        assert rc == 0, (name, rc, ""  if True else '')
        res.append([d[o].clone() for o in outs])
    return list(zip(*res))


def close(a, b, tol):
    return float((a.double() - b.double()).abs().max()) <= tol * max(1.0, float(b.abs().max()))


@pytest.mark.parametrize('B,HW,Cc,groups,swish,with_cond,pad', [(2, 64, 32, 32, 1, True, 0), (3, 16, 64, 32, 0, False, 8),
                                                                 (1, 256, 128, 32, 1, True, 4), (2, 9, 96, 32, 1, False, 0)])
def test_groupnorm_bwd_source(m2lib, B, HW, Cc, groups, swish, with_cond, pad):
    g = torch.Generator().manual_seed(B * 1000 + HW + Cc)
    ld = Cc + pad

    def args():
        d = dict(x=torch.randn(B * HW, ld, generator=g.manual_seed(1)), dy=torch.randn(B * HW, ld, generator=g.manual_seed(2)),
                 cond=torch.randn(B, Cc, generator=g.manual_seed(3)) if with_cond else None,
                 gamma=1 + 0.2 * torch.randn(Cc, generator=g.manual_seed(4)), beta=0.1 * torch.randn(Cc, generator=g.manual_seed(5)),
                 dx=torch.full((B * HW, ld), 7.0), dgamma=torch.full((Cc,), 0.5), dbeta=torch.full((Cc,), -0.25),
                 dcond=torch.full((B, Cc), 3.0) if with_cond else None)
        a = (P(d['x']), ld, B, C.c_int64(HW), Cc, groups, P(d['cond']), Cc, P(d['gamma']), P(d['beta']), C.c_float(1e-6), swish,
             P(d['dy']), ld, P(d['dx']), ld, P(d['dgamma']), P(d['dbeta']), P(d['dcond']), Cc, C.c_void_p(0))
        return d, a
    outs = ['dx', 'dgamma', 'dbeta'] + (['dcond'] if with_cond else [])
    for name, (got, want) in zip(outs, both(m2lib, 'cd_groupnorm_bwd', args, outs)):
        if name == 'dx':
            got, want = got[:, :Cc], want[:, :Cc]
        assert close(got, want, 3e-5), name


def test_groupnorm_bwd_leaves_row_padding_alone(m2lib):
    B, HW, Cc, ld = 2, 16, 32, 40
    x, dy = torch.randn(B * HW, ld), torch.randn(B * HW, ld)
    dx = torch.full((B * HW, ld), 7.0)
    gamma, beta, dg, db = torch.ones(Cc), torch.zeros(Cc), torch.zeros(Cc), torch.zeros(Cc)
    assert m2lib.cd_groupnorm_bwd(P(x), ld, B, C.c_int64(HW), Cc, 32, P(None), 0, P(gamma), P(beta), C.c_float(1e-6), 1, P(dy), ld,
                                  P(dx), ld, P(dg), P(db), P(None), 0, C.c_void_p(0)) == 0
    assert bool((dx[:, Cc:] == 7.0).all()) and bool((dx[:, :Cc] != 7.0).any())


@pytest.mark.parametrize('npix,Cc,pad,p', [(37, 5, 3, 0.1), (1000, 64, 0, 0.5), (3, 1, 0, 0.0)])
def test_dropout_source(m2lib, npix, Cc, pad, p):
    ld = Cc + pad

    def args():
        d = dict(x=torch.randn(npix, ld, generator=torch.Generator().manual_seed(7)), y=torch.full((npix, ld), 9.0))
        return d, (P(d['x']), ld, C.c_int64(npix), Cc, C.c_float(p), C.c_uint64(0x1234567890ABCDEF), P(d['y']), ld, C.c_void_p(0))
    (got, want), = both(m2lib, 'cd_dropout', args, ['y'])
    assert torch.equal(got, want)                                     # same hash, same mask, same scaling: bit-exact
    if p > 0:
        kept = float((got[:, :Cc] != 0).float().mean())
        assert abs(kept - (1 - p)) < 0.08


@pytest.mark.parametrize('rows,n,pad', [(5, 7, 1), (33, 64, 0), (8, 100, 4)])
def test_softmax_bwd_rows_source(m2lib, rows, n, pad):
    ld = n + pad

    def args():
        g = torch.Generator().manual_seed(3)
        s = torch.softmax(torch.randn(rows, n, generator=g), dim=1)
        d = dict(s=torch.nn.functional.pad(s, (0, pad)).contiguous(), ds=torch.nn.functional.pad(torch.randn(rows, n, generator=g), (0, pad), value=5.0).contiguous())
        return d, (P(d['s']), P(d['ds']), ld, C.c_int64(rows), n, C.c_float(0.125), C.c_void_p(0))
    (got, want), = both(m2lib, 'cd_softmax_bwd_rows', args, ['ds'])
    assert close(got[:, :n], want[:, :n], 2e-6) and bool((got[:, n:] == 5.0).all())


@pytest.mark.parametrize('B,H,W,Cc,pad', [(2, 3, 5, 8, 0), (1, 4, 4, 32, 4)])
def test_upsample_bwd_source(m2lib, B, H, W, Cc, pad):
    ld = Cc + pad

    def args():
        d = dict(dy=torch.randn(B * 4 * H * W, ld, generator=torch.Generator().manual_seed(5)), dx=torch.full((B * H * W, ld), 2.0))
        return d, (P(d['dy']), ld, B, H, W, Cc, P(d['dx']), ld, C.c_void_p(0))
    (got, want), = both(m2lib, 'cd_upsample_nearest2x_bwd', args, ['dx'])
    assert close(got[:, :Cc], want[:, :Cc], 1e-6) and bool((got[:, Cc:] == 2.0).all())


def test_swish_embedding_linear_sources(m2lib):
    n = 1000

    def a_swish():
        g = torch.Generator().manual_seed(1)
        d = dict(dy=torch.randn(n, generator=g), pre=3 * torch.randn(n, generator=g), y=torch.zeros(n), act=torch.zeros(n))
        return d, (P(d['dy']), P(d['pre']), C.c_int64(n), P(d['y']), P(d['act']), C.c_void_p(0))
    for got, want in both(m2lib, 'cd_swish', a_swish, ['y', 'act']):
        assert close(got, want, 2e-6)

    def a_swish_fwd_only():
        d = dict(pre=torch.linspace(-6, 6, 50), act=torch.zeros(50))
        return d, (P(None), P(d['pre']), C.c_int64(50), P(None), P(d['act']), C.c_void_p(0))
    (got, want), = both(m2lib, 'cd_swish', a_swish_fwd_only, ['act'])
    assert close(got, want, 2e-6)

    for dim in (128, 32, 7):
        def a_emb():
            d = dict(t=torch.tensor([0, 1, 49, 999], dtype=torch.int64), emb=torch.full((4, dim), 4.0))
            return d, (P(d['t']), 4, dim, P(d['emb']), C.c_void_p(0))
        (got, want), = both(m2lib, 'cd_timestep_embedding', a_emb, ['emb'])
        assert close(got, want, 2e-4), dim                         # sin / cos of arguments up to 999 in fp32

    for M, K, N, bias in ((3, 128, 512, True), (2, 33, 5, False), (1, 512, 128, True)):
        def a_lin():
            g = torch.Generator().manual_seed(9)
            d = dict(x=torch.randn(M, K, generator=g), w=torch.randn(N, K, generator=g) / K ** 0.5, b=torch.randn(N, generator=g) if bias else None,
                     y=torch.zeros(M, N))
            return d, (P(d['x']), K, P(d['w']), P(d['b']), M, N, P(d['y']), C.c_void_p(0))
        (got, want), = both(m2lib, 'cd_linear_fwd', a_lin, ['y'])
        assert close(got, want, 5e-6), (M, K, N)


def test_augment_u8_source(m2lib):
    N, Hs, Ws, B, S = 5, 20, 24, 4, 16

    def args():
        g = torch.Generator().manual_seed(2)
        d = dict(src=torch.randint(0, 256, (N, Hs, Ws, 3), dtype=torch.uint8, generator=g), index=torch.tensor([4, 0, 2, 2], dtype=torch.int64),
                 oy=torch.tensor([0, 4, 2, 1], dtype=torch.int32), ox=torch.tensor([8, 0, 3, 5], dtype=torch.int32),
                 flip=torch.tensor([0, 1, 1, 0], dtype=torch.int32), out=torch.zeros(B, 3, S, S))
        return d, (P(d['src']), N, Hs, Ws, P(d['index']), P(d['oy']), P(d['ox']), P(d['flip']), B, S, P(d['out']), C.c_void_p(0))
    (got, want), = both(m2lib, 'cd_augment_u8', args, ['out'])
    assert torch.equal(got, want)
    d, a = args()
    a = list(a); a[9] = 32                                            # crop larger than the source: refused, with a message
    assert m2lib.cd_augment_u8(*a) == -1
    buf = C.create_string_buffer(256)
    m2lib.cd_last_error(buf, 256)
    assert b'does not fit' in buf.value


@pytest.fixture(scope='module')
def cpulib():
    import build
    return C.CDLL(build.build_all())


@pytest.mark.parametrize('with_temb', [True, False])
@pytest.mark.parametrize('B,dim,hid,tdim,act,sumC', [(3, 128, 512, 512, 1, 700), (2, 32, 128, 128, 1, 65), (2, 64, 256, 64, 0, 130), (1, 33, 40, 24, 1, 5)])
def test_time_mlp2_source_both_paths(cpulib, with_temb, B, dim, hid, tdim, act, sumC):
    """generalised time MLP (DDPM `Model`): the two-launch path taken when a temb buffer is given (dense layers warp-per-output,
    conditioning rows over the grid) and the one-block-per-sample path without it, against the numpy statement"""
    def args():
        g = torch.Generator().manual_seed(dim + sumC)
        r = lambda *s: torch.randn(*s, generator=g)
        d = dict(t=torch.tensor([0, 17, 999][:B], dtype=torch.int64), w1=r(hid, dim) / dim ** 0.5, b1=0.1 * r(hid), w2=r(tdim, hid) / hid ** 0.5,
                 b2=0.1 * r(tdim), wc=r(sumC, tdim) / tdim ** 0.5, bc=0.1 * r(sumC), temb=torch.full((B, tdim), 9.0) if with_temb else None,
                 cond=torch.full((B, sumC), 9.0))
        return d, (P(d['t']), B, dim, hid, tdim, act, P(d['w1']), P(d['b1']), P(d['w2']), P(d['b2']), P(d['wc']), P(d['bc']), sumC, P(d['temb']),
                   P(d['cond']), C.c_void_p(0))
    outs = ['cond'] + (['temb'] if with_temb else [])
    for got, want in both(cpulib, 'cd_time_mlp2_fwd', args, outs):
        assert close(got, want, 2e-4)            # sin / cos of arguments up to 999 in fp32, then three dense layers


def unaligned(t):
    """a copy of `t` whose data starts 4 bytes past a 16-byte boundary (selects the kernels that take any alignment)"""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype)
    u = buf[1:].view(t.shape)
    u.copy_(t)
    assert u.data_ptr() % 16 != 0
    return u


@pytest.mark.parametrize('B,dim', [(2, 64), (3, 512), (1, 40), (2, 100)])
def test_linattn_staged_kernels_equal_the_unaligned_fallback(cpulib, B, dim):
    """csrc/linattn_small.cu: the shared-memory-staged cd_linattn_weff / cd_linattn_bwd_small keep the arithmetic order of
    weff_kernel / attn_bwd_small_kernel, which serve a w_out / dweff that is not 16-byte aligned -> bit-identical results (the CPU
    execution runs the blocks, hence the float atomics into dW_out, in the same order for both); every output also agrees with
    the float64 numpy statement"""
    g = torch.Generator().manual_seed(B * 7 + dim)
    r = lambda *s: torch.randn(*s, generator=g)
    ctx, ksum, w_out, dweff = r(B, 4, 32, 32), 1.0 + torch.rand(B, 128, generator=g) * 30, r(dim, 128) / 11, r(B, dim, 128)
    res = {}
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        for aligned in (1, 0):
            wo, dwe = (w_out, dweff) if aligned else (unaligned(w_out), unaligned(dweff))
            for rnd in (0, 1):
                weff = torch.full((B, dim, 128), 7.0)
                assert cpulib.cd_linattn_weff(P(ctx), P(ksum), P(wo), B, dim, C.c_float(0.17), rnd, P(weff), C.c_void_p(0)) == 0
                res[('weff', rnd, aligned, order)] = weff
            dw_out, dctxn, rowdot = 0.5 * torch.ones(dim, 128), torch.full((B, 4, 32, 32), 7.0), torch.full((B, 128), 7.0)
            assert cpulib.cd_linattn_bwd_small(P(dwe), P(ctx), P(ksum), P(w_out), B, dim, C.c_float(0.17), P(dw_out), P(dctxn), P(rowdot),
                                               C.c_void_p(0)) == 0
            res[('bwd', 0, aligned, order)] = torch.cat([dw_out.reshape(-1), dctxn.reshape(-1), rowdot.reshape(-1)])
    cpulib.simt_set_reverse_order(0)
    for key in [('weff', 0), ('weff', 1), ('bwd', 0)]:
        base = res[key + (0, 0)]
        for aligned in (0, 1):
            for order in (0, 1):
                assert torch.equal(res[key + (aligned, order)], base), (key, aligned, order)
    weff = torch.zeros(B, dim, 128)
    assert E.cd_linattn_weff(P(ctx), P(ksum), P(w_out), B, dim, C.c_float(0.17), 0, P(weff), None) == 0
    assert close(res[('weff', 0, 1, 0)], weff, 1e-5)
    dw_out, dctxn, rowdot = 0.5 * torch.ones(dim, 128), torch.zeros(B, 4, 32, 32), torch.zeros(B, 128)
    assert E.cd_linattn_bwd_small(P(dweff), P(ctx), P(ksum), P(w_out), B, dim, C.c_float(0.17), P(dw_out), P(dctxn), P(rowdot), None) == 0
    got = res[('bwd', 0, 1, 0)]
    assert close(got, torch.cat([dw_out.reshape(-1), dctxn.reshape(-1), rowdot.reshape(-1)]), 1e-4)
    n0, n1 = dim * 128, dim * 128 + B * 4096
    assert close(got[:n0], dw_out.reshape(-1), 1e-4)
    assert close(got[n0:n1], dctxn.reshape(-1), 1e-4)
    assert close(got[n1:], rowdot.reshape(-1), 1e-4)


@pytest.mark.parametrize('B,n,ld,dld,misalign', [(2, 256, 385, 384, False), (1, 1000, 393, 388, False), (3, 40, 387, 384, False),
                                                 (2, 256, 384, 384, True)])
def test_linattn_bwd_kv_cuda_core_kernel(cpulib, B, n, ld, dld, misalign):
    """attn_bwd_kv_kernel (csrc/backward.cu), which serves the qkv the tensor-core kernel refuses (ld % 4 != 0, or qkv not 16-byte
    aligned): a warp owns one head and four pixel quads; identical under both thread orders, also for a ragged last tile, and
    dk / dv at fp32 accuracy against the float64 statement; q columns and row padding untouched"""
    g = torch.Generator().manual_seed(n)
    qkv = torch.randn(B, n, ld, generator=g)
    kmax = qkv[:, :, 128:256].max(dim=1).values.contiguous()
    ksum = torch.exp(qkv[:, :, 128:256] - kmax[:, None, :]).sum(dim=1).contiguous()
    dctxn, rowdot = torch.randn(B, 4, 32, 32, generator=g), torch.randn(B, 128, generator=g)
    q_in = unaligned(qkv) if misalign else qkv
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        dqkv = torch.full((B, n, dld), 7.0)
        assert cpulib.cd_linattn_bwd_kv(P(q_in), ld, B, n, P(kmax), P(ksum), P(dctxn), P(rowdot), P(dqkv), dld, C.c_void_p(0)) == 0
        res.append(dqkv)
    cpulib.simt_set_reverse_order(0)
    assert torch.equal(res[0], res[1])
    want = torch.full((B, n, dld), 7.0)
    assert E.cd_linattn_bwd_kv(P(qkv), ld, B, n, P(kmax), P(ksum), P(dctxn), P(rowdot), P(want), dld, None) == 0
    assert close(res[1][:, :, 128:384], want[:, :, 128:384], 2e-5)
    assert bool((res[1][:, :, :128] == 7.0).all()) and bool((res[1][:, :, 384:] == 7.0).all())


@pytest.mark.parametrize('B,n,ld,dld', [(2, 256, 384, 384), (1, 1000, 392, 388), (3, 40, 384, 384), (1, 16, 384, 384)])
def test_linattn_bwd_kv_tensor_core_kernel(cpulib, B, n, ld, dld):
    """attn_bwd_kv_mma_kernel (csrc/linattn_bwd.cu, what cd_linattn_bwd_kv runs on aligned operands): mma.sync fragments in the 3xTF32 split
    -> dk / dv at fp32 accuracy against the float64 statement; ragged spans; q columns and row padding untouched; identical
    under both thread orders"""
    g = torch.Generator().manual_seed(n + 1)
    qkv = torch.randn(B, n, ld, generator=g)
    kmax = qkv[:, :, 128:256].max(dim=1).values.contiguous()
    ksum = torch.exp(qkv[:, :, 128:256] - kmax[:, None, :]).sum(dim=1).contiguous()
    dctxn, rowdot = torch.randn(B, 4, 32, 32, generator=g), torch.randn(B, 128, generator=g)
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        dqkv = torch.full((B, n, dld), 7.0)
        assert cpulib.cd_linattn_bwd_kv(P(qkv), ld, B, n, P(kmax), P(ksum), P(dctxn), P(rowdot), P(dqkv), dld, C.c_void_p(0)) == 0
        res.append(dqkv)
    cpulib.simt_set_reverse_order(0)
    assert torch.equal(res[0], res[1])
    want = torch.full((B, n, dld), 7.0)
    assert E.cd_linattn_bwd_kv(P(qkv), ld, B, n, P(kmax), P(ksum), P(dctxn), P(rowdot), P(want), dld, None) == 0
    assert close(res[0][:, :, 128:256], want[:, :, 128:256], 2e-5) and close(res[0][:, :, 256:384], want[:, :, 256:384], 2e-5)
    assert bool((res[0][:, :, :128] == 7.0).all()) and bool((res[0][:, :, 384:] == 7.0).all())


@pytest.mark.parametrize('npix,C,pad,stats,rnd', [(4096, 64, 0, True, 1), (5000, 128, 8, False, 0), (4099, 32, 4, True, 0), (70000, 64, 0, True, 0)])
def test_layernorm_multi_pixel_forward_equals_the_fallback_kernel(cpulib, npix, C, pad, stats, rnd):
    """csrc/layernorm_multi.cu: 4 pixels per lane group in flight on 4096 pixels or more, same per-pixel arithmetic ->
    bit-identical to layernorm_kernel<1>, which serves fewer pixels (here the same rows in slices of 4095 pixels); ragged pixel
    counts and padded rows included; identical under both thread orders; output against the float64 statement"""
    g = torch.Generator().manual_seed(npix + C)
    ld = C + pad
    x = torch.randn(npix, ld, generator=g) * 3 + 0.5
    gam, bet = 1 + 0.2 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        for sl in (npix, 4095):
            y, st = torch.full((npix, ld), 7.0), (torch.full((npix, 2), 7.0) if stats else None)
            for p0 in range(0, npix, sl):
                m = min(sl, npix - p0)
                assert cpulib.cd_layernorm_fwd(P(x[p0:]), ld, ctypes_mod.c_int64(m), C, P(gam), P(bet), ctypes_mod.c_float(1e-5),
                                               P(y[p0:]), ld, P(st[p0:] if stats else None), rnd, None) == 0
            res.append((y, st))
    cpulib.simt_set_reverse_order(0)
    for y, st in res[1:]:
        assert torch.equal(y, res[0][0])
        if stats:
            assert torch.equal(st, res[0][1])
    assert bool((res[0][0][:, C:] == 7.0).all())
    xm = x[:, :C].double()
    want = (xm - xm.mean(1, keepdim=True)) / torch.sqrt(xm.var(1, unbiased=False, keepdim=True) + 1e-5) * gam.double() + bet.double()
    assert close(res[0][0][:, :C], want.float(), 2e-3 if rnd else 2e-5)
    if stats:
        assert close(res[0][1][:, 0], xm.mean(1).float(), 2e-5)
        assert close(res[0][1][:, 1], (1 / torch.sqrt(xm.var(1, unbiased=False) + 1e-5)).float(), 2e-5)


@pytest.mark.parametrize('B,n,ld,ppb', [(2, 256, 384, 64), (1, 1000, 392, 96), (3, 40, 384, 64), (1, 16, 384, 64)])
def test_linattn_context_deterministic_one_pass_kernel(cpulib, B, n, ld, ppb):
    """cd_linattn_context_det (csrc/linattn_ctx.cu): running-max recurrence + 3xTF32 mma fragments + ordered merge of the
    per-block partials -> kmax exact, ksum / ctx at fp32 accuracy against the float64 statement, and bit-identical under both
    thread orders of the CPU executor (no atomics anywhere)"""
    g = torch.Generator().manual_seed(n + ld)
    qkv = torch.randn(B, n, ld, generator=g) * 3.0
    nblk = -(-n // ppb)
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        kmax, ksum, ctx = torch.full((B, 128), 7.0), torch.full((B, 128), 7.0), torch.full((B, 4, 32, 32), 7.0)
        ws = torch.full((B, nblk, 4352), float('nan'))
        assert cpulib.cd_linattn_context_det(P(qkv), ld, B, n, nblk, ppb, P(ws), P(kmax), P(ksum), P(ctx), C.c_void_p(0)) == 0
        res.append(torch.cat([kmax.reshape(-1), ksum.reshape(-1), ctx.reshape(-1)]))
    cpulib.simt_set_reverse_order(0)
    assert torch.equal(res[0], res[1])
    kmax, ksum, ctx = torch.zeros(B, 128), torch.zeros(B, 128), torch.zeros(B, 4, 32, 32)
    assert E.cd_linattn_context(P(qkv), ld, B, n, P(kmax), P(ksum), P(ctx), None) == 0
    assert torch.equal(res[0][:B * 128], kmax.reshape(-1))
    assert close(res[0], torch.cat([kmax.reshape(-1), ksum.reshape(-1), ctx.reshape(-1)]), 3e-6)


def conv_taps_f64(x, taps, w):
    """float64 tap-list convolution: out[b, y, x, o] = sum_t sum_c x[b, y + dy_t, x + dx_t, c] w[t, o, c], zero outside the image"""
    B, H, W, _ = x.shape
    pad = 4
    xp = torch.nn.functional.pad(x.double(), (0, 0, pad, pad, pad, pad))
    return sum(torch.einsum('bhwc,oc->bhwo', xp[:, pad + tp[2]:pad + tp[2] + H, pad + tp[3]:pad + tp[3] + W], w[t].double())
               for t, tp in enumerate(taps))


@pytest.mark.parametrize('Cout,k,Cin', [(128, 3, 3), (64, 1, 3), (64, 4, 2)])
def test_image_edge_kernels_against_float64(cpulib, Cout, k, Cin):
    """conv_smallc4_kernel / wgrad_smallc4_kernel (image edge, Cin <= 4): receptive fields staged with all loads of a chunk in
    flight (stage_patches_preload) for up to 12 taps, by the plain loop (stage_patches) for the 16 taps of a 4 x 4 kernel;
    outputs and pre-activations identical under both thread orders; those and the weight / bias gradients (float atomics) at
    fp32 accuracy against float64"""
    from cold_diffusion_models_b200 import ops
    g = torch.Generator().manual_seed(Cout + k)
    B, H = 2, 24                                            # 1152 pixels: 18 chunks of 64
    x = torch.zeros(B, H, H, 4)
    x[..., :Cin] = torch.randn(B, H, H, Cin, generator=g)
    taps = ops.taps_conv(k, (k - 1) // 2)
    wp = torch.randn(len(taps), Cout, Cin, generator=g) / 3
    bias, dy = torch.randn(Cout, generator=g), torch.randn(B, H, H, Cout, generator=g)
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        out, pre_act = torch.full((B, H, H, Cout), 7.0), torch.full((B, H, H, Cout), 7.0)
        d = ops.make_conv_desc([(ops.View(x, 0, Cin), taps, wp, False)], ops.View(out), (B, H, H), Cout=Cout, bias=bias, act=ops.ACT_GELU,
                               out2=ops.View(pre_act))
        assert cpulib.cd_conv_fwd(C.byref(d), 0, None) == 0
        dw, db = torch.zeros(len(taps), Cout, Cin), torch.zeros(Cout)
        dd = ops.make_conv_desc([(ops.View(x, 0, Cin), taps, dw, False)], ops.View(dy), (B, H, H), Cout=Cout)
        assert cpulib.cd_conv_wgrad(C.byref(dd), P(dy), Cout, P(dw), P(db), 0, None) == 0
        res.append((out, pre_act, dw, db))
    cpulib.simt_set_reverse_order(0)
    for a, b in zip(res[0][:2], res[1][:2]):                # forward: the same sums in the same order under both thread orders
        assert torch.equal(a, b)
    want = conv_taps_f64(x[..., :Cin], taps, wp) + bias.double()
    assert close(res[1][1], want.float(), 2e-5)
    assert close(res[1][0], torch.nn.functional.gelu(want).float(), 2e-5)
    xs = x[..., :Cin].double()
    want_dw = torch.stack([torch.einsum('bhwo,bhwc->oc', dy.double(), conv_taps_f64(xs, [tp], torch.eye(Cin)[None])) for tp in taps])
    assert close(res[1][2], want_dw.float(), 2e-5)
    assert close(res[1][3], dy.double().sum(dim=(0, 1, 2)).float(), 2e-5)


@pytest.mark.parametrize('B,H,Cc,pad,Co,resid', [(2, 24, 64, 0, 3, True), (1, 17, 64, 8, 3, False), (3, 8, 32, 0, 1, True), (1, 16, 128, 0, 5, False),
                                                 (2, 12, 48, 0, 3, True)])
def test_final_projection_tiled_and_fallback_against_float64(cpulib, B, H, Cc, pad, Co, resid):
    """csrc/final_proj.cu: the NHWC -> NCHW 1x1 projection through a shared-memory tile (C = 32, 64, 128) and
    conv1x1_to_nchw_kernel for the other C (here 48): identical under both thread orders and against the float64 statement,
    ragged last tile and padded rows included"""
    g = torch.Generator().manual_seed(B * H + Cc)
    ld = Cc + pad
    x = torch.randn(B, H, H, ld, generator=g)
    w, bias = torch.randn(Co, Cc, generator=g) / 8, torch.randn(Co, generator=g)
    r = torch.randn(B, Co, H, H, generator=g) if resid else None
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        out = torch.full((B, Co, H, H), 7.0)
        assert cpulib.cd_conv1x1_to_nchw(P(x), ld, B, H, H, Cc, P(w), P(bias), Co, P(r), P(out), None) == 0
        res.append(out)
    cpulib.simt_set_reverse_order(0)
    for o in res[1:]:
        assert torch.equal(o, res[0])
    want = torch.einsum('bhwc,oc->bohw', x[..., :Cc].double(), w.double()) + bias.double()[None, :, None, None] + (r.double() if resid else 0)
    assert close(res[0], want.float(), 2e-5)


@pytest.mark.parametrize('B,H,Cc,Co', [(2, 24, 64, 3), (1, 17, 64, 3), (3, 40, 32, 1)])
def test_final_projection_backward_four_pixels_per_trip(cpulib, B, H, Cc, Co):
    """conv1x1_to_nchw_bwd_kernel: four pixels per trip with their loads first, then one pixel per trip for the tail; the same
    sums in the same order under both thread orders -> dx, dW, db bit-identical, and at fp32 accuracy against float64"""
    g = torch.Generator().manual_seed(B + H + Cc)
    x, dout = torch.randn(B, H, H, Cc, generator=g), torch.randn(B, Co, H, H, generator=g)
    w = torch.randn(Co, Cc, generator=g) / 8
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        dx, dw, db = torch.full((B, H, H, Cc), 7.0), torch.zeros(Co, Cc), torch.zeros(Co)
        assert cpulib.cd_conv1x1_to_nchw_bwd(P(dout), P(x), Cc, B, H, H, Cc, P(w), Co, P(dx), Cc, P(dw), P(db), None) == 0
        res.append(torch.cat([dx.reshape(-1), dw.reshape(-1), db.reshape(-1)]))
    cpulib.simt_set_reverse_order(0)
    assert torch.equal(res[0], res[1])
    want_dx = torch.einsum('bohw,oc->bhwc', dout.double(), w.double())
    want_dw = torch.einsum('bohw,bhwc->oc', dout.double(), x.double())
    want = torch.cat([want_dx.reshape(-1), want_dw.reshape(-1), dout.double().sum(dim=(0, 2, 3))]).float()
    assert close(res[1], want, 1e-4)


@pytest.mark.parametrize('B,rows,Cc,pad,out_ld', [(2, 1024, 64, 0, 80), (3, 300, 128, 8, 128), (1, 5000, 32, 0, 32), (2, 256, 512, 0, 600),
                                                  (2, 200, 64, 0, 64), (2, 1024, 30, 2, 40), (2, 512, 64, 1, 64), (3, 2048, 128, 4, 136)])
def test_batched_column_sums_float4_variant(cpulib, B, rows, Cc, pad, out_ld):
    """colsum_batched_vec_kernel (float4 loads, four in flight) where C % 4 == 0, ld % 4 == 0 and rows >= 256; the scalar
    colsum_batched_kernel for fewer rows, other C or ld; both accumulate into `out`, to fp32 rounding of the float64 sums"""
    g = torch.Generator().manual_seed(rows + Cc)
    ld = Cc + pad
    x = torch.randn(B, rows, ld, generator=g)
    res = []
    for order in (0, 1):
        cpulib.simt_set_reverse_order(order)
        out = torch.full((B, out_ld), 0.5)
        assert cpulib.cd_colsum_batched(P(x), ld, B, ctypes_mod.c_int64(rows), Cc, P(out), out_ld, None) == 0
        res.append(out)
    cpulib.simt_set_reverse_order(0)
    want = torch.full((B, out_ld), 0.5)
    want[:, :Cc] += x[:, :, :Cc].double().sum(dim=1).float()
    for o in res:
        assert close(o, want, 2e-5)
        assert bool((o[:, Cc:] == 0.5).all())


@pytest.mark.parametrize('h,level,T,single,SB', [(32, 1, 6, False, 1), (32, 2, 5, True, 4), (87, 3, 3, False, 1), (128, 4, 3, True, 2),
                                                 (150, 1, 2, False, 1), (64, 2, 4, True, 3)])
def test_snow_layer_generator_source_against_scipy_and_torch(cpulib, h, level, T, single, SB):
    """cd_snow_layers (csrc/snow_gen.cu) from its CUDA source: the zoomed base field is BIT-IDENTICAL to scipy.ndimage.zoom + centre
    trim (FP:32-42; sizes 87 and 150 include the coordinate that rounds past the last sample, where scipy returns the constant 0),
    the layers equal oracle/snow_oracle.py's restatement of FP:252-355 (threshold, clip, conv2d motion blur) to 1e-6, and the numpy
    emulator agrees with both"""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
    import snow_oracle as SO
    from cold_diffusion_models_b200.snowification import Snow
    np.random.seed(1000 + h); torch.manual_seed(h)
    st_np, st_t = np.random.get_state(), torch.get_rng_state()
    ref, _ = SO.generate_snow_layers((h, h), snow_level=level, num_timesteps=T, random_snow=True, single_snow=single, batch_size=SB)
    c = SO.SNOW_LEVELS[level][0]
    np.random.set_state(st_np)
    ref_base = np.stack([SO.clipped_zoom(np.random.normal(size=(h, h), loc=c[0], scale=c[1])[..., None], c[2])[..., 0]
                         for _ in range(SB if single else 1)]).astype(np.float32)
    np.random.set_state(st_np); torch.set_rng_state(st_t)
    sn = Snow(image_size=(h, h), snow_level=level, num_timesteps=T, random_snow=True, single_snow=single, batch_size=SB)   # same draws
    ch, m, trim, hh = sn._geom
    nsb = sn._vertical.shape[1]
    outs = []
    for impl in (cpulib.cd_snow_layers, E.cd_snow_layers):
        base, out = torch.full((nsb, h, h), 7.0), torch.full((T, nsb, 3, h, h), 7.0)
        rc = impl(P(sn._noise), nsb, ch, m, trim, hh, P(sn._thres), P(sn._taps), int(sn._taps.shape[1]), P(sn._vertical), T, P(base), P(out), None)
        assert rc == 0
        outs.append((base, out))
    for base, out in outs:
        assert np.array_equal(base.numpy(), ref_base), (h, level)
        assert float((out - ref).abs().max()) < 1e-6, (h, level)
    assert float((outs[0][1] - outs[1][1]).abs().max()) < 1e-6
