"""GPU parity of the tap-list convolution (wgmma TC path and fp32 SIMT path) through the C ABI,
against torch's fp64 CPU convolution on identical inputs."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def tf32_rn(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def nhwc(x):   # NCHW -> contiguous [B,H,W,C]
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.fixture(scope='module')
def ops():
    from cold_diffusion_models_b200 import ops
    return ops


def run_conv(ops, d, impl):
    """impl: 'simt' | 'tc' (one-CTA wgmma kernel) | 'tc2' (SM-pair two-CTA cluster kernel where eligible, 256-wide tiles) | 'tc2n'
    (the pair kernel also for the 128- and 64-wide N tiles)."""
    from cold_diffusion_models_b200._lib import lib
    lib.cd_conv_tc_set_2cta(2 if impl in ('tc2', 'tc2n') else 0)
    lib.cd_conv_tc_set_2cta_bn(192 if impl == 'tc2n' else 0)
    lib.cd_conv_tc_set_halo(1 if impl in ('tc3', 'tc3x2') else (6 if impl == 'tc4' else 0))   # 'tc3' / 'tc4': halo-tile kernel, 16 x 8 / 16 x 16 tiles, where eligible
    lib.cd_conv_tc_set_two_ctas(192 if impl in ('tcx2', 'tc3x2') else 0)  # '..x2': two CTAs per SM for the N <= 128 tiles
    try:
        ops.conv_fwd(d, ops.CONV_SIMT if impl == 'simt' else ops.CONV_TC)
        torch.cuda.synchronize()
    finally:
        lib.cd_conv_tc_set_2cta(_DEFAULT_2CTA)
        lib.cd_conv_tc_set_2cta_bn(_DEFAULT_2CTA_BN)
        lib.cd_conv_tc_set_halo(_DEFAULT_HALO)
        lib.cd_conv_tc_set_two_ctas(_DEFAULT_TWO_CTAS)


_DEFAULT_TWO_CTAS = 192         # library default of cd_conv_tc_set_two_ctas
_DEFAULT_HALO = 0               # library default of cd_conv_tc_set_halo
_DEFAULT_2CTA = 0               # library default of cd_conv_tc_set_2cta
_DEFAULT_2CTA_BN = 0            # library default of cd_conv_tc_set_2cta_bn

CASES = [
    # (B, Cin, Cout, H, W, k, pad)
    (2, 64, 128, 32, 32, 3, 1),
    (1, 64, 64, 128, 128, 3, 1),
    (3, 256, 512, 16, 16, 3, 1),
    (4, 64, 64, 8, 8, 3, 1),
    (2, 128, 96, 16, 16, 1, 0),
    (2, 32, 384, 32, 32, 1, 0),
    (5, 64, 64, 4, 4, 3, 1),
    (2, 64, 256, 32, 32, 3, 1),
    (9, 64, 256, 8, 8, 3, 1),          # odd number of 128-pixel tiles: the pair's second CTA runs past the end
    (1, 32, 512, 128, 128, 1, 0),
]


@pytest.mark.parametrize('impl', ['simt', 'tc', 'tc2', 'tc2n', 'tc3', 'tc4', 'tcx2', 'tc3x2'])
@pytest.mark.parametrize('case', CASES)
def test_conv_stride1(ops, case, impl):
    B, Ci, Co, H, W, k, pad = case
    g = torch.Generator().manual_seed(hash(case) % 1000)
    x = tf32_rn(torch.randn(B, Ci, H, W, generator=g))
    w = tf32_rn(torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5)
    b = torch.randn(Co, generator=g)
    r = torch.randn(B, Co, H, W, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=pad) + r.double()
    ref_act = F.gelu(ref)
    xd, wd, bd, rd = nhwc(x).cuda(), w.cuda(), b.cuda(), nhwc(r).cuda()
    taps = ops.taps_conv(k, pad)
    pw = ops.pack_weight(wd, taps, round_tf32=False)
    out = torch.empty(B, H, W, Co, device='cuda')
    pre = torch.empty(B, H, W, Co, device='cuda')
    d = ops.make_conv_desc([(ops.View(xd), taps, pw, False)], ops.View(out), (B, H, W), Cout=Co, bias=bd,
                           resid=ops.View(rd), act=ops.ACT_GELU, out2=ops.View(pre))
    run_conv(ops, d, impl)
    assert rel(nchw(pre.cpu()), ref) < 1e-5
    assert rel(nchw(out.cpu()), ref_act) < 1e-5


@pytest.mark.parametrize('impl', ['simt', 'tc', 'tc2', 'tc3', 'tc4'])
def test_conv_two_sources_channel_slices(ops, impl):
    """3x3 over h plus the 1x1 res_conv over x accumulated in one GEMM (ConvNextBlock tail, DB:151-154,164);
    sources/outputs are channel slices of wider NHWC buffers."""
    g = torch.Generator().manual_seed(5)
    B, H, W, C1, C2, Co = 2, 16, 16, 128, 64, (256 if impl == 'tc2' else 64)
    hbuf = tf32_rn(torch.randn(B, H, W, C1 + 32, generator=g))
    xbuf = tf32_rn(torch.randn(B, H, W, C2 + 64, generator=g))
    w1 = tf32_rn(torch.randn(Co, C1, 3, 3, generator=g) * 0.03)
    w2 = tf32_rn(torch.randn(Co, C2, 1, 1, generator=g) * 0.1)
    bias = torch.randn(Co, generator=g)
    h = hbuf[..., 32:].permute(0, 3, 1, 2).double()
    x = xbuf[..., 64:].permute(0, 3, 1, 2).double()
    ref = F.conv2d(h, w1.double(), bias.double(), padding=1) + F.conv2d(x, w2.double())
    hd, xd = hbuf.cuda(), xbuf.cuda()
    t3, t1 = ops.taps_conv(3, 1), ops.taps_conv(1, 0)
    p1, p2 = ops.pack_weight(w1.cuda(), t3, round_tf32=False), ops.pack_weight(w2.cuda(), t1, round_tf32=False)
    obuf = torch.zeros(B, H, W, 2 * Co, device='cuda')
    d = ops.make_conv_desc([(ops.View(hd, 32, C1), t3, p1, False), (ops.View(xd, 64, C2), t1, p2, False)],
                           ops.View(obuf, Co, Co), (B, H, W), Cout=Co, bias=bias.cuda(), round_tf32=True)
    run_conv(ops, d, impl)
    o = obuf.cpu()
    assert o[..., :Co].abs().max() == 0
    got = o[..., Co:].permute(0, 3, 1, 2)
    assert rel(got, ref) < 4e-4                      # output rounded to TF32
    assert torch.equal(got, tf32_rn(got))


@pytest.mark.parametrize('case', [(2, 64, 64, 16, 8, 3), (1, 128, 128, 32, 24, 3), (3, 96, 320, 16, 16, 3), (2, 64, 64, 64, 64, 3),
                                  (1, 32, 64, 128, 128, 3), (2, 256, 256, 16, 16, 3)])
def test_conv_halo_tile_kernel_forward_and_data_gradient(ops, case):
    """halo-tile kernel, 16 x 8 tiles: one 18 x 10 halo patch per channel chunk read by all nine taps as shifted register
    fragments -- forward taps, flipped (data-gradient) taps with the GELU' epilogue, single patch (16 x 8 image),
    non-square grids, Cout that is not a tile multiple, all three N tiles; against fp64 and against the per-tap kernel"""
    B, Ci, Co, H, W, k = case
    g = torch.Generator().manual_seed(sum(case))
    x = tf32_rn(torch.randn(B, Ci, H, W, generator=g))
    w = tf32_rn(torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5)
    b = torch.randn(Co, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    xd = nhwc(x).cuda()
    outs = []
    pow2 = lambda v: v & (v - 1) == 0
    impls = ('tc', 'tc3') if (pow2(W) and pow2(H)) else ('tc3',)      # the per-tap kernel tiles power-of-two grids only
    for impl in impls:
        out = torch.full((B, H, W, Co), 7.0, device='cuda')
        d = ops.make_conv_desc([(ops.View(xd), ops.taps_conv(3, 1), ops.pack_weight(w.cuda(), ops.taps_conv(3, 1), round_tf32=False), False)],
                               ops.View(out), (B, H, W), Cout=Co, bias=b.cuda())
        run_conv(ops, d, impl)
        assert rel(nchw(out.cpu()), ref) < 1e-5, impl
        outs.append(out)
    assert rel(outs[-1], outs[0]) < 1e-5                    # same products, other summation order
    # data gradient: dX = conv(dY, flipped W^T), multiplied by GELU'(pre) in the epilogue
    dy = tf32_rn(torch.randn(B, Co, H, W, generator=g))
    pre = torch.randn(B, Ci, H, W, generator=g)
    refd = F.conv_transpose2d(dy.double(), w.double(), padding=1)
    cdf = 0.5 * (1 + torch.erf(pre.double() / 2 ** 0.5)); pdf = torch.exp(-0.5 * pre.double() ** 2) / (2 * np.pi) ** 0.5
    refd = refd * (cdf + pre.double() * pdf)
    dyd, pred = nhwc(dy).cuda(), nhwc(pre).cuda()
    pwT = ops.pack_weight(w.cuda(), ops.taps_conv_dgrad(3, 1), mode=1, round_tf32=False)
    for impl in impls:
        dx = torch.full((B, H, W, Ci), 7.0, device='cuda')
        d = ops.make_conv_desc([(ops.View(dyd), ops.taps_conv_dgrad(3, 1), pwT, False)], ops.View(dx), (B, H, W), Cout=Ci,
                               act=ops.ACT_GELU_BWD, aux=ops.View(pred))
        run_conv(ops, d, impl)
        assert rel(nchw(dx.cpu()), refd) < 1e-5, impl


@pytest.mark.parametrize('case', [(2, 64, 64, 16, 16, 3), (1, 128, 128, 32, 48, 3), (3, 96, 100, 16, 32, 3), (2, 128, 64, 64, 64, 3),
                                  (1, 32, 64, 128, 128, 3), (2, 256, 128, 32, 32, 3), (5, 64, 128, 16, 16, 3)])
def test_conv_wide_halo_tile_kernel_forward_and_data_gradient(ops, case):
    """halo-tile kernel, 16 x 16 tiles: one 18 x 18 halo patch per channel chunk, two accumulators per consumer warpgroup that
    share every weight tile -- forward taps and flipped (data-gradient) taps with the GELU' epilogue, single patch,
    non-square grids, Cout that is not a tile multiple, both N tiles, more tiles than SMs; against fp64 and the per-tap kernel"""
    B, Ci, Co, H, W, k = case
    g = torch.Generator().manual_seed(sum(case))
    x = tf32_rn(torch.randn(B, Ci, H, W, generator=g))
    w = tf32_rn(torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5)
    b = torch.randn(Co, generator=g)
    r = torch.randn(B, H, W, Co, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1) + nchw(r).double()
    xd = nhwc(x).cuda()
    outs = []
    pow2 = lambda v: v & (v - 1) == 0
    impls = ('tc', 'tc4') if (pow2(W) and pow2(H)) else ('tc4',)      # the per-tap kernel tiles power-of-two grids only
    for impl in impls:
        out, out2 = torch.full((B, H, W, Co), 7.0, device='cuda'), torch.full((B, H, W, Co), 7.0, device='cuda')
        d = ops.make_conv_desc([(ops.View(xd), ops.taps_conv(3, 1), ops.pack_weight(w.cuda(), ops.taps_conv(3, 1), round_tf32=False), False)],
                               ops.View(out), (B, H, W), Cout=Co, bias=b.cuda(), resid=ops.View(r.cuda()), act=ops.ACT_GELU, out2=ops.View(out2))
        run_conv(ops, d, impl)
        assert rel(nchw(out2.cpu()), ref) < 1e-5, impl
        assert rel(nchw(out.cpu()), F.gelu(ref)) < 1e-5, impl
        outs.append(out2)
    assert rel(outs[-1], outs[0]) < 1e-5                    # same products, other summation order
    dy = tf32_rn(torch.randn(B, Co, H, W, generator=g))
    pre = torch.randn(B, Ci, H, W, generator=g)
    refd = F.conv_transpose2d(dy.double(), w.double(), padding=1)
    cdf = 0.5 * (1 + torch.erf(pre.double() / 2 ** 0.5)); pdf = torch.exp(-0.5 * pre.double() ** 2) / (2 * np.pi) ** 0.5
    refd = refd * (cdf + pre.double() * pdf)
    dyd, pred = nhwc(dy).cuda(), nhwc(pre).cuda()
    pwT = ops.pack_weight(w.cuda(), ops.taps_conv_dgrad(3, 1), mode=1, round_tf32=False)
    if Ci <= 128 and Co % 32 == 0:
        for impl in impls:
            dx = torch.full((B, H, W, Ci), 7.0, device='cuda')
            d = ops.make_conv_desc([(ops.View(dyd), ops.taps_conv_dgrad(3, 1), pwT, False)], ops.View(dx), (B, H, W), Cout=Ci,
                                   act=ops.ACT_GELU_BWD, aux=ops.View(pred))
            run_conv(ops, d, impl)
            assert rel(nchw(dx.cpu()), refd) < 1e-5, impl


@pytest.mark.parametrize('impl', ['simt', 'tc', 'tc2'])
def test_conv_4x4_stride2_and_transpose(ops, impl):
    """Downsample nn.Conv2d(C,C,4,2,1) (DB:108-109) via strided TMA boxes and Upsample
    nn.ConvTranspose2d(C,C,4,2,1) (DB:105-106) as four output-parity tap lists."""
    g = torch.Generator().manual_seed(9)
    B, C, H, W = 2, (256 if impl == 'tc2' else 64), 32, 32
    x = tf32_rn(torch.randn(B, C, H, W, generator=g))
    w = tf32_rn(torch.randn(C, C, 4, 4, generator=g) / (C * 16) ** 0.5)
    b = torch.randn(C, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), stride=2, padding=1)
    xd = nhwc(x).cuda()
    taps = ops.taps_conv(4, 1)
    pw = ops.pack_weight(w.cuda(), taps, round_tf32=False)
    out = torch.empty(B, H // 2, W // 2, C, device='cuda')
    d = ops.make_conv_desc([(ops.View(xd), taps, pw, False)], ops.View(out), (B, H // 2, W // 2), stride=2,
                           Cout=C, bias=b.cuda())
    run_conv(ops, d, impl)
    tol = 3e-6 * max(1.0, C / 64)                    # fp32 accumulation error grows with the contraction length (6.5e-6 at C=256)
    assert rel(nchw(out.cpu()), ref) < tol
    # transpose conv: weight layout (in, out, 4, 4)
    wt = tf32_rn(torch.randn(C, C, 4, 4, generator=g) / (C * 4) ** 0.5)
    reft = F.conv_transpose2d(x.double(), wt.double(), b.double(), stride=2, padding=1)
    outt = torch.empty(B, 2 * H, 2 * W, C, device='cuda')
    for py in (0, 1):
        for px in (0, 1):
            tp = ops.taps_convT4_parity(py, px)
            pwt = ops.pack_weight(wt.cuda(), tp, transposed_conv=True, round_tf32=False)
            d = ops.make_conv_desc([(ops.View(xd), tp, pwt, False)], ops.View(outt), (B, H, W), Cout=C,
                                   bias=b.cuda(), out_map=(2, 2, py, px))
            run_conv(ops, d, impl)
    assert rel(nchw(outt.cpu()), reft) < tol


@pytest.mark.parametrize('impl', ['simt', 'tc'])
def test_conv_per_batch_weights(ops, impl):
    """to_out(einsum(context, q)) folded into a per-batch 1x1 convolution (DB:183-187)."""
    g = torch.Generator().manual_seed(11)
    B, C, Co, H, W = 3, 128, 64, 16, 16
    q = tf32_rn(torch.randn(B, H, W, 384, generator=g))
    weff = tf32_rn(torch.randn(B, Co, C, generator=g) * 0.1)
    res = torch.randn(B, H, W, Co, generator=g)
    bias = torch.randn(Co, generator=g)
    ref = torch.einsum('bhwc,boc->bhwo', q[..., :C].double(), weff.double()) + bias.double() + res.double()
    out = torch.empty(B, H, W, Co, device='cuda')
    tp = ops.taps_conv(1, 0)
    d = ops.make_conv_desc([(ops.View(q.cuda(), 0, C), tp, weff.cuda(), True)], ops.View(out), (B, H, W),
                           Cout=Co, bias=bias.cuda(), resid=ops.View(res.cuda()))
    ops.conv_fwd(d, ops.CONV_TC if impl == 'tc' else ops.CONV_SIMT)
    torch.cuda.synchronize()
    assert rel(out.cpu(), ref) < 3e-6


def test_tf32_operand_rounding_probe(ops):
    """Diagnostic (always passes): how does the TC path treat UNROUNDED fp32 operands under FLOAT32 vs
    TFLOAT32 tensor maps?  The errors are written next to the other test diagnostics."""
    import os
    from cold_diffusion_models_b200._lib import lib
    g = torch.Generator().manual_seed(21)
    B, Ci, Co, H, W = 2, 128, 128, 32, 32
    x = torch.randn(B, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5
    ref = F.conv2d(x.double(), w.double(), padding=1)
    ref_rn = F.conv2d(tf32_rn(x).double(), tf32_rn(w).double(), padding=1)
    ref_tr = F.conv2d((x.view(torch.int32) & ~0x1FFF).view(torch.float32).double(),
                      (w.view(torch.int32) & ~0x1FFF).view(torch.float32).double(), padding=1)
    taps = ops.taps_conv(3, 1)
    lines = []
    for mode in (0, 1):
        lib.cd_conv_tc_set_tf32_maps(mode)
        pw = ops.pack_weight(w.cuda(), taps, round_tf32=False)
        out = torch.empty(B, H, W, Co, device='cuda')
        d = ops.make_conv_desc([(ops.View(nhwc(x).cuda()), taps, pw, False)], ops.View(out), (B, H, W), Cout=Co)
        try:
            ops.conv_fwd(d, ops.CONV_TC)
            torch.cuda.synchronize()
            o = nchw(out.cpu())
            lines.append('map_dtype=%s rel_vs_fp64=%.3e rel_vs_rn=%.3e rel_vs_trunc=%.3e' % (
                'TFLOAT32' if mode else 'FLOAT32', rel(o, ref), rel(o, ref_rn), rel(o, ref_tr)))
        except Exception as e:  # noqa
            lines.append('map_dtype=%d failed: %s' % (mode, e))
    lib.cd_conv_tc_set_tf32_maps(1)
    os.makedirs('gpurun_out', exist_ok=True)
    with open('gpurun_out/tf32_probe.txt', 'w') as f:
        f.write('\n'.join(lines) + '\n')
    print('\n'.join(lines))


WG_CASES = [
    # (B, Cin, Cout, H, W, kind)
    (2, 64, 128, 32, 32, '3x3'),
    (1, 128, 64, 128, 128, '3x3'),
    (3, 256, 512, 16, 16, '3x3'),
    (2, 128, 384, 16, 16, '1x1'),
    (2, 64, 64, 32, 32, '4x4s2'),
    (2, 64, 64, 16, 16, 'convT'),
    (4, 64, 64, 8, 8, '3x3'),
]


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
@pytest.mark.parametrize('case', WG_CASES)
def test_wgrad_tc_matches_fp64(ops, case, mode):
    """tensor-core weight gradient (pixel-axis GEMM, MN-major operands) vs fp64; mode 0 = one X tile per tap,
    otherwise the dx taps share one halo tile addressed by shifted pixel rows."""
    import os
    from cold_diffusion_models_b200._lib import lib
    B, Ci, Co, H, W, kind = case
    g = torch.Generator().manual_seed(17)
    x = tf32_rn(torch.randn(B, Ci, H, W, generator=g))
    lib.cd_wgrad_tc_set_mode(mode)
    try:
        if kind in ('3x3', '1x1'):
            k, pad = (3, 1) if kind == '3x3' else (1, 0)
            w = torch.zeros(Co, Ci, k, k, dtype=torch.double, requires_grad=True)
            y = F.conv2d(x.double(), w, padding=pad)
            dy = tf32_rn(torch.randn(y.shape, generator=g))
            (y * dy.double()).sum().backward()
            taps = ops.taps_conv(k, pad)
            dwp = torch.zeros(len(taps), Co, Ci, device='cuda')
            dyv = ops.View(nhwc(dy).cuda())
            d = ops.make_conv_desc([(ops.View(nhwc(x).cuda()), taps, dwp, False)], dyv, (B, H, W), Cout=Co)
            ops.conv_wgrad(d, dyv, dwp, None, impl=ops.CONV_TC)
            wg = torch.zeros(Co, Ci, k, k, device='cuda')
            ops.unpack_wgrad(dwp, taps, wg, accumulate=False)
            ref = w.grad
        elif kind == '4x4s2':
            w = torch.zeros(Co, Ci, 4, 4, dtype=torch.double, requires_grad=True)
            y = F.conv2d(x.double(), w, stride=2, padding=1)
            dy = tf32_rn(torch.randn(y.shape, generator=g))
            (y * dy.double()).sum().backward()
            taps = ops.taps_conv(4, 1)
            dwp = torch.zeros(16, Co, Ci, device='cuda')
            dyv = ops.View(nhwc(dy).cuda())
            d = ops.make_conv_desc([(ops.View(nhwc(x).cuda()), taps, dwp, False)], dyv, (B, H // 2, W // 2), stride=2, Cout=Co)
            ops.conv_wgrad(d, dyv, dwp, None, impl=ops.CONV_TC)
            wg = torch.zeros(Co, Ci, 4, 4, device='cuda')
            ops.unpack_wgrad(dwp, taps, wg, accumulate=False)
            ref = w.grad
        else:
            w = torch.zeros(Ci, Co, 4, 4, dtype=torch.double, requires_grad=True)
            y = F.conv_transpose2d(x.double(), w, stride=2, padding=1)
            dy = tf32_rn(torch.randn(y.shape, generator=g))
            (y * dy.double()).sum().backward()
            wg = torch.zeros(Ci, Co, 4, 4, device='cuda')
            dyv = ops.View(nhwc(dy).cuda())
            for py in (0, 1):
                for px in (0, 1):
                    tp = ops.taps_convT4_parity(py, px)
                    dwp = torch.zeros(4, Co, Ci, device='cuda')
                    d = ops.make_conv_desc([(ops.View(nhwc(x).cuda()), tp, dwp, False)], dyv, (B, H, W), Cout=Co, out_map=(2, 2, py, px))
                    ops.conv_wgrad(d, dyv, dwp, None, impl=ops.CONV_TC)
                    ops.unpack_wgrad(dwp, tp, wg, transposed_conv=True, accumulate=True)
            ref = w.grad
        torch.cuda.synchronize()
        e = rel(wg.cpu(), ref)
        os.makedirs('gpurun_out', exist_ok=True)
        with open('gpurun_out/wgrad_modes.txt', 'a') as f:
            f.write('mode %d case %s rel %.3e\n' % (mode, case, e))
        assert e < 1e-5, e
    finally:
        lib.cd_wgrad_tc_set_mode(1)


@pytest.mark.parametrize('impl', ['simt', 'tc'])
@pytest.mark.parametrize('hw', [16, 64])
def test_wgrad_per_batch(ops, impl, hw):
    """per-batch weight gradient dweff[b][co][hd] = sum_pix dy[b,pix,co] * q[b,pix,hd] (LinearAttention backward)."""
    g = torch.Generator().manual_seed(23)
    B, dim = 3, 64
    q = tf32_rn(torch.randn(B, hw, hw, 384, generator=g))
    dy = tf32_rn(torch.randn(B, hw, hw, dim, generator=g))
    ref = torch.einsum('bhwo,bhwc->boc', dy.double(), q[..., :128].double())
    dweff = torch.zeros(B, dim, 128, device='cuda')
    dyv = ops.View(dy.cuda())
    d = ops.make_conv_desc([(ops.View(q.cuda(), 0, 128), ops.taps_conv(1, 0), dweff, True)], dyv, (B, hw, hw), Cout=dim)
    ops.conv_wgrad(d, dyv, dweff, None, impl=ops.CONV_TC if impl == 'tc' else ops.CONV_SIMT)
    torch.cuda.synchronize()
    assert rel(dweff.cpu(), ref) < 1e-5


@pytest.mark.parametrize('case', [(2, 64, 128, 32, 32, 3), (3, 128, 256, 16, 16, 3), (2, 64, 192, 32, 32, 1), (4, 256, 64, 16, 16, 3)])
def test_wgrad_tc_fused_bias_gradient(ops, case):
    """bias gradient folded into the tensor-core weight gradient (summed from the dY fragments the MMAs load):
    db and dW against fp64, and against the separate column-sum path"""
    from cold_diffusion_models_b200._lib import lib
    B, Ci, Co, H, W, k = case
    g = torch.Generator().manual_seed(31)
    x = tf32_rn(torch.randn(B, Ci, H, W, generator=g))
    dy = tf32_rn(torch.randn(B, Co, H, W, generator=g))
    w = torch.zeros(Co, Ci, k, k, dtype=torch.double, requires_grad=True)
    bias = torch.zeros(Co, dtype=torch.double, requires_grad=True)
    y = F.conv2d(x.double(), w, bias, padding=k // 2)
    (y * dy.double()).sum().backward()
    taps = ops.taps_conv(k, k // 2)
    dyv = ops.View(nhwc(dy).cuda())
    res = {}
    for fused in (0, 1):
        lib.cd_wgrad_tc_set_bias_fusion(fused)
        try:
            dwp = torch.zeros(len(taps), Co, Ci, device='cuda')
            db = torch.zeros(Co, device='cuda')
            d = ops.make_conv_desc([(ops.View(nhwc(x).cuda()), taps, dwp, False)], dyv, (B, H, W), Cout=Co)
            ops.conv_wgrad(d, dyv, dwp, db, impl=ops.CONV_TC)
            wg = torch.zeros(Co, Ci, k, k, device='cuda')
            ops.unpack_wgrad(dwp, taps, wg, accumulate=False)
            torch.cuda.synchronize()
            res[fused] = (wg.cpu(), db.cpu())
        finally:
            lib.cd_wgrad_tc_set_bias_fusion(0)
    for fused in (0, 1):
        assert rel(res[fused][0], w.grad) < 1e-5, fused
        assert rel(res[fused][1], bias.grad) < 1e-5, fused
