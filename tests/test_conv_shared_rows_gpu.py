"""Shared-row tensor-core convolution (stride 1, taps in [-1, 1]^2: one TMA box per 32-channel chunk and tap column, read by the
three row taps of that column through shifted wgmma descriptors) against the per-tap kernel, which fetches one box per tap and
sums the same products in another order, and against torch's fp64 convolution on the CPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROWS, PER_TAP = 1, 8          # cd_conv_tc_set_halo modes; 0 = library default (shape-based choice)
TWO_CTAS = [0, 192]           # cd_conv_tc_set_two_ctas masks: one CTA per SM; two for the 64- and 128-wide N tiles (default)


def tf32_rn(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def fp64_tol(k):
    """fp32 accumulation error grows with the contraction length k (1e-5 up to the 2304-long sums)"""
    return 1e-5 * max(1.0, (k / 2304) ** 0.5)


@pytest.fixture(scope='module')
def ops():
    from cold_diffusion_models_b200 import ops
    return ops


def run(ops, d, mode, two_ctas=192):
    from cold_diffusion_models_b200._lib import lib
    lib.cd_conv_tc_set_halo(mode)
    lib.cd_conv_tc_set_two_ctas(two_ctas)
    try:
        ops.conv_fwd(d, ops.CONV_TC)
        torch.cuda.synchronize()
    finally:
        lib.cd_conv_tc_set_halo(0)
        lib.cd_conv_tc_set_two_ctas(192)


# every single-source 3x3 forward convolution of Unet(64, (1, 2, 4, 8)) on 128 x 128 images: (H, W, Cin, Cout)
UNET_3X3 = [(128, 128, 32, 128), (128, 128, 64, 128), (128, 128, 128, 64), (64, 64, 64, 256), (64, 64, 128, 256),
            (64, 64, 256, 128), (64, 64, 64, 128), (64, 64, 128, 64), (32, 32, 128, 512), (32, 32, 256, 512), (32, 32, 512, 256),
            (32, 32, 128, 256), (32, 32, 256, 128), (16, 16, 256, 1024), (16, 16, 512, 1024), (16, 16, 1024, 512),
            (16, 16, 256, 512), (16, 16, 512, 256)]


def conv3x3_case(ops, B, H, W, Ci, Co, seed, modes, ctas=192):
    g = torch.Generator().manual_seed(seed)
    x = tf32_rn(torch.randn(B, Ci, H, W, generator=g))
    w = tf32_rn(torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5)
    b = torch.randn(Co, generator=g)
    r = torch.randn(B, H, W, Co, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1) + nchw(r).double()
    taps = ops.taps_conv(3, 1)
    xd, pw = nhwc(x).cuda(), ops.pack_weight(w.cuda(), taps, round_tf32=False)
    outs = {}
    for mode in modes:
        out, pre = torch.full((B, H, W, Co), 7.0, device='cuda'), torch.full((B, H, W, Co), 7.0, device='cuda')
        d = ops.make_conv_desc([(ops.View(xd), taps, pw, False)], ops.View(out), (B, H, W), Cout=Co, bias=b.cuda(),
                               resid=ops.View(r.cuda()), act=ops.ACT_GELU, out2=ops.View(pre))
        run(ops, d, mode, ctas)
        assert rel(nchw(pre.cpu()), ref) < fp64_tol(9 * Ci), mode
        assert rel(nchw(out.cpu()), F.gelu(ref)) < fp64_tol(9 * Ci), mode
        outs[mode] = pre
    if PER_TAP in outs:
        for mode in modes:
            assert rel(outs[mode], outs[PER_TAP]) < 1e-5, mode       # same products, other summation order


@pytest.mark.parametrize('ctas', TWO_CTAS)
@pytest.mark.parametrize('shape', UNET_3X3)
def test_rows_unet_3x3_forward_shapes(ops, shape, ctas):
    H, W, Ci, Co = shape
    conv3x3_case(ops, 2, H, W, Ci, Co, sum(shape), [PER_TAP, ROWS], ctas)


# the fused ConvNextBlock tail [3x3 over h | 1x1 res_conv over x] of the same network: (H, W, C_h, C_x, Cout)
UNET_TWO_SOURCE = [(128, 128, 128, 32, 64), (64, 64, 256, 64, 128), (64, 64, 128, 256, 64), (32, 32, 512, 128, 256),
                   (32, 32, 256, 512, 128), (16, 16, 1024, 256, 512), (16, 16, 512, 1024, 256)]


@pytest.mark.parametrize('ctas', TWO_CTAS)
@pytest.mark.parametrize('shape', UNET_TWO_SOURCE)
def test_rows_two_sources_channel_slices(ops, shape, ctas):
    """3x3 over a channel slice of h plus 1x1 over a channel slice of x in one GEMM, written into a channel slice of a wider
    buffer with TF32 rounding; out2 keeps the unrounded sum"""
    H, W, C1, C2, Co = shape
    B = 2
    g = torch.Generator().manual_seed(sum(shape))
    hbuf = tf32_rn(torch.randn(B, H, W, C1 + 32, generator=g))
    xbuf = tf32_rn(torch.randn(B, H, W, C2 + 64, generator=g))
    w1 = tf32_rn(torch.randn(Co, C1, 3, 3, generator=g) / (C1 * 9) ** 0.5)
    w2 = tf32_rn(torch.randn(Co, C2, 1, 1, generator=g) / C2 ** 0.5)
    bias = torch.randn(Co, generator=g)
    h = hbuf[..., 32:].permute(0, 3, 1, 2).double()
    x = xbuf[..., 64:].permute(0, 3, 1, 2).double()
    ref = F.conv2d(h, w1.double(), bias.double(), padding=1) + F.conv2d(x, w2.double())
    hd, xd = hbuf.cuda(), xbuf.cuda()
    t3, t1 = ops.taps_conv(3, 1), ops.taps_conv(1, 0)
    p1, p2 = ops.pack_weight(w1.cuda(), t3, round_tf32=False), ops.pack_weight(w2.cuda(), t1, round_tf32=False)
    pres = {}
    for m in (PER_TAP, ROWS):
        obuf = torch.zeros(B, H, W, 2 * Co, device='cuda')
        pre = torch.zeros(B, H, W, Co, device='cuda')
        d = ops.make_conv_desc([(ops.View(hd, 32, C1), t3, p1, False), (ops.View(xd, 64, C2), t1, p2, False)],
                               ops.View(obuf, Co, Co), (B, H, W), Cout=Co, bias=bias.cuda(), round_tf32=True, out2=ops.View(pre))
        run(ops, d, m, ctas)
        o = obuf.cpu()
        assert o[..., :Co].abs().max() == 0
        got = o[..., Co:].permute(0, 3, 1, 2)
        assert rel(got, ref) < 4e-4, m                        # output rounded to TF32
        assert torch.equal(got, tf32_rn(got)), m
        assert rel(nchw(pre.cpu()), ref) < fp64_tol(9 * C1 + C2), m
        pres[m] = pre
    assert rel(pres[ROWS], pres[PER_TAP]) < 1e-5


# data gradients of the network's 3x3 convolutions: (H, W, Cin, Cout) of the forward convolution
DGRAD = [(128, 128, 64, 128), (64, 64, 128, 256), (32, 32, 256, 512), (16, 16, 1024, 512), (64, 64, 256, 128)]


@pytest.mark.parametrize('ctas', TWO_CTAS)
@pytest.mark.parametrize('shape', DGRAD)
def test_rows_data_gradient_gelu_bwd(ops, shape, ctas):
    """dX = conv(dY, flipped W^T) on the flipped taps, multiplied by GELU'(pre) in the epilogue"""
    H, W, Ci, Co = shape
    B = 2
    g = torch.Generator().manual_seed(sum(shape) + 1)
    w = tf32_rn(torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5)
    dy = tf32_rn(torch.randn(B, Co, H, W, generator=g))
    pre = torch.randn(B, Ci, H, W, generator=g)
    refd = F.conv_transpose2d(dy.double(), w.double(), padding=1)
    cdf = 0.5 * (1 + torch.erf(pre.double() / 2 ** 0.5)); pdf = torch.exp(-0.5 * pre.double() ** 2) / (2 * np.pi) ** 0.5
    refd = refd * (cdf + pre.double() * pdf)
    dyd, pred = nhwc(dy).cuda(), nhwc(pre).cuda()
    tT = ops.taps_conv_dgrad(3, 1)
    pwT = ops.pack_weight(w.cuda(), tT, mode=1, round_tf32=False)
    outs = {}
    for m in (PER_TAP, ROWS):
        dx = torch.full((B, H, W, Ci), 7.0, device='cuda')
        d = ops.make_conv_desc([(ops.View(dyd), tT, pwT, False)], ops.View(dx), (B, H, W), Cout=Ci, act=ops.ACT_GELU_BWD,
                               aux=ops.View(pred))
        run(ops, d, m, ctas)
        assert rel(nchw(dx.cpu()), refd) < fp64_tol(9 * Co), m
        outs[m] = dx
    assert rel(outs[ROWS], outs[PER_TAP]) < 1e-5


@pytest.mark.parametrize('ctas', TWO_CTAS)
@pytest.mark.parametrize('case', [(2, 32, 32, 64, 96), (2, 16, 16, 128, 320), (2, 32, 32, 64, 36), (3, 16, 16, 256, 200)])
def test_rows_cout_not_tile_multiple(ops, case, ctas):
    """Cout that is not a multiple of the N tile (64 / 128): the weight box reads past Cout as zeros, the epilogue masks
    the columns (36: the last column pair is a single column)"""
    B, H, W, Ci, Co = case
    conv3x3_case(ops, B, H, W, Ci, Co, sum(case), [PER_TAP, ROWS], ctas)


@pytest.mark.parametrize('ctas', TWO_CTAS)
@pytest.mark.parametrize('case', [(2, 24, 40, 64, 128), (1, 10, 20, 32, 64), (3, 40, 24, 128, 256), (1, 7, 130, 64, 64)])
def test_rows_grid_not_tile_multiple(ops, case, ctas):
    """grids that are not multiples of the pixel tile (the per-tap kernel cannot tile them): zero-filled loads, masked stores"""
    B, H, W, Ci, Co = case
    conv3x3_case(ops, B, H, W, Ci, Co, sum(case), [ROWS], ctas)


@pytest.mark.parametrize('ctas', TWO_CTAS)
def test_rows_more_tiles_than_sms(ops, ctas):
    """persistent CTAs walk several tiles each: 8 images x 64 pixel tiles = 512 tiles of 128 pixels and 128 channels, several per CTA"""
    conv3x3_case(ops, 8, 64, 128, 64, 128, 3, [PER_TAP, ROWS], ctas)


def test_rows_default_selection_matches_per_tap(ops):
    """the library default (shape-based choice between the two kernels) against the forced per-tap kernel"""
    conv3x3_case(ops, 2, 64, 64, 128, 128, 4, [PER_TAP, 0])
    conv3x3_case(ops, 2, 16, 16, 512, 512, 5, [PER_TAP, 0])
