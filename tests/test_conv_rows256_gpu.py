"""Shared-row tensor-core convolution with 16 x 16 pixel tiles (two accumulators per consumer warpgroup, one CTA per SM, output
stored by TMA from shared-memory staging slices) against the 16 x 8 shared-row kernel, which runs the same wgmma sequence for
every output element and must agree bit for bit, and against torch's fp64 convolution on the CPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROWS, ROWS256 = 1, 4          # cd_conv_tc_set_halo modes: 16 x 8 tiles, 16 x 16 tiles wherever eligible


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


def run(ops, d, mode):
    from cold_diffusion_models_b200._lib import lib
    lib.cd_conv_tc_set_halo(mode)
    try:
        ops.conv_fwd(d, ops.CONV_TC)
        torch.cuda.synchronize()
    finally:
        lib.cd_conv_tc_set_halo(0)


def gelu_grad(x):
    cdf = 0.5 * (1 + torch.erf(x / 2 ** 0.5))
    return cdf + x * torch.exp(-0.5 * x * x) / (2 * np.pi) ** 0.5


def forward_case(ops, B, H, W, Ci, Co, seed, drop_tap=None):
    """3x3 conv + bias + resid -> out2, GELU -> out; both kernels, bit for bit; the 16 x 16 one against fp64.  drop_tap: the
    16 x 16 kernel runs without that tap (negative control) and its relative error against fp64 is returned."""
    g = torch.Generator().manual_seed(seed)
    x = tf32_rn(torch.randn(B, Ci, H, W, generator=g))
    w = tf32_rn(torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5)
    b = torch.randn(Co, generator=g)
    r = torch.randn(B, H, W, Co, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1) + nchw(r).double()
    taps = ops.taps_conv(3, 1)
    xd, rd, bd = nhwc(x).cuda(), r.cuda(), b.cuda()
    res = {}
    for mode in (ROWS, ROWS256):
        tl = [t for i, t in enumerate(taps) if not (mode == ROWS256 and i == drop_tap)]
        pw = ops.pack_weight(w.cuda(), tl, round_tf32=False)
        out, pre = torch.full((B, H, W, Co), 7.0, device='cuda'), torch.full((B, H, W, Co), 7.0, device='cuda')
        d = ops.make_conv_desc([(ops.View(xd), tl, pw, False)], ops.View(out), (B, H, W), Cout=Co, bias=bd, resid=ops.View(rd),
                               act=ops.ACT_GELU, out2=ops.View(pre))
        run(ops, d, mode)
        res[mode] = (out.cpu(), pre.cpu())
    if drop_tap is not None:
        return rel(nchw(res[ROWS256][1]), ref)
    assert torch.equal(res[ROWS256][0], res[ROWS][0])
    assert torch.equal(res[ROWS256][1], res[ROWS][1])
    assert rel(nchw(res[ROWS256][1]), ref) < fp64_tol(9 * Ci)
    assert rel(nchw(res[ROWS256][0]), F.gelu(ref)) < fp64_tol(9 * Ci)


def dgrad_case(ops, B, H, W, Ci, Co, seed):
    """dX = conv(dY, flipped W^T) on the flipped taps, times GELU'(pre) in the epilogue (aux); dX has Ci channels"""
    g = torch.Generator().manual_seed(seed)
    w = tf32_rn(torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5)
    dy = tf32_rn(torch.randn(B, Co, H, W, generator=g))
    pre = torch.randn(B, Ci, H, W, generator=g)
    refd = F.conv_transpose2d(dy.double(), w.double(), padding=1) * gelu_grad(pre.double())
    dyd, pred = nhwc(dy).cuda(), nhwc(pre).cuda()
    tT = ops.taps_conv_dgrad(3, 1)
    pwT = ops.pack_weight(w.cuda(), tT, mode=1, round_tf32=False)
    outs = {}
    for mode in (ROWS, ROWS256):
        dx = torch.full((B, H, W, Ci), 7.0, device='cuda')
        d = ops.make_conv_desc([(ops.View(dyd), tT, pwT, False)], ops.View(dx), (B, H, W), Cout=Ci, act=ops.ACT_GELU_BWD,
                               aux=ops.View(pred))
        run(ops, d, mode)
        outs[mode] = dx.cpu()
    assert torch.equal(outs[ROWS256], outs[ROWS])
    # GELU' (up to 1.13) scales the accumulation error: 1.25 x the forward bound (K = 9216 reaches 1.02 x of it on both kernels)
    assert rel(nchw(outs[ROWS256]), refd) < 1.25 * fp64_tol(9 * Co)


# every single-source 3x3 convolution of Unet(64, (1, 2, 4, 8)) on 128 x 128 images: (H, W, Cin, Cout)
UNET_3X3 = [(128, 128, 32, 128), (128, 128, 64, 128), (128, 128, 128, 64), (64, 64, 64, 256), (64, 64, 128, 256),
            (64, 64, 256, 128), (64, 64, 64, 128), (64, 64, 128, 64), (32, 32, 128, 512), (32, 32, 256, 512), (32, 32, 512, 256),
            (32, 32, 128, 256), (32, 32, 256, 128), (16, 16, 256, 1024), (16, 16, 512, 1024), (16, 16, 1024, 512),
            (16, 16, 256, 512), (16, 16, 512, 256)]


@pytest.mark.parametrize('shape', UNET_3X3)
def test_rows256_unet_3x3_forward(ops, shape):
    H, W, Ci, Co = shape
    forward_case(ops, 2, H, W, Ci, Co, sum(shape))


@pytest.mark.parametrize('shape', UNET_3X3)
def test_rows256_unet_3x3_data_gradient(ops, shape):
    """the data gradient of each of those convolutions (GELU' epilogue with aux)"""
    H, W, Ci, Co = shape
    dgrad_case(ops, 2, H, W, Ci, Co, sum(shape) + 1)


# the fused ConvNextBlock tail [3x3 over h | 1x1 res_conv over x] of the same network: (H, W, C_h, C_x, Cout)
UNET_TWO_SOURCE = [(128, 128, 128, 32, 64), (64, 64, 256, 64, 128), (64, 64, 128, 256, 64), (32, 32, 512, 128, 256),
                   (32, 32, 256, 512, 128), (16, 16, 1024, 256, 512), (16, 16, 512, 1024, 256)]


@pytest.mark.parametrize('shape', UNET_TWO_SOURCE)
def test_rows256_two_sources_channel_slices(ops, shape):
    """3x3 over a channel slice of h plus 1x1 over a channel slice of x in one GEMM, written into a channel slice of a wider
    buffer with TF32 rounding (the TMA store must leave the neighbouring channels alone); out2 keeps the unrounded sum"""
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
    res = {}
    for m in (ROWS, ROWS256):
        obuf = torch.full((B, H, W, 3 * Co), 5.0, device='cuda')
        pre = torch.zeros(B, H, W, Co, device='cuda')
        d = ops.make_conv_desc([(ops.View(hd, 32, C1), t3, p1, False), (ops.View(xd, 64, C2), t1, p2, False)],
                               ops.View(obuf, Co, Co), (B, H, W), Cout=Co, bias=bias.cuda(), round_tf32=True, out2=ops.View(pre))
        run(ops, d, m)
        res[m] = (obuf.cpu(), pre.cpu())
    o, pre = res[ROWS256]
    assert torch.equal(o, res[ROWS][0]) and torch.equal(pre, res[ROWS][1])
    assert (o[..., :Co] == 5.0).all() and (o[..., 2 * Co:] == 5.0).all()
    got = o[..., Co:2 * Co].permute(0, 3, 1, 2)
    assert rel(got, ref) < 4e-4                                   # output rounded to TF32
    assert torch.equal(got, tf32_rn(got))
    assert rel(nchw(pre), ref) < fp64_tol(9 * C1 + C2)


@pytest.mark.parametrize('case', [(2, 32, 32, 64, 64), (2, 32, 32, 64, 128), (2, 32, 32, 128, 384), (2, 16, 16, 64, 96),
                                  (2, 16, 16, 64, 36)])
def test_rows256_cout(ops, case):
    """N tiles of 64 (Cout = 64) and 128 columns, Cout = 384 (three N tiles), and Cout that is not a multiple of the N tile or of
    the 32-channel store box (36: the last column pair is a single column)"""
    B, H, W, Ci, Co = case
    forward_case(ops, B, H, W, Ci, Co, sum(case))


@pytest.mark.parametrize('case', [(2, 24, 24, 64, 128), (2, 40, 40, 64, 128), (2, 8, 24, 64, 64), (1, 24, 40, 32, 64),
                                  (3, 7, 130, 64, 64)])
def test_rows256_grid_not_tile_multiple(ops, case):
    """grids that are not multiples of the 16 x 16 tile: zero-filled loads, stores clipped by the output map (8 x 24: the second
    warpgroup of every tile lies wholly outside the image and stores nothing)"""
    B, H, W, Ci, Co = case
    forward_case(ops, B, H, W, Ci, Co, sum(case))


@pytest.mark.parametrize('case', [(2, 40, 40, 128, 64), (2, 8, 24, 64, 64)])
def test_rows256_ragged_data_gradient(ops, case):
    B, H, W, Ci, Co = case
    dgrad_case(ops, B, H, W, Ci, Co, sum(case))


def test_rows256_tiles_not_multiple_of_sms(ops):
    """5 images x 64 tiles x 2 N tiles = 640 tiles: every CTA walks several, and the last round leaves some CTAs idle"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert 640 % sms != 0
    forward_case(ops, 5, 128, 128, 64, 256, 11)


def test_rows256_negative_control(ops):
    """one tap left out of the 16 x 16 kernel's tap list: the error against fp64 must exceed the bound the tests use"""
    err = forward_case(ops, 2, 32, 32, 64, 128, 12, drop_tap=4)
    assert err > 10 * fp64_tol(9 * 64), err


def test_rows256_default_selection_bitwise(ops):
    """the library default picks the 16 x 16 kernel with most of a wave of its tiles (8 x 128^2: 512 tiles) and the 16 x 8
    kernel below that (5 x 64^2: 80 tiles of 16 x 16, 160 of 16 x 8): both agree with the forced 16 x 8 kernel bit for bit"""
    for B, H, W, Ci, Co in [(8, 128, 128, 64, 32), (5, 64, 64, 64, 128)]:
        g = torch.Generator().manual_seed(H + Co)
        x = nhwc(tf32_rn(torch.randn(B, Ci, H, W, generator=g))).cuda()
        w = tf32_rn(torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5).cuda()
        taps = ops.taps_conv(3, 1)
        pw = ops.pack_weight(w, taps, round_tf32=False)
        outs = []
        for mode in (ROWS, 0):
            out = torch.full((B, H, W, Co), 7.0, device='cuda')
            run(ops, ops.make_conv_desc([(ops.View(x), taps, pw, False)], ops.View(out), (B, H, W), Cout=Co), mode)
            outs.append(out.cpu())
        assert torch.equal(outs[0], outs[1])
