"""Epilogue operands of the 16 x 16 shared-row convolution, which TMA-loads resid / aux into shared memory: channel views of wider
buffers (ld > Cout) with the output written in place over resid, Cout that is not a multiple of the 32-channel slice, more tiles
than CTAs so that the operand buffers are reused across tiles, and aux together with out2.  Every case bitwise against the 16 x 8
shared-row kernel, which reads the operands from global memory; a negative control shows that an operand shifted by one slice
is caught."""
import pytest
import torch

pytestmark = pytest.mark.gpu

ROWS, ROWS256 = 1, 4          # cd_conv_tc_set_halo modes: 16 x 8 tiles, 16 x 16 tiles wherever eligible
PAD = 40                      # extra channels of the wider operand buffers; views start at channel 8


def tf32_rn(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


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


def problem(ops, B, H, W, Ci, Co, seed, dgrad):
    """NHWC source and packed weights of a 3x3 forward (dgrad: data-gradient taps) convolution with Co output channels"""
    g = torch.Generator().manual_seed(seed)
    x = tf32_rn(torch.randn(B, H, W, Ci, generator=g)).cuda()
    if dgrad:
        w = tf32_rn(torch.randn(Ci, Co, 3, 3, generator=g) / (Ci * 9) ** 0.5).cuda()
        taps = ops.taps_conv_dgrad(3, 1)
        pw = ops.pack_weight(w, taps, mode=1, round_tf32=False)
    else:
        w = tf32_rn(torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5).cuda()
        taps = ops.taps_conv(3, 1)
        pw = ops.pack_weight(w, taps, round_tf32=False)
    return g, [(ops.View(x), taps, pw, False)]


def resid_in_place(ops, B, H, W, Ci, Co, seed):
    """out = conv + bias + out on a channel view of a wider buffer, as the engine's second block convolution does; returns the
    buffer as each kernel leaves it"""
    g, srcs = problem(ops, B, H, W, Ci, Co, seed, False)
    bias = torch.randn(Co, generator=g).cuda()
    buf0 = torch.randn(B, H, W, Co + PAD, generator=g).cuda()
    res = []
    for mode in (ROWS, ROWS256):
        buf = buf0.clone()
        v = ops.View(buf, 8, Co)
        run(ops, ops.make_conv_desc(srcs, v, (B, H, W), Cout=Co, bias=bias, resid=v), mode)
        res.append(buf.cpu())
    assert not torch.equal(res[0], buf0.cpu())
    return res


def aux_view(ops, B, H, W, Ci, Co, seed, out2=False):
    """dX = conv(dY, W^T) x GELU'(aux) with aux a channel view of a wider buffer (and out2 = the product's first factor)"""
    g, srcs = problem(ops, B, H, W, Ci, Co, seed, True)
    abuf = torch.randn(B, H, W, Co + PAD, generator=g).cuda()
    res = []
    for mode in (ROWS, ROWS256):
        out = torch.full((B, H, W, Co), 7.0, device='cuda')
        pre = torch.full((B, H, W, Co), 7.0, device='cuda') if out2 else None
        d = ops.make_conv_desc(srcs, ops.View(out), (B, H, W), Cout=Co, act=ops.ACT_GELU_BWD, aux=ops.View(abuf, 8, Co),
                               out2=ops.View(pre) if out2 else None)
        run(ops, d, mode)
        res.append((out.cpu(), pre.cpu() if out2 else None))
    assert not (res[0][0] == 7.0).any()
    return res


@pytest.mark.parametrize('Co', [64, 128, 36, 100, 160])
def test_resid_view_wider_than_cout_in_place(ops, Co):
    """Cout 36 / 100 / 160: the last slice is partly beyond Cout (100: four channels), so the staged operand is zero-filled there
    and the neighbouring channels of the buffer must keep their values"""
    a, b = resid_in_place(ops, 2, 32, 32, 64, Co, Co)
    assert torch.equal(a, b)


@pytest.mark.parametrize('Co', [64, 128, 36, 100, 160])
def test_aux_view_wider_than_cout(ops, Co):
    a, b = aux_view(ops, 2, 32, 32, 64, Co, Co + 1)
    assert torch.equal(a[0], b[0])


@pytest.mark.parametrize('case', [(2, 40, 40, 64, 96), (1, 24, 40, 32, 36), (2, 8, 24, 64, 64)])
def test_aux_with_out2_ragged(ops, case):
    """out2 overwrites the staged aux in place, so aux must be read first; ragged grids zero-fill the operand outside the image"""
    B, H, W, Ci, Co = case
    a, b = aux_view(ops, B, H, W, Ci, Co, sum(case), out2=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize('Co', [128, 192])
def test_operand_buffers_reused_across_tiles(ops, Co):
    """5 images of 128 x 128 pixels: 320 or 640 tiles of 16 x 16, not a multiple of the SM count, so every CTA walks several
    tiles and the last round leaves some CTAs idle"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert 320 % sms != 0 and 640 % sms != 0
    a, b = resid_in_place(ops, 5, 128, 128, 32, Co, 3 * Co)
    assert torch.equal(a, b)
    a, b = aux_view(ops, 5, 128, 128, 32, Co, 3 * Co + 1)
    assert torch.equal(a[0], b[0])


def test_operand_shifted_by_one_slice_is_caught(ops):
    """the 16 x 16 kernel given resid 32 channels (one slice) further along differs from the 16 x 8 kernel given the right one,
    and agrees with it given the same shifted view"""
    B, H, W, Co = 2, 32, 32, 64
    g, srcs = problem(ops, B, H, W, 64, Co, 5, False)
    rbuf = torch.randn(B, H, W, Co + PAD, generator=g).cuda()

    def conv(mode, c0):
        out = torch.full((B, H, W, Co), 7.0, device='cuda')
        run(ops, ops.make_conv_desc(srcs, ops.View(out), (B, H, W), Cout=Co, resid=ops.View(rbuf, c0, Co)), mode)
        return out.cpu()

    assert not torch.equal(conv(ROWS, 8), conv(ROWS256, 40))
    assert torch.equal(conv(ROWS, 40), conv(ROWS256, 40))


@pytest.mark.parametrize('case', [(128, 8, 8, 128, 256), (128, 4, 4, 256, 256), (128, 16, 16, 128, 128)])
def test_small_grids_many_images(ops, case):
    """grids smaller than one 16 x 16 tile with many images, as the DDPM Model's lower levels at batch 128: every CTA walks
    several tiles whose second warpgroup lies wholly outside the image (8 x 8) or whose second operand half does (4 x 4)"""
    B, H, W, Ci, Co = case
    a, b = resid_in_place(ops, B, H, W, Ci, Co, sum(case))
    assert torch.equal(a, b)
    a, b = aux_view(ops, B, H, W, Ci, Co, sum(case) + 1)
    assert torch.equal(a[0], b[0])
