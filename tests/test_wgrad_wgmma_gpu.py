"""wgmma weight gradient of the stride-1 3x3 convolutions (csrc/wgrad_tc.cu: wgrad_wgmma_kernel; X fed from registers, dY
transposed once per chunk in shared memory) against torch's fp64 reference and against the forced mma.sync halo kernel
(cd_wgrad_tc_set_mode(8)), which rounds both operands the same way but sums in another order."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEFAULT, MMA_SYNC = 1, 8          # cd_wgrad_tc_set_mode


def tf32_rn(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.fixture(scope='module')
def ops():
    from cold_diffusion_models_b200 import ops
    return ops


@pytest.fixture(scope='module')
def lib():
    from cold_diffusion_models_b200._lib import lib
    return lib


# every 3x3 convolution of Unet(64, (1, 2, 4, 8)) on 128 x 128 images: (H, W, Cin, Cout).  (128, 128, 32, 128) is the image-edge
# block (3 channels padded to 32), which stays on the mma.sync kernel.
UNET_3X3 = [(128, 128, 32, 128), (128, 128, 64, 128), (128, 128, 128, 64), (64, 64, 64, 256), (64, 64, 128, 256),
            (64, 64, 256, 128), (64, 64, 64, 128), (64, 64, 128, 64), (32, 32, 128, 512), (32, 32, 256, 512), (32, 32, 512, 256),
            (32, 32, 128, 256), (32, 32, 256, 128), (16, 16, 256, 1024), (16, 16, 512, 1024), (16, 16, 1024, 512),
            (16, 16, 256, 512), (16, 16, 512, 256)]


def problem(B, H, W, Ci, Co, seed, round_inputs):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Ci, H, W, generator=g)
    dy = torch.randn(B, Co, H, W, generator=g)
    if round_inputs:
        x, dy = tf32_rn(x), tf32_rn(dy)
    return x.cuda(), dy.cuda()


def ref_packed(x, dy, taps):
    """fp64 packed gradient [tap][Cout][Cin] = sum over pixels of dY[p][co] * X[p + (dy, dx)][ci] (zero outside the image)"""
    B, Ci, H, W = x.shape
    xp = torch.nn.functional.pad(x.double(), (1, 1, 1, 1))
    d = dy.double()
    out = [torch.einsum('bohw,bihw->oi', d, xp[:, :, 1 + ty:1 + ty + H, 1 + tx:1 + tx + W]) for (_, _, ty, tx) in taps]
    return torch.stack(out)


def run(ops, lib, x, dy, mode, dw0=None, db=None):
    B, Ci, H, W = x.shape
    Co = dy.shape[1]
    taps = ops.taps_conv(3, 1)
    dwp = torch.zeros(9, Co, Ci, device='cuda') if dw0 is None else dw0.clone()
    lib.cd_wgrad_tc_set_mode(mode)
    try:
        dyv = ops.View(nhwc(dy))
        d = ops.make_conv_desc([(ops.View(nhwc(x)), taps, dwp, False)], dyv, (B, H, W), Cout=Co)
        ops.conv_wgrad(d, dyv, dwp, db, impl=ops.CONV_TC)
        torch.cuda.synchronize()
    finally:
        lib.cd_wgrad_tc_set_mode(DEFAULT)
    return dwp, taps


@pytest.mark.parametrize('shape', UNET_3X3, ids=lambda s: '%dx%d-%d-%d' % s)
def test_unet_shapes_vs_fp64(ops, lib, shape):
    H, W, Ci, Co = shape
    x, dy = problem(2, H, W, Ci, Co, 5, True)
    dwp, taps = run(ops, lib, x, dy, DEFAULT)
    e = rel(dwp, ref_packed(x, dy, taps))
    print('wgmma vs fp64 %-22s rel %.3e' % (shape, e))
    assert e < 1e-5, e


@pytest.mark.parametrize('shape', UNET_3X3, ids=lambda s: '%dx%d-%d-%d' % s)
def test_unet_shapes_vs_mma_sync_unrounded(ops, lib, shape):
    """unrounded fp32 inputs: both kernels must round X and dY RN to TF32 identically"""
    H, W, Ci, Co = shape
    x, dy = problem(2, H, W, Ci, Co, 6, False)
    a, _ = run(ops, lib, x, dy, DEFAULT)
    b, _ = run(ops, lib, x, dy, MMA_SYNC)
    e = rel(a, b)
    print('wgmma vs mma.sync %-22s rel %.3e' % (shape, e))
    assert e < 1e-5, e


def test_accumulates_into_existing_gradient(ops, lib):
    x, dy = problem(2, 32, 32, 128, 256, 7, True)
    dw0 = torch.randn(9, 256, 128, generator=torch.Generator().manual_seed(8)).cuda()
    dwp, taps = run(ops, lib, x, dy, DEFAULT, dw0=dw0)
    e = rel(dwp, dw0.double() + ref_packed(x, dy, taps))
    assert e < 1e-5, e


@pytest.mark.parametrize('shape', [(3, 64, 64, 128, 64), (2, 16, 16, 1024, 64), (4, 8, 8, 64, 64), (2, 16, 16, 1024, 128)],
                         ids=lambda s: '%d-%dx%d-%d-%d' % s)
def test_narrow_cout_and_wide_cin(ops, lib, shape):
    """Cout = 64 (64-wide N tiles, four taps per consumer warpgroup), Cin = 1024, and an 8 x 8 grid (8-pixel chunk rows)"""
    B, H, W, Ci, Co = shape
    x, dy = problem(B, H, W, Ci, Co, 9, True)
    dwp, taps = run(ops, lib, x, dy, DEFAULT)
    e = rel(dwp, ref_packed(x, dy, taps))
    assert e < 1e-5, e


def test_ragged_last_split(ops, lib):
    """5 images of 16 x 16 = 20 chunks of 64 pixels; at most one wave of splits gives 3 splits of 7, 7 and 6 chunks"""
    x, dy = problem(5, 16, 16, 64, 128, 10, True)
    lib.cd_wgrad_tc_set_split(1, 0)
    try:
        dwp, taps = run(ops, lib, x, dy, DEFAULT)
    finally:
        lib.cd_wgrad_tc_set_split(3, 12000)
    ref = ref_packed(x, dy, taps)
    assert rel(dwp, ref) < 1e-5
    b, _ = run(ops, lib, x, dy, MMA_SYNC)
    assert rel(dwp, b) < 1e-5


def test_image_edge_and_bias_fusion_fall_back(ops, lib):
    """Cin = 32 (image-edge block) and the opt-in bias fusion run on the mma.sync kernel and stay correct"""
    x, dy = problem(2, 32, 32, 32, 128, 11, True)
    dwp, taps = run(ops, lib, x, dy, DEFAULT)
    assert rel(dwp, ref_packed(x, dy, taps)) < 1e-5
    x, dy = problem(2, 32, 32, 64, 128, 12, True)
    db = torch.zeros(128, device='cuda')
    lib.cd_wgrad_tc_set_bias_fusion(1)
    try:
        dwp, taps = run(ops, lib, x, dy, DEFAULT, db=db)
    finally:
        lib.cd_wgrad_tc_set_bias_fusion(0)
    assert rel(dwp, ref_packed(x, dy, taps)) < 1e-5
    assert rel(db, dy.double().sum(dim=(0, 2, 3))) < 1e-5
