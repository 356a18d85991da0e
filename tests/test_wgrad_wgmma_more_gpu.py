"""wgmma weight gradient (csrc/wgrad_tc.cu: wgrad_wgmma_kernel) of the non-3x3 problems of the Unet: 1x1 (res_conv, to_qkv),
the per-batch attention product dweff, the 4x4 stride-2 downsample (split into input-parity classes), the transposed-convolution
parity problems of the upsample, and the image-edge block (Cin = 32).  Checked against an fp64 reference on TF32-rounded inputs
and against the forced mma.sync halo kernel (cd_wgrad_tc_set_mode(8)) on unrounded inputs: both round X and dY RN to TF32."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEFAULT, MMA_SYNC = 1, 8          # cd_wgrad_tc_set_mode


def tf32_rn(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


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


def reference(x, dy, taps, stride, out_map, per_batch):
    """fp64: dW[tap][co][ci] = sum over the grid g of dY[g * os + o0][co] * X[g * s + d][ci] (zero outside the image); x, dy NHWC
    over the grid (B, Hg, Wg) = dy's sub-grid.  per_batch: one gradient per image."""
    B, Hx, Wx, Ci = x.shape
    oys, oxs, oy0, ox0 = out_map
    d = dy.double()[:, oy0::oys, ox0::oxs, :]
    Hg, Wg = d.shape[1], d.shape[2]
    xp = torch.nn.functional.pad(x.double(), (0, 0, 2, 2 + stride * Wg, 2, 2 + stride * Hg))
    out = []
    for (_, _, ty, tx) in taps:
        xs = xp[:, 2 + ty:2 + ty + stride * Hg:stride, 2 + tx:2 + tx + stride * Wg:stride, :]
        out.append(torch.einsum('bhwo,bhwi->boi' if per_batch else 'bhwo,bhwi->oi', d, xs))
    return torch.stack(out, dim=1).flatten(1, 2) if per_batch else torch.stack(out)      # per batch: [B][tap * Cout][Cin]


def problem(seed, B, Hx, Wx, Ci, Ho, Wo, Co, round_inputs, x_ld=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Hx, Wx, x_ld or Ci, generator=g)
    dy = torch.randn(B, Ho, Wo, Co, generator=g)
    if round_inputs:
        x, dy = tf32_rn(x), tf32_rn(dy)
    return x.cuda(), dy.cuda()


def run(ops, lib, x, dy, taps, grid, stride, out_map, mode, Ci, per_batch=False, dw0=None):
    Co = dy.shape[-1]
    shape = (grid[0], Co, Ci) if per_batch else (len(taps), Co, Ci)
    dw = torch.zeros(shape, device='cuda') if dw0 is None else dw0.clone()
    lib.cd_wgrad_tc_set_mode(mode)
    try:
        dyv = ops.View(dy)
        d = ops.make_conv_desc([(ops.View(x, 0, Ci), taps, dw, per_batch)], dyv, grid, stride=stride, Cout=Co, out_map=out_map)
        ops.conv_wgrad(d, dyv, dw, None, impl=ops.CONV_TC)
        torch.cuda.synchronize()
    finally:
        lib.cd_wgrad_tc_set_mode(DEFAULT)
    return dw


# (kind, H, W, Cin, Cout) of Unet(64, (1, 2, 4, 8)) on 128 x 128 images; H x W is the input grid of the layer
DOWN = [('down', 128, 128, 64, 64), ('down', 64, 64, 128, 128), ('down', 32, 32, 256, 256)]
UP = [('up%d%d' % (py, px), h, h, c, c) for (h, c) in ((16, 256), (32, 128), (64, 64)) for py in (0, 1) for px in (0, 1)]
ONE = [('1x1', 128, 128, 64, 384), ('1x1', 64, 64, 64, 128), ('1x1', 64, 64, 128, 384), ('1x1', 64, 64, 256, 64),
       ('1x1', 32, 32, 128, 256), ('1x1', 32, 32, 256, 384), ('1x1', 32, 32, 512, 128), ('1x1', 32, 32, 256, 128),
       ('1x1', 16, 16, 256, 512), ('1x1', 16, 16, 256, 384), ('1x1', 16, 16, 1024, 256), ('1x1', 16, 16, 512, 384),
       ('1x1', 16, 16, 512, 256)]
DWEFF = [('dweff', h, h, 128, c) for (h, c) in ((128, 64), (64, 128), (32, 256), (16, 512))]
EDGE = [('edge3', 128, 128, 32, 128), ('edge1', 128, 128, 32, 64)]
SHAPES = DOWN + UP + ONE + DWEFF + EDGE


def setup(ops, kind, H, W, Ci, Co, seed, round_inputs, B=2):
    """-> (x, dy, taps, grid, stride, out_map, per_batch)"""
    if kind == 'down':
        x, dy = problem(seed, B, H, W, Ci, H // 2, W // 2, Co, round_inputs)
        return x, dy, ops.taps_conv(4, 1), (B, H // 2, W // 2), 2, (1, 1, 0, 0), False
    if kind.startswith('up'):
        py, px = int(kind[2]), int(kind[3])
        x, dy = problem(seed, B, H, W, Ci, 2 * H, 2 * W, Co, round_inputs)
        return x, dy, ops.taps_convT4_parity(py, px), (B, H, W), 1, (2, 2, py, px), False
    if kind == 'dweff':        # q: the first 128 channels of the 384-channel qkv rows
        x, dy = problem(seed, B, H, W, Ci, H, W, Co, round_inputs, x_ld=384)
        return x, dy, ops.taps_conv(1, 0), (B, H, W), 1, (1, 1, 0, 0), True
    x, dy = problem(seed, B, H, W, Ci, H, W, Co, round_inputs)
    taps = ops.taps_conv(3, 1) if kind == 'edge3' else ops.taps_conv(1, 0)
    return x, dy, taps, (B, H, W), 1, (1, 1, 0, 0), False


def ident(s):
    return '%s-%dx%d-%d-%d' % s


@pytest.mark.parametrize('shape', SHAPES, ids=ident)
def test_vs_fp64(ops, lib, shape):
    kind, H, W, Ci, Co = shape
    x, dy, taps, grid, stride, om, pb = setup(ops, kind, H, W, Ci, Co, 21, True)
    dw = run(ops, lib, x, dy, taps, grid, stride, om, DEFAULT, Ci, per_batch=pb)
    e = rel(dw, reference(x[..., :Ci], dy, taps, stride, om, pb))
    print('wgmma vs fp64 %-28s rel %.3e' % (ident(shape), e))
    assert e < 1e-5, e


@pytest.mark.parametrize('shape', SHAPES, ids=ident)
def test_vs_mma_sync_unrounded(ops, lib, shape):
    kind, H, W, Ci, Co = shape
    x, dy, taps, grid, stride, om, pb = setup(ops, kind, H, W, Ci, Co, 22, False)
    a = run(ops, lib, x, dy, taps, grid, stride, om, DEFAULT, Ci, per_batch=pb)
    b = run(ops, lib, x, dy, taps, grid, stride, om, MMA_SYNC, Ci, per_batch=pb)
    e = rel(a, b)
    print('wgmma vs mma.sync %-28s rel %.3e' % (ident(shape), e))
    assert e < 1e-5, e


@pytest.mark.parametrize('kind', ['1x1', 'down', 'up11'])
def test_accumulates_into_existing_gradient(ops, lib, kind):
    x, dy, taps, grid, stride, om, pb = setup(ops, kind, 32, 32, 128, 128, 23, True)
    dw0 = torch.randn(len(taps), 128, 128, generator=torch.Generator().manual_seed(24)).cuda()
    dw = run(ops, lib, x, dy, taps, grid, stride, om, DEFAULT, 128, dw0=dw0)
    assert rel(dw, dw0.double() + reference(x, dy, taps, stride, om, pb)) < 1e-5


@pytest.mark.parametrize('kind', ['1x1', 'down', 'up01'])
def test_ragged_last_split(ops, lib, kind):
    """5 images of 16 x 16 (8 x 8 for the downsample) with at most one wave of splits: the last split is shorter"""
    x, dy, taps, grid, stride, om, pb = setup(ops, kind, 16, 16, 64, 128, 25, True, B=5)
    lib.cd_wgrad_tc_set_split(1, 0)
    try:
        dw = run(ops, lib, x, dy, taps, grid, stride, om, DEFAULT, 64)
    finally:
        lib.cd_wgrad_tc_set_split(3, 12000)
    assert rel(dw, reference(x, dy, taps, stride, om, pb)) < 1e-5


def test_per_batch_several_splits_per_image(ops, lib):
    """dweff at 64 x 64: 64 chunks per image; two full waves of splits give every image several splits"""
    x, dy, taps, grid, stride, om, pb = setup(ops, 'dweff', 64, 64, 128, 64, 26, True, B=3)
    lib.cd_wgrad_tc_set_split(2, 0)
    try:
        dw = run(ops, lib, x, dy, taps, grid, stride, om, DEFAULT, 128, per_batch=True)
    finally:
        lib.cd_wgrad_tc_set_split(3, 12000)
    assert rel(dw, reference(x[..., :128], dy, taps, stride, om, True)) < 1e-5


@pytest.mark.parametrize('kind', ['1x1', 'up10', 'edge3', 'dweff'])
def test_8x8_grid(ops, lib, kind):
    Ci = 32 if kind == 'edge3' else 128
    x, dy, taps, grid, stride, om, pb = setup(ops, kind, 8, 8, Ci, 64, 27, True, B=3)
    dw = run(ops, lib, x, dy, taps, grid, stride, om, DEFAULT, Ci, per_batch=pb)
    assert rel(dw, reference(x[..., :Ci], dy, taps, stride, om, pb)) < 1e-5
