"""`Unet(64, (1, 2, 4, 8))` at the 32² shapes of the MNIST and CIFAR-10 drivers (train_batch_size = 32) on the default
tensor-core path, against float64 references computed on the GPU from oracle/.

At 32² the two deepest levels are 8 x 8 (256 channels) and 4 x 4 (512 channels and the mid block), where dispatch picks kernels
that larger images never reach: the depthwise tile kernel, the per-tap convolution with several images per 128-row tile, the
small-npix LayerNorm, the scalar batched column sums and one mostly-empty linear-attention span per image.

1. End to end (B = 32 with 3 and 1 channels, and B = 5, whose multi-image tiles are left partly empty): parameter gradients,
   input gradient, one Trainer step (two micro-batches, Adam + EMA), a CUDA-graph EMA sample and batch independence.
2. Each small-level entry point called directly at the (B, H, W, C, ld) the engine passes, against float64.  The convolutions
   are the engine's own descriptors, recorded from a 32² training step and replayed on TF32-rounded operands.
3. A profiler run of one training step shows that these kernel variants really run.

Every comparison also evaluates its metric on a deliberately wrong reference (a negative control) and asserts that it exceeds
the bound.  Every bound is at most 3x the value measured on an H100 80GB HBM3 (700 W), which is in the comment beside it.  Set
COLDDIFF_TEST_METRICS=<file> to write all values and controls as JSON.  The file runs in about 55 s on that card; its peak
device memory is 6.8 GiB."""
import contextlib
import ctypes as C
import io
import math

import pytest
import torch
import torch.nn.functional as F

import deblur_oracle as DO
import unet_oracle as UO
from test_config3_step_gpu import (Checks, _metrics_file, _free_between_tests, _METRICS, rel, gen, blur_per_image,  # noqa: F401
                                   ref_step, engine_grads, grad_errors, stats, call, ptr, stream, sentinel, randn, F32,
                                   _attn_core64)
from test_input_grad_gpu import _unet_ref, _engine_dx, _check_dx, _record_calls

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
S = 32                     # image side: the 8 x 8 and 4 x 4 levels below exist only for S = 32
T = 20
LR = 1e-3


def tf32_rn(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def _unet(channels, seed=3):
    import cold_diffusion_models_b200 as cdm
    with contextlib.redirect_stdout(io.StringIO()):
        unet = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=channels).to(DEV)
        sd = UO.make_unet_state_dict(64, (1, 2, 4, 8), channels, seed=seed)
        unet.load_state_dict(sd)
    return unet, sd


def _gd(unet, channels):
    import cold_diffusion_models_b200 as cdm
    return cdm.GaussianDiffusion(unet, image_size=S, device_of_kernel='cuda', channels=channels, timesteps=T, kernel_std=0.1,
                                 kernel_size=11, blur_routine='Exponential_reflect', loss_type='l2',
                                 sampling_routine='x0_step_down').to(DEV)


def _blur(channels, denoise_fn=None, **kw):
    kw.update(image_size=S, channels=channels, timesteps=T, kernel_std=0.1, kernel_size=11, blur_routine='Exponential_reflect')
    o = DO.DeblurOracle(denoise_fn, **kw)
    o.kernels2d = [k.double().cuda() for k in o.kernels2d]
    return o


def _fp64_net(sd):
    sd64 = {k: v.detach().to(DEV, F64) for k, v in sd.items()}
    return lambda a, s: UO.unet_forward(sd64, a, s.to(a.device, F64))


def _batch(B, channels, seed):
    x = torch.rand(B, channels, S, S, generator=gen(seed), device=DEV) * 2 - 1
    t = torch.randint(0, T, (B,), generator=gen(seed + 1), device=DEV)
    t[0], t[1] = 0, T - 1
    return x, t


def _groups(B):
    """reference chunks: the images of one 4 x 4-level tile (TN = 8) at B = 32; the last image alone at B = 5"""
    return [(i, min(i + 8, B)) for i in range(0, B, 8)] if B % 8 == 0 else [(0, B - 1), (B - 1, B)]


def _ref_parts(sd, x, xt64, t, norm):
    return [ref_step(sd, x[a:b], xt64[a:b], t[a:b], norm=norm, chunk=8)[0] for a, b in _groups(x.shape[0])]


def _sum(parts):
    return {k: sum(p[k] for p in parts) for k in parts[0]}


def _grad_check(ck, name, eg, ref, ctrl, bmed, bworst):
    errs = grad_errors(eg, ref)
    med, p90, worst = stats(errs)
    cmed, _, cworst = stats(grad_errors(eg, ctrl))
    _METRICS['%s::%s p90' % (ck.test, name)] = p90
    _METRICS['%s::%s worst parameters' % (ck.test, name)] = [(e, n) for e, n in errs[-5:]]
    ck.require('%s: %d parameter gradients' % (name, len(errs)), len(errs) == 238)
    ck('%s median' % name, med, bmed, cmed)
    ck('%s worst' % name, worst, bworst, cworst)
    ck.require('%s: controls 10x past the bounds (%.3e, %.3e)' % (name, cmed, cworst), cmed > 10 * bmed and cworst > 10 * bworst)


# ==========================================================================================================================
# 1. end to end on the default tensor-core path
# ==========================================================================================================================
CASES = [('cifar-b32', 3, 32), ('mnist-b32', 1, 32), ('cifar-b5', 3, 5)]
# bounds per case, each at most 3x the value measured on the H100 (in the comment below it): grad median, grad worst, dx,
# step-gradient median and worst, after-step median and worst, graphed sample's direct reconstruction, graphed sample
BOUNDS = {
    'cifar-b32': (2.9e-3, 7.5e-3, 3.2e-3, 2.8e-3, 8.0e-3, 1.6e-3, 3.6e-3, 3.9e-4, 9.2e-4),
    # measured in two runs 9.7e-4, 2.5e-3 / 1.9e-3 (downs.0.0.ds_conv.weight), 1.08e-3, 9.4e-4, 2.7e-3 / 2.5e-3, 5.4e-4,
    # 1.3e-3, 1.3e-4, 3.1e-4
    'mnist-b32': (2.8e-3, 5.5e-3, 3.1e-3, 2.8e-3, 5.8e-3, 1.4e-3, 1.26e-2, 3.5e-4, 5.0e-4),
    # measured in two runs 9.4e-4, 1.85e-3, 1.04e-3, 9.6e-4, 1.95e-3, 4.7e-4, 4.2e-3 / 5.4e-3 (downs.0.0 conditioning),
    # 1.17e-4, 1.67e-4
    'cifar-b5': (2.8e-3, 5.8e-3, 3.3e-3, 2.8e-3, 5.0e-3, 1.7e-3, 5.7e-3, 3.8e-4, 9.5e-4),
    # measured in two runs 9.6e-4, 1.95e-3, 1.10e-3, 9.4e-4, 1.67e-3, 5.8e-4, 1.9e-3, 1.31e-4, 3.2e-4
}


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_unet32_gradients_step_and_graphed_sample(case, tmp_path):
    """parameter and input gradients of one micro-batch, one Trainer step (gradient_accumulate_every = 2, Adam + EMA) and the
    gradient at the new weights, and a graphed 3-step sample of the EMA model, against float64"""
    import cold_diffusion_models_b200 as cdm
    name, ch, B = case
    bmed, bworst, bdx, bsmed, bsworst, bamed, baworst, bdirect, bsample = BOUNDS[name]
    ck = Checks('unet32 %s' % name)
    unet, sd = _unet(ch, seed=3)
    gd = _gd(unet, ch)
    o = _blur(ch)
    x, t = _batch(B, ch, 40 + B + ch)
    x2, t2 = _batch(B, ch, 60 + B + ch)
    xt64 = blur_per_image(o, x.double(), t)
    xt64_2 = blur_per_image(o, x2.double(), t2)
    N = x.numel()
    # ---- gradients of one micro-batch; control: the images of the last 4 x 4-level tile (B = 5: the last image) left out
    unet.zero_grad(set_to_none=True)
    gd.p_losses(x, t).backward()
    eg = engine_grads(unet)
    parts = _ref_parts(sd, x, xt64, t, N)
    ref_old = _sum(parts)
    _grad_check(ck, 'grad', eg, ref_old, _sum(parts[:-1]), bmed, bworst)
    del eg, parts
    # ---- input gradient (L2 against a fixed target); controls: one term of dx left out, images 0 and 1 swapped
    unet.zero_grad(set_to_none=True)
    target = torch.rand(B, ch, S, S, generator=gen(77), device=DEV) * 2 - 1
    ref, dw, res, _ = _unet_ref(unet, x, target, t, False)
    dx = _engine_dx(unet, x, target, t)
    _check_dx(ck, 'dx', dx, ref, {'the depthwise path': dw, 'the res_conv path': res}, bdx)
    swapped = rel(dx, ref[torch.tensor([1, 0] + list(range(2, B)), device=DEV)])
    ck('dx vs images 0 and 1 swapped', 0.0, bdx, swapped)
    ck.require('dx swap control %.3e not 10x past %.1e' % (swapped, bdx), swapped > 10 * bdx)
    del ref, dw, res, dx
    unet.zero_grad(set_to_none=True)
    # ---- one Trainer step over the micro-batches (x, t) and (x2, t2): what the optimizer read is snapshotted
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=LR, train_num_steps=10 ** 9,
                         gradient_accumulate_every=2, ema_decay=0.995, fp16=False, results_folder=str(tmp_path),
                         dataset='synthetic')
    eng = unet.engine
    ts = iter([t, t2])
    gd.forward = lambda d: gd.p_losses(d, next(ts))          # the Trainer's micro-batches with fixed per-image t
    snap = {}
    step = tr.opt.step

    def snapshot_step(**kw):
        snap.update(p0=eng.flat_param.clone(), g0=eng.flat_grad.clone(), eg=engine_grads(unet), kw=kw)
        step(**kw)
    tr.opt.step = snapshot_step
    try:
        loss = tr.train_step([x, x2]).item()
        torch.cuda.synchronize()
    finally:
        tr.opt.step = step
        del gd.forward
    ck.require('train_step loss finite (%r)' % loss, math.isfinite(loss))
    parts2 = _ref_parts(sd, x2, xt64_2, t2, N)
    ref_mb2 = _sum(parts2)
    ref_step_g = {k: (ref_old[k] + ref_mb2[k]) / 2 for k in ref_old}
    ctrl = {k: ref_step_g[k] - parts2[-1][k] / 2 for k in ref_old}          # the second micro-batch's last tile left out
    _grad_check(ck, 'step gradient', snap['eg'], ref_step_g, ctrl, bsmed, bsworst)
    del parts2, ref_mb2, ref_step_g, ctrl
    # the update against Adam (step 1, the kernel's fp32 betas) in fp64 on the gradient it read; control: no bias correction
    gs = snap['kw'].get('grad_scale', 1.0)
    b1, b2 = F32(0.9), F32(0.999)
    g64 = snap['g0'].double() * gs
    m64, v64 = (1 - b1) * g64, (1 - b2) * g64 * g64
    d_r = -LR / (1 - b1) * m64 / (v64.sqrt() / math.sqrt(1 - b2) + 1e-8)
    d_k = eng.flat_param.double() - snap['p0'].double()
    wrong = -LR * m64 / (v64.sqrt() + 1e-8)
    ck('Adam update (max |err| / lr)', (d_k - d_r).abs().max().item() / LR, 1.8e-4,      # measured 6.0e-5 (fp32 rounding of p)
       (wrong - d_r).abs().max().item() / LR)
    ck.require('EMA copied the new weights at step 0', bool(torch.equal(tr._ema_unet.engine.flat_param, eng.flat_param)))
    del g64, m64, v64, d_r, d_k, wrong, snap
    # ---- gradient at the new weights; control: the reference at the old weights
    tr.opt.zero_grad()
    gd.p_losses(x, t).backward()
    torch.cuda.synchronize()
    eg = engine_grads(unet)
    tr.opt.zero_grad()
    sd1 = {k: v.detach().clone() for k, v in unet.state_dict().items()}
    ref_new = _sum(_ref_parts(sd1, x, xt64, t, N))
    _grad_check(ck, 'grad after the step', eg, ref_new, ref_old, bamed, baworst)
    del ref_new, ref_old, eg, sd1
    # ---- the graphed 3-step x0_step_down sample of the EMA model
    ema = tr.ema_model
    eeng = ema.denoise_fn.engine
    eeng.enable_cuda_graph(True)
    try:
        with torch.no_grad():
            xt, dr, img = ema.sample(batch_size=B, img=x, t=3)
        torch.cuda.synchronize()
    finally:
        eeng.enable_cuda_graph(False)
    os_ = _blur(ch, denoise_fn=_fp64_net(ema.denoise_fn.state_dict()), sampling_routine='x0_step_down')
    with torch.no_grad():
        r = os_.sample(B, x.double(), t=3)
    ck('graphed sample x_t', rel(xt, r[0]), 3.4e-7,                    # measured 1.15e-7
       rel(xt, blur_per_image(o, x.double(), torch.full((B,), 1))))
    ck('graphed sample direct', rel(dr, r[1]), bdirect, rel(xt, r[1]))
    ck('graphed sample', rel(img, r[2]), bsample, rel(xt, r[2]))
    ck.done()


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_unet32_batch_independence(case):
    """the gradient of the whole batch in one pass against the sum of the same engine's gradients over B one-image passes
    (other tiles, spans and weight-gradient splits; the same arithmetic per image).  Control: image 3's pass left out."""
    name, ch, B = case
    ck = Checks('unet32 batch independence %s' % name)
    unet, _ = _unet(ch, seed=6)
    gd = _gd(unet, ch)
    x, t = _batch(B, ch, 90 + B + ch)
    unet.zero_grad(set_to_none=True)
    gd.p_losses(x, t).backward()
    whole = engine_grads(unet)
    unet.zero_grad(set_to_none=True)
    for i in [i for i in range(B) if i != 3] + [3]:
        if i == 3:
            partial = engine_grads(unet)
        (gd.p_losses(x[i:i + 1], t[i:i + 1]) / B).backward()
    split = engine_grads(unet)
    unet.zero_grad(set_to_none=True)
    # measured median 1.8e-4 / 1.3e-4 / 2.2e-4 (cifar-b32 / mnist-b32 / cifar-b5), worst 6.4e-4 / 4.4e-4 / 7.9e-4; image 3's pass
    # left out: median 4.3e-2 / 3.4e-2 / 0.29
    bmed, bworst = {'cifar-b32': (5.4e-4, 1.9e-3), 'mnist-b32': (3.9e-4, 1.3e-3), 'cifar-b5': (6.7e-4, 2.3e-3)}[name]
    _grad_check(ck, 'grad', split, whole, partial, bmed, bworst)
    ck.done()


# ==========================================================================================================================
# 2. the small-level kernels called directly
# ==========================================================================================================================
def _dw_refs(x, dh, add, w, bias, cond):
    """float64 depthwise 7x7 forward (+ bias + cond + addend), its data gradient (flipped kernel) and weight gradient; NHWC in"""
    Cc = w.shape[0]
    xc = x.double().permute(0, 3, 1, 2)
    dhc = dh.double().permute(0, 3, 1, 2)
    fwd = (F.conv2d(xc, w.double(), bias.double(), padding=3, groups=Cc) + cond.double()[:, :, None, None]).permute(0, 2, 3, 1)
    fwd = fwd + add.double()
    flip = F.conv_transpose2d(dhc, w.double(), padding=3, groups=Cc).permute(0, 2, 3, 1)
    wg = torch.nn.grad.conv2d_weight(xc, w.shape, dhc, padding=3, groups=Cc).reshape(Cc, 49)
    return fwd, flip, wg


DW_CASES = [(32, 8, 256, 256), (32, 8, 512, 512), (32, 4, 512, 512), (32, 4, 256, 256), (32, 4, 1024, 1024),
            (5, 8, 256, 256), (5, 4, 512, 512), (32, 8, 256, 260), (32, 4, 512, 516)]


@pytest.mark.parametrize('case', DW_CASES, ids=['B%d-%dx%d-C%d-ld%d' % (c[0], c[1], c[1], c[2], c[3]) for c in DW_CASES])
def test_depthwise_small_levels_against_fp64(case):
    """cd_dwconv7_fwd (bias, cond with the engine's wider row, addend), its flip with addend, and cd_dwconv7_wgrad called twice
    (it accumulates); padding columns stay untouched.  Control: the reference without the last tap column (kx = 6)."""
    B, H, Cc, ld = case
    W = H
    ck = Checks('dwconv7 %s' % (case,))
    g = gen(1000 + B + H + Cc + ld)
    x, dh, add, add2 = (randn(B, H, W, ld, g=g) for _ in range(4))
    w = randn(Cc, 1, 7, 7, g=g, scale=1 / 7)
    bias = randn(Cc, g=g)
    cond_ld = Cc + 12
    condbuf = randn(B, cond_ld, g=g)
    cond = condbuf[:, 4:4 + Cc]
    out, dx = sentinel(B, H, W, ld), sentinel(B, H, W, ld)
    call('cd_dwconv7_fwd', ptr(x), ld, B, H, W, Cc, ptr(w), ptr(bias), C.c_void_p(cond.data_ptr()), cond_ld, ptr(out), ld, 0,
         ptr(add), ld, stream())
    call('cd_dwconv7_fwd', ptr(dh), ld, B, H, W, Cc, ptr(w), C.c_void_p(0), C.c_void_p(0), 0, ptr(dx), ld, 1, ptr(add2), ld,
         stream())
    dw0 = randn(Cc, 49, g=g)
    dw = dw0.clone()
    for _ in range(2):
        call('cd_dwconv7_wgrad', ptr(dh), ld, ptr(x), ld, B, H, W, Cc, ptr(dw), stream())
    torch.cuda.synchronize()
    xs, dhs = x[..., :Cc], dh[..., :Cc]
    fwd, flip, wg = _dw_refs(xs, dhs, add[..., :Cc], w, bias, cond)
    flip = flip + add2[..., :Cc].double()
    wc = w.clone()
    wc[..., 6] = 0
    fwd_c, flip_c, _ = _dw_refs(xs, dhs, add[..., :Cc], wc, bias, cond)
    ck('forward', rel(out[..., :Cc], fwd), 1.8e-7, rel(fwd_c, fwd))                                 # measured <= 6.0e-8
    ck('flip', rel(dx[..., :Cc], flip), 2.1e-7, rel(flip_c + add2[..., :Cc].double(), flip))        # measured <= 7.0e-8
    wg_c = wg.clone().reshape(Cc, 7, 7)
    wg_c[..., 6] = 0
    ck('wgrad x2', rel(dw, dw0.double() + 2 * wg), 5.7e-7,                                          # measured <= 1.9e-7
       rel(dw0.double() + 2 * wg_c.reshape(Cc, 49), dw0.double() + 2 * wg))
    ck.require('padding columns untouched', bool((out[..., Cc:] == 7.0).all() and (dx[..., Cc:] == 7.0).all()))
    ck.done()


# ---- convolutions: the engine's descriptors at 8 x 8 and 4 x 4, replayed ---------------------------------------------------
def _engine_tensors(eng):
    ts = [t for t in eng._bufs.values()] + [t for t in eng._packed.values() if torch.is_tensor(t)]
    for a in ('flat_grad', 'flat_param'):
        if getattr(eng, a, None) is not None:
            ts.append(getattr(eng, a))
    return [(t.data_ptr(), t.numel() * 4) for t in ts]


def _c0(addr, ld, spans):
    """channel offset of a view at `addr` in an NHWC engine buffer of row length ld"""
    for base, nb in spans:
        if base <= addr < base + nb:
            return ((addr - base) // 4) % ld
    raise AssertionError('address not in an engine buffer')


def _spec(kind, d, impl, spans, dout=None, db=False):
    """a recorded cd_conv_fwd / cd_conv_wgrad as plain values (shapes, strides, offsets, taps, epilogue)"""
    srcs = tuple((s.ld, s.C, s.H, s.W, _c0(s.src, s.ld, spans), tuple((s.dy[j], s.dx[j]) for j in range(s.ntaps)), s.w_per_batch)
                 for s in (d.s[i] for i in range(d.nsrc)))
    sp = dict(kind=kind, impl=impl, B=d.B, Hg=d.Hg, Wg=d.Wg, sy=d.sy, sx=d.sx, Cout=d.Cout, srcs=srcs,
              omap=(d.oys, d.oxs, d.oy0, d.ox0), rnd=d.round_tf32)
    if kind == 'fwd':
        sp.update(out=(d.out_ld, _c0(d.out, d.out_ld, spans), d.Ho, d.Wo), bias=bool(d.bias), act=d.act,
                  resid=(d.resid_ld, _c0(d.resid, d.resid_ld, spans), d.resid == d.out) if d.resid else None,
                  out2=(d.out2_ld, _c0(d.out2, d.out2_ld, spans)) if d.out2 else None,
                  aux=(d.aux_ld, _c0(d.aux, d.aux_ld, spans)) if d.aux else None)
    else:
        sp.update(out=(dout[1], _c0(dout[0], dout[1], spans), d.Ho, d.Wo), db=db)
    return sp


@pytest.fixture(scope='module')
def recorded():
    """every cd_conv_fwd / cd_conv_wgrad of a 32² training forward + backward at B = 32 and B = 5 whose pixel grid is at most
    8 x 8 (the 8 x 8 and 4 x 4 levels, the mid block, the 8 -> 4 downsample and the 4 -> 8 transposed convolution), deduplicated"""
    unet, _ = _unet(3, seed=11)
    gd = _gd(unet, 3)
    eng = unet.engine
    specs = {}
    for B in (32, 5):
        x, t = _batch(B, 3, 500 + B)
        unet.zero_grad(set_to_none=True)
        with _record_calls() as calls:
            gd.p_losses(x, t).backward()
            torch.cuda.synchronize()
        spans = _engine_tensors(eng)
        for name, args in calls:
            if name not in ('cd_conv_fwd', 'cd_conv_wgrad'):
                continue
            d = args[0]._obj
            if d.Hg > 8 or d.Wg > 8:
                continue
            if name == 'cd_conv_fwd':
                sp = _spec('fwd', d, args[1], spans)
            else:
                sp = _spec('wgrad', d, args[5], spans, dout=(args[1].value, args[2]), db=bool(args[4].value))
            specs.setdefault(repr(sorted(sp.items())), sp)
    yield list(specs.values())
    del unet, gd


def _shifted(x, Hg, Wg, sy, sx, dy, dx):
    """x[b, gy*sy+dy, gx*sx+dx, :] on the Hg x Wg grid, zero outside the image"""
    B, H, W, _ = x.shape
    ys = torch.arange(Hg, device=x.device) * sy + dy
    xs = torch.arange(Wg, device=x.device) * sx + dx
    my, mx = (ys >= 0) & (ys < H), (xs >= 0) & (xs < W)
    v = x[:, ys.clamp(0, H - 1)][:, :, xs.clamp(0, W - 1)]
    return v * (my[None, :, None, None] & mx[None, None, :, None])


def _region(buf, sp, c0, n):
    oys, oxs, oy0, ox0 = sp['omap']
    return buf[:, oy0:oy0 + oys * sp['Hg']:oys, ox0:ox0 + oxs * sp['Wg']:oxs, c0:c0 + n]


def _outside_untouched(buf, before, sp, c0, n):
    a, b = buf.clone(), before.clone()
    _region(a, sp, c0, n).zero_()
    _region(b, sp, c0, n).zero_()
    return bool(torch.equal(a, b))


def _gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * math.pi) ** 0.5


def _replay(sp, g):
    """-> list of (name, value, control, K) for one recorded descriptor, run on fresh TF32-rounded operands"""
    from cold_diffusion_models_b200 import ops
    B, Hg, Wg, Cout = sp['B'], sp['Hg'], sp['Wg'], sp['Cout']
    srcs, descs = [], []
    for ld, Cc, H, W, c0, taps, wpb in sp['srcs']:
        buf = tf32_rn(randn(B, H, W, ld, g=g))
        nw = B if wpb else 1
        w = tf32_rn(randn(*((nw, len(taps), Cout, Cc) if wpb else (len(taps), Cout, Cc)), g=g, scale=(Cc * len(taps)) ** -0.5))
        srcs.append((buf, c0, Cc, taps, wpb, w))
        descs.append((ops.View(buf, c0, Cc), [(0, 0, dy, dx) for dy, dx in taps], w, bool(wpb)))
    out_ld, oc0, Ho, Wo = sp['out']
    xs = [[_shifted(buf[..., c0:c0 + Cc].double(), Hg, Wg, sp['sy'], sp['sx'], dy, dx) for dy, dx in taps]
          for buf, c0, Cc, taps, wpb, w in srcs]
    res = []
    if sp['kind'] == 'fwd':
        out = randn(B, Ho, Wo, out_ld, g=g) if sp['resid'] and sp['resid'][2] else sentinel(B, Ho, Wo, out_ld)
        before = out.clone()
        bias = randn(Cout, g=g) if sp['bias'] else None
        resid = rv = None
        if sp['resid']:
            rld, rc0, alias = sp['resid']
            resid = out if alias else randn(B, Ho, Wo, rld, g=g)
            rv = ops.View(resid, rc0, Cout)
            rref = _region(resid, sp, rc0, Cout).double().clone()
        out2 = sentinel(B, Ho, Wo, sp['out2'][0]) if sp['out2'] else None
        aux = randn(B, Ho, Wo, sp['aux'][0], g=g) if sp['aux'] else None
        d = ops.make_conv_desc(descs, ops.View(out, oc0, Cout), (B, Hg, Wg), stride=sp['sy'], Cout=Cout, bias=bias, resid=rv,
                               act=sp['act'], round_tf32=bool(sp['rnd']), out_map=sp['omap'],
                               out2=ops.View(out2, sp['out2'][1], Cout) if out2 is not None else None,
                               aux=ops.View(aux, sp['aux'][1], Cout) if aux is not None else None)
        ops.conv_fwd(d, sp['impl'])
        torch.cuda.synchronize()
        acc = 0
        for (buf, c0, Cc, taps, wpb, w), xl in zip(srcs, xs):
            for j, xj in enumerate(xl):
                wj = (w[:, j] if wpb else w[j][None].expand(B, -1, -1)).double()
                acc = acc + torch.einsum('bhwc,boc->bhwo', xj, wj)
        pre = acc + (bias.double() if bias is not None else 0) + (rref if resid is not None else 0)
        if sp['act'] == ops.ACT_GELU:
            ref = F.gelu(pre)
        elif sp['act'] == ops.ACT_GELU_BWD:
            ref = pre * _gelu_grad(_region(aux, sp, sp['aux'][1], Cout).double())
        else:
            ref = pre
        got = _region(out, sp, oc0, Cout)
        wrong = ref.clone()
        wrong[-1] = ref[0]                       # control: the last image's output taken from the first image
        K = sum(len(s[3]) * s[2] for s in srcs)
        res.append(('out', rel(got, ref), rel(got, wrong), K))
        ok = _outside_untouched(out, before, sp, oc0, Cout)
        if out2 is not None:
            res.append(('out2', rel(_region(out2, sp, sp['out2'][1], Cout), pre), rel(_region(out2, sp, sp['out2'][1], Cout), ref), K))
            ok = ok and _outside_untouched(out2, torch.full_like(out2, 7.0), sp, sp['out2'][1], Cout)
        return res, ok
    (buf, c0, Cc, taps, wpb, _), = srcs
    dout = tf32_rn(randn(B, Ho, Wo, out_ld, g=g))
    dw0 = randn(*((B, len(taps), Cout, Cc) if wpb else (len(taps), Cout, Cc)), g=g)
    dw = dw0.clone()
    db0 = randn(Cout, g=g) if sp['db'] else None
    db = db0.clone() if sp['db'] else None
    d = ops.make_conv_desc([descs[0][:2] + (dw, bool(wpb))], ops.View(dout, oc0, Cout), (B, Hg, Wg), stride=sp['sy'], Cout=Cout,
                           out_map=sp['omap'])
    ops.conv_wgrad(d, ops.View(dout, oc0, Cout), dw, db, impl=sp['impl'])
    torch.cuda.synchronize()
    dy64 = _region(dout, sp, oc0, Cout).double()
    eq = 'bhwo,bhwc->boc' if wpb else 'bhwo,bhwc->oc'
    ref = torch.stack([torch.einsum(eq, dy64, xj) for xj in xs[0]], dim=1 if wpb else 0)
    short = torch.stack([torch.einsum(eq, dy64[:-1], xj[:-1]) for xj in xs[0]], dim=1 if wpb else 0)
    if wpb:
        short = torch.cat([short, torch.zeros_like(ref[-1:])])
    K = B * Hg * Wg
    res.append(('dw', rel(dw, dw0.double() + ref), rel(dw, dw0.double() + short), K))
    if db is not None:
        res.append(('db', rel(db, db0.double() + dy64.sum((0, 1, 2))), rel(db, db0.double() + dy64[:-1].sum((0, 1, 2))), K))
    return res, True


def _label(sp):
    s = '+'.join('%dx[C%d ld%d c0=%d]%s' % (len(tp), Cc, ld, c0, ' per-image' if wpb else '')
                 for ld, Cc, H, W, c0, tp, wpb in sp['srcs'])
    return '%s B%d %dx%d s%d omap%s Cout%d %s impl%d' % (sp['kind'], sp['B'], sp['Hg'], sp['Wg'], sp['sy'], sp['omap'][:2] if
                                                        sp['omap'] != (1, 1, 0, 0) else '', sp['Cout'], s, sp['impl'])


# relative error against fp64 over max(1, sqrt(K / 2304)) (fp32 accumulation error grows with the contraction length K); over
# the 210 replayed descriptors this measured at most 8.5e-6 (out), 5.3e-6 (out2), 2.2e-6 (dw) and 7.3e-8 (db)
CONV_BOUND = {'out': 1e-5, 'out2': 1e-5, 'dw': 6.5e-6, 'db': 2.2e-7}


def test_small_level_convolutions_replayed_against_fp64(recorded):
    """every convolution (forward, data gradient, weight gradient) of the 8 x 8 and 4 x 4 levels and the mid block, with the
    descriptor the engine built (channel slices, two-source concat GEMMs, bias / GELU / out2 / aux epilogues, the 4 x 4 stride-2
    downsample, the transposed-convolution parity taps, per-image weights of the attention) on TF32-rounded operands.  Control:
    the last image's reference replaced by the first image's (forward), the last image left out (weight gradient)."""
    from cold_diffusion_models_b200 import ops
    ck = Checks('small-level convolutions')
    g = gen(2024)
    seen = set()
    for sp in recorded:
        ck.require('%s: engine asked for TF32-rounded outputs' % _label(sp), not sp['rnd'])
        res, ok = _replay(sp, g)
        ck.require('%s: outside the written region untouched' % _label(sp), ok)
        for what, v, c, K in res:
            b = CONV_BOUND[what] * max(1.0, (K / 2304) ** 0.5)
            ck('%s %s' % (_label(sp), what), v, b, c)
        if sp['impl'] == ops.CONV_TC:
            nt = tuple(len(s[5]) for s in sp['srcs'])
            seen.add((sp['kind'], sp['Hg'], nt, sp['sy'], sp['omap'][0], len(sp['srcs'])))
    _METRICS['small-level convolutions::replayed'] = len(recorded)
    # what the list must contain: 3x3 at both levels, two-source [3x3 | 1x1], 1x1, the stride-2 downsample, convT parity taps
    for kind in ('fwd', 'wgrad'):
        for H in (8, 4):
            ck.require('%s 3x3 at %dx%d ran' % (kind, H, H), (kind, H, (9,), 1, 1, 1) in seen)
            ck.require('%s 1x1 at %dx%d ran' % (kind, H, H), (kind, H, (1,), 1, 1, 1) in seen)
        ck.require('%s parity taps 4 -> 8 ran' % kind, (kind, 4, (4,), 1, 2, 1) in seen)
    ck.require('fwd [3x3 | 1x1] at 8x8 and 4x4 ran', ('fwd', 8, (9, 1), 1, 1, 2) in seen and ('fwd', 4, (9, 1), 1, 1, 2) in seen)
    ck.require('fwd 4x4 stride-2 downsample ran', ('fwd', 4, (16,), 2, 1, 1) in seen)
    ck.require('wgrad 4x4 stride-2 downsample ran', ('wgrad', 4, (16,), 2, 1, 1) in seen)
    ck.done()


# ---- linear attention ---------------------------------------------------------------------------------------------------
LA_CASES = [(32, 16, 512), (32, 16, 256), (32, 64, 256), (32, 64, 128), (5, 16, 512), (5, 64, 256)]


@pytest.mark.parametrize('case', LA_CASES, ids=['B%d-n%d-dim%d' % c for c in LA_CASES])
def test_linear_attention_small_levels_against_fp64(case):
    """cd_linattn_context_det with the engine's plan (n = 16: one 64-pixel span, three quarters empty) and, at n = 64, a hand
    plan of two 32-pixel spans per image to merge; cd_linattn_weff, cd_linattn_bwd_small and cd_linattn_bwd_kv against fp64
    autograd of the attention core.  Controls: the last quarter of the pixels dropped, neighbouring images' results."""
    from cold_diffusion_models_b200 import ops
    B, n, dim = case
    ck = Checks('linattn %s' % (case,))
    scale = 32 ** -0.5
    g = gen(3000 + B + n + dim)
    qkv = randn(B, n, 384, g=g)
    qkv[..., 128:256] *= 2.0
    k64, v64 = qkv[..., 128:256].double(), qkv[..., 256:].double()
    kmax_ref = qkv[..., 128:256].max(dim=1).values
    cut = n - n // 4

    def ctx_of(k, v):
        e = torch.exp(k - k.max(1, keepdim=True).values)
        c = torch.einsum('bnc,bne->bce', e, v).reshape(-1, 4, 32, 4, 32).diagonal(dim1=1, dim2=3).permute(0, 3, 1, 2)
        return e.sum(1), c / e.sum(1).reshape(-1, 4, 32, 1)
    ksum_ref = torch.exp(k64 - kmax_ref.double()[:, None, :]).sum(1)
    _, ctxn_ref = ctx_of(k64, v64)
    _, ctxn_tail = ctx_of(k64[:, :cut], v64[:, :cut])
    plans = [('engine', ops.linattn_ctx_plan(B, n, DEV))]
    if n == 64:
        plans.append(('two spans', (2, 32)))
    ctx = ksum = kmax = None
    for tag, (nblk, ppb) in plans:
        ws = torch.empty(B, nblk, 4352, device=DEV)
        kmax, ksum, ctx = sentinel(B, 128), sentinel(B, 128), sentinel(B, 4, 32, 32)
        call('cd_linattn_context_det', ptr(qkv), 384, B, n, nblk, ppb, ptr(ws), ptr(kmax), ptr(ksum), ptr(ctx), stream())
        key = 'ctx %s (nblk %d, ppb %d)' % (tag, nblk, ppb)
        ck.require(key + ': kmax exact', bool(torch.equal(kmax, kmax_ref)))
        ck(key + ' ksum', rel(ksum, ksum_ref), 1.8e-7, rel(ksum.roll(1, 0), ksum_ref))       # measured <= 6.0e-8
        ckn = ctx.double() / ksum.double().reshape(B, 4, 32, 1)
        ck(key + ' ctx', rel(ckn, ctxn_ref), 1.4e-6, rel(ctxn_tail, ctxn_ref))               # measured <= 4.7e-7
    w_out = randn(dim, 128, g=g, scale=128 ** -0.5)
    weff = sentinel(B, dim, 128)
    call('cd_linattn_weff', ptr(ctx), ptr(ksum), ptr(w_out), B, dim, C.c_float(scale), 0, ptr(weff), stream())
    cn = ctx.double() / ksum.double().reshape(B, 4, 32, 1)
    wref = (scale * torch.einsum('che,bhde->bchd', w_out.double().reshape(dim, 4, 32), cn)).reshape(B, dim, 128)
    ck('weff', rel(weff, wref), 3.3e-7, rel(weff.roll(1, 0), wref))                           # measured <= 1.1e-7
    dweff = randn(B, dim, 128, g=g)
    kl, vl, wl = k64.clone().requires_grad_(True), v64.clone().requires_grad_(True), w_out.double().requires_grad_(True)
    wr, _ = _attn_core64(kl, vl, wl, scale)
    dk_ref, dv_ref, dw_ref = torch.autograd.grad(wr, (kl, vl, wl), dweff.double())
    dw0 = randn(dim, 128, g=g)
    dw = dw0.clone()
    dctxn, rowdot = sentinel(B, 4, 32, 32), sentinel(B, 128)
    call('cd_linattn_bwd_small', ptr(dweff), ptr(ctx), ptr(ksum), ptr(w_out), B, dim, C.c_float(scale), ptr(dw), ptr(dctxn),
         ptr(rowdot), stream())
    ck('bwd_small dw_out', rel(dw, dw0.double() + dw_ref), 8.3e-7, rel(dw_ref, dw0.double() + dw_ref))   # measured <= 2.8e-7
    for dld in (384, 392):
        dq = sentinel(B, n, dld)
        call('cd_linattn_bwd_kv', ptr(qkv), 384, B, n, ptr(kmax), ptr(ksum), ptr(dctxn), ptr(rowdot), ptr(dq), dld, stream())
        key = 'bwd_kv dld=%d' % dld
        ck(key + ' dk', rel(dq[..., 128:256], dk_ref), 1.7e-6, rel(dq[..., 128:256].roll(1, 0), dk_ref))   # measured <= 5.7e-7
        ck(key + ' dv', rel(dq[..., 256:384], dv_ref), 1.4e-6, rel(dq[..., 256:384].roll(1, 0), dv_ref))   # measured <= 4.9e-7
        ck.require(key + ': q columns and padding untouched', bool((dq[..., :128] == 7.0).all() and (dq[..., 384:] == 7.0).all()))
    ck.done()


# ---- LayerNorm and column sums ------------------------------------------------------------------------------------------
LN_CASES = [(32, 16, 512), (32, 16, 256), (32, 64, 256), (32, 64, 512), (5, 16, 512), (5, 64, 256)]


@pytest.mark.parametrize('case', LN_CASES, ids=['B%d-px%d-C%d' % c for c in LN_CASES])
def test_layernorm_small_levels_against_fp64(case):
    """cd_layernorm_fwd / cd_layernorm_bwd at npix = B * 16 and B * 64 (the small-npix kernel), with the engine's row stride and
    a padded one (ld = C + 4), with and without addend, with dg / dbeta accumulating and with both NULL"""
    B, px, Cc = case
    npix = B * px
    ck = Checks('layernorm %s' % (case,))
    g = gen(4000 + npix + Cc)
    for ld in (Cc, Cc + 4):
        xbuf = randn(npix, ld, g=g, scale=2.0) + 0.3
        xv = xbuf[:, :Cc]
        gam, bet = 1 + randn(Cc, g=g, scale=0.2), randn(Cc, g=g, scale=0.1)
        y, st = sentinel(npix, ld), sentinel(npix, 2)
        call('cd_layernorm_fwd', ptr(xbuf), ld, C.c_int64(npix), Cc, ptr(gam), ptr(bet), C.c_float(1e-5), ptr(y), ld, ptr(st), 0,
             stream())
        x64 = xv.double().t().reshape(1, Cc, npix, 1).requires_grad_(True)
        g64, b64 = gam.double().reshape(1, Cc, 1, 1), bet.double().reshape(1, Cc, 1, 1)
        y64 = UO.layer_norm(x64, g64, b64)
        yref = y64.detach().reshape(Cc, npix).t()
        var_nm1 = torch.var(x64.detach(), dim=1, unbiased=True, keepdim=True)
        ywrong = ((x64.detach() - x64.detach().mean(1, keepdim=True)) / (var_nm1 + 1e-5).sqrt() * g64 + b64).reshape(Cc, npix).t()
        ck('fwd ld%d' % ld, rel(y[:, :Cc], yref), 1.8e-7, rel(ywrong, yref))                 # measured <= 6.2e-8
        ck.require('fwd ld%d: padding untouched' % ld, bool((y[:, Cc:] == 7.0).all()))
        dy = randn(npix, ld, g=g)
        gx, = torch.autograd.grad(y64, x64, dy[:, :Cc].double().t().reshape(1, Cc, npix, 1))
        gx = gx.reshape(Cc, npix).t()
        xd = x64.detach().reshape(Cc, npix).t()
        dgr = (dy[:, :Cc].double() * ((xd - xd.mean(1, keepdim=True)) / (xd.var(1, unbiased=False, keepdim=True) + 1e-5).sqrt())).sum(0)
        dbr = dy[:, :Cc].double().sum(0)
        for with_add in (0, 1):
            for params in (1, 0):
                add = randn(npix, ld, g=g) if with_add else None
                dg0, db0 = randn(Cc, g=g), randn(Cc, g=g)
                dg, db = dg0.clone(), db0.clone()
                dh = sentinel(npix, ld)
                call('cd_layernorm_bwd', ptr(dy), ld, ptr(xbuf), ld, ptr(st), ptr(gam), C.c_int64(npix), Cc,
                     ptr(add), ld if with_add else 0, ptr(dh), ld, ptr(dg) if params else C.c_void_p(0),
                     ptr(db) if params else C.c_void_p(0), stream())
                dref = gx + (add[:, :Cc].double() if with_add else 0)
                k = 'bwd ld%d add%d params%d' % (ld, with_add, params)
                ck(k + ' dh', rel(dh[:, :Cc], dref), 2e-7, rel(dh[:, :Cc].roll(1, 0), dref))       # measured <= 6.8e-8
                ck.require(k + ': padding untouched', bool((dh[:, Cc:] == 7.0).all()))
                if params:
                    ck(k + ' dg', rel(dg, dg0.double() + dgr), 6e-7, rel(dgr, dg0.double() + dgr))          # measured <= 2.0e-7
                    ck(k + ' dbeta', rel(db, db0.double() + dbr), 5.2e-7, rel(dbr, db0.double() + dbr))     # measured <= 1.8e-7
                else:
                    ck.require(k + ': dg / dbeta untouched', bool(torch.equal(dg, dg0) and torch.equal(db, db0)))
    ck.done()


COLSUM_CASES = [(32, 16, 512), (32, 16, 1024), (32, 64, 256), (32, 64, 512), (5, 16, 256), (5, 64, 128)]


@pytest.mark.parametrize('case', COLSUM_CASES, ids=['B%d-rows%d-C%d' % c for c in COLSUM_CASES])
def test_colsum_batched_small_levels_against_fp64(case):
    """cd_colsum_batched at rows = 16 and 64 (the scalar kernel) into a slice of a wider output row that starts non-zero, as
    the engine's dcond slices are; control: the last row of every image dropped"""
    B, rows, Cc = case
    ck = Checks('colsum_batched %s' % (case,))
    g = gen(5000 + rows + Cc)
    ld = Cc + 4
    x = randn(B, rows, ld, g=g)
    out_ld, off = 3 * Cc + 12, Cc + 4
    ob0 = randn(B, out_ld, g=g)
    ob = ob0.clone()
    call('cd_colsum_batched', ptr(x), ld, B, C.c_int64(rows), Cc, C.c_void_p(ob.data_ptr() + 4 * off), out_ld, stream())
    ref = ob0[:, off:off + Cc].double() + x[..., :Cc].double().sum(1)
    ck('colsum_batched', rel(ob[:, off:off + Cc], ref), 2.6e-7,                               # measured <= 8.8e-8
       rel(ob0[:, off:off + Cc].double() + x[:, :-1, :Cc].double().sum(1), ref))
    ck.require('other columns untouched', bool(torch.equal(ob[:, :off], ob0[:, :off]) and torch.equal(ob[:, off + Cc:], ob0[:, off + Cc:])))
    ck.done()


# ==========================================================================================================================
# 3. the kernel variants that run at 32²
# ==========================================================================================================================
SMALL_LEVEL_KERNELS = ('dwconv7_tile_kernel', 'dwconv7_wgrad_kernel', 'layernorm_kernel', 'colsum_batched_kernel',
                       'conv_tc_kernel', 'conv_rows256_kernel')


def test_small_level_kernels_run_in_a_32_training_step():
    """one S² training step at B = 32 under torch.profiler: the kernels this file checks are the ones that run (names only)"""
    from torch.profiler import profile, ProfilerActivity
    unet, _ = _unet(3, seed=12)
    gd = _gd(unet, 3)
    x, t = _batch(32, 3, 700)
    gd.p_losses(x, t).backward()                   # first step outside the trace: buffers, packs, function attributes
    torch.cuda.synchronize()
    unet.zero_grad(set_to_none=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gd.p_losses(x, t).backward()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    missing = [k for k in SMALL_LEVEL_KERNELS if not any(k in n for n in names)]
    assert not missing, (missing, sorted(n for n in names if 'kernel' in n)[:60])
