"""`Unet(64, (1, 2, 4, 8))` at the 64² shape of the CelebA defading driver (train_batch_size = 100, two micro-batches, the
Incremental Gaussian fade with T = 100, kernel_std = 0.1, initial_mask = 11, the L1 loss) on the default tensor-core path, and
the defading degradation at that driver's and its sampling driver's parameters, against float64 references computed on the
GPU from oracle/.

At 64² every level pairs a plane size with a channel count no other checked size has (64² x 64, 32² x 128, 16² x 256,
8² x 512 and the mid block), and B = 100 sends the 16² and 8 x 8 convolutions to the shared-row kernels, where one 16 x 16 or
16 x 8 tile covers a whole 8 x 8 image (zero-filled halo loads, clipped TMA stores).

1. End to end (B = 100, B = 7 and B = 100 with residual=True, with_time_emb=False): parameter gradients of one micro-batch,
   input gradient, one Trainer step (Adam + EMA), graphed `sample(t=3)` and strided `sample(steps=10)` of the EMA model for
   both sampling routines, and batch independence.
2. Every convolution of a training step on grids up to 16 x 16 replayed with the engine's descriptors on TF32-rounded
   operands, and a profiler run that shows which shared-row kernels run.
3. The shared-row kernels forced onto grids narrower than one tile.
4. The memory-bound entry points at the arguments a B = 100 step passes.
5. The cumulative mask table, q_sample, the Algorithm-2 step and the 8-bit truncation at S = 64 and S = 128.

Every comparison also evaluates its metric on a deliberately wrong reference (a negative control) and asserts that it exceeds
the bound.  Every bound is at most 3x the value measured on an H100 80GB HBM3 (700 W), which is in the comment beside it.  Set
COLDDIFF_TEST_METRICS=<file> to write all values and controls as JSON.  The file runs in about 65 s on that card; its peak
device memory is 27.5 GiB."""
import contextlib
import ctypes as C
import io
import math

import pytest
import torch
import torch.nn.functional as F

import defading_oracle as FO
import strided_oracle as SO
import unet_oracle as UO
import test_unet_32_gpu as U32
from test_config3_step_gpu import (Checks, _metrics_file, _free_between_tests, _METRICS, rel, gen, randn, sentinel,  # noqa: F401
                                   engine_grads, grad_errors, stats, call, ptr, stream, maxabs, F32, _attn_core64)
from test_unet_32_gpu import _replay, _spec, _engine_tensors, _label, CONV_BOUND, tf32_rn, _dw_refs  # noqa: F401
from test_input_grad_gpu import _record_calls, _unet_ref, _engine_dx, _check_dx

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
S = 64
T = 100
LR = 2e-5                 # the driver's train_lr
DEFADE = dict(timesteps=T, kernel_std=0.1, initial_mask=11, fade_routine='Incremental', loss_type='l1')


def _v(a):
    return a.value if hasattr(a, 'value') else a


def _unet(residual=False, with_time_emb=True, seed=3):
    import cold_diffusion_models_b200 as cdm
    sd = UO.make_unet_state_dict(64, (1, 2, 4, 8), 3, seed=seed, with_time_emb=with_time_emb)
    with contextlib.redirect_stdout(io.StringIO()):
        unet = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3, with_time_emb=with_time_emb, residual=residual)
    unet.load_state_dict(sd)
    return unet.to(DEV), sd


def _gd(unet, routine='x0_step_down', size=S, **kw):
    from cold_diffusion_models_b200 import defading
    args = dict(DEFADE, **kw)
    return defading.GaussianDiffusion(unet, image_size=size, device_of_kernel='cuda', channels=3, sampling_routine=routine,
                                      **args).to(DEV)


def _oracle(net=None, routine='x0_step_down', size=S, **kw):
    args = dict(DEFADE, **kw)
    args.pop('loss_type')
    o = FO.DefadeOracle(net, image_size=size, channels=3, sampling_routine=routine, **args)
    o.fade_kernels = o.fade_kernels.to(DEV, F64)
    return o


def _xt64(o, x64, t, chunk=10, rx=None, ry=None):
    """the oracle's float64 sequential fade, `chunk` images at a time"""
    return torch.cat([o.q_sample(x64[c:c + chunk], t[c:c + chunk], None if rx is None else rx[c:c + chunk],
                                 None if ry is None else ry[c:c + chunk]) for c in range(0, x64.shape[0], chunk)])


def _fp64_net(sd, residual):
    sd64 = {k: v.detach().to(DEV, F64) for k, v in sd.items()}
    return lambda a, s: UO.unet_forward(sd64, a, s.to(a.device, F64), residual=residual)


def _batch(B, seed):
    x = torch.rand(B, 3, S, S, generator=gen(seed), device=DEV) * 2 - 1
    t = torch.randint(0, T, (B,), generator=gen(seed + 1), device=DEV)
    t[0], t[1] = 0, T - 1
    return x, t


def _groups(B):
    """reference chunks of ten images at B = 100; at B = 7 the last image alone (the half-empty two-image 8 x 8 tile)"""
    return [(i, min(i + 10, B)) for i in range(0, B, 10)] if B % 10 == 0 else [(0, 4), (4, B - 1), (B - 1, B)]


def _ref_parts(sd, xt64, t, gy, residual):
    """float64 autograd of sum_b <R(x_t_b, t_b), gy_b> over each group of images -> ([gradients by parameter name], output)"""
    leaves = {k: v.detach().to(DEV, F64).requires_grad_(True) for k, v in sd.items()}
    names = list(leaves)
    parts, ys = [], []
    for a, b in _groups(xt64.shape[0]):
        y = UO.unet_forward(leaves, xt64[a:b], t[a:b].to(F64), residual=residual)
        gr = torch.autograd.grad(y, [leaves[k] for k in names], gy[a:b], allow_unused=True)
        parts.append({k: (g if g is not None else torch.zeros_like(leaves[k])) for k, g in zip(names, gr)})
        ys.append(y.detach())
        del y, gr
    return parts, torch.cat(ys)


def _sum(parts):
    return {k: sum(p[k] for p in parts) for k in parts[0]}


def _gy(y, x):
    """upstream gradient of the L1 loss mean |x0 - y| at the engine's own output"""
    return torch.sign(y.double() - x.double()) / y.numel()


def _engine_output(unet, gd, x, t):
    """R(q_sample(x, t), t) on the training path (the forward p_losses runs)"""
    y = unet(gd.q_sample(x, t), t).detach()
    torch.cuda.synchronize()
    unet.zero_grad(set_to_none=True)
    return y


def _grad_check(ck, name, eg, ref, ctrl, bmed, bworst, nparams):
    errs = grad_errors(eg, ref)
    med, p90, worst = stats(errs)
    cmed, _, cworst = stats(grad_errors(eg, ctrl))
    _METRICS['%s::%s p90' % (ck.test, name)] = p90
    _METRICS['%s::%s worst parameters' % (ck.test, name)] = [(e, n) for e, n in errs[-5:]]
    ck.require('%s: %d parameter gradients, expected %d' % (name, len(errs), nparams), len(errs) == nparams)
    ck('%s median' % name, med, bmed, cmed)
    ck('%s worst' % name, worst, bworst, cworst)
    ck.require('%s: controls 10x past the bounds (%.3e, %.3e)' % (name, cmed, cworst), cmed > 10 * bmed and cworst > 10 * bworst)


# ==========================================================================================================================
# 1. end to end at the driver's configuration
# ==========================================================================================================================
CASES = [('b100', 100, False, True), ('b7', 7, False, True), ('b100-residual-notime', 100, True, False)]
# bounds per case, each at most 3x the value measured on the H100 (in the comment below it): x_t (max abs), fraction of L1
# signs that differ, grad median and worst, dx, step-gradient median and worst, after-step median and worst, the direct
# reconstruction (both routines), sample(t=3) and sample(steps=10) per routine
BOUNDS = {
    'b100': dict(xt=1.7e-7, flip=1.3e-4, gmed=2.8e-3, gworst=5.5e-3, dx=3.3e-3, smed=2.8e-3, sworst=5.5e-3, amed=2.8e-3,
                 aworst=6.5e-3, direct=2.4e-3, sample={'x0_step_down': 1.9e-5, 'default': 2.7e-3},
                 strided={'x0_step_down': 4.2e-4, 'default': 2.5e-3}),
    # measured 5.9e-8, 4.5e-5, 9.5e-4, 1.85e-3, 1.11e-3, 9.5e-4, 1.85e-3, 9.6e-4, 2.2e-3, 8.2e-4, 6.4e-6 / 9.2e-4, 1.40e-4 / 8.6e-4
    'b7': dict(xt=1.7e-7, flip=1.0e-4, gmed=2.6e-3, gworst=5.3e-3, dx=3.3e-3, smed=2.5e-3, sworst=5.3e-3, amed=2.9e-3,
               aworst=5.3e-3, direct=2.4e-3, sample={'x0_step_down': 1.9e-5, 'default': 2.7e-3},
               strided={'x0_step_down': 4.3e-4, 'default': 2.5e-3}),
    # measured 5.9e-8, 3.5e-5, 8.7e-4, 1.79e-3, 1.10e-3, 8.5e-4, 1.80e-3, 1.0e-3, 1.80e-3, 8.3e-4, 6.6e-6 / 9.1e-4, 1.45e-4 / 8.5e-4
    'b100-residual-notime': dict(xt=1.7e-7, flip=6.4e-4, gmed=2.2e-3, gworst=5.3e-3, dx=4.5e-4),
    # measured 5.9e-8, 2.1e-4, 7.4e-4, 1.79e-3, 1.51e-4
}


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_unet64_defading_gradients_step_and_graphed_samples(case, tmp_path):
    """parameter gradients of one micro-batch (L1, upstream sign(R(x_t) - x0) / N at the engine's output), the input gradient,
    one Trainer step (two micro-batches, Adam + EMA at the driver's lr) and the gradient at the new weights, and graphed
    sample(t=3) / strided sample(steps=10) of the EMA model for x0_step_down and default, against float64"""
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.strided import reverse_levels
    name, B, residual, with_t = case
    bd = BOUNDS[name]
    ck = Checks('unet64 defading %s' % name)
    unet, sd = _unet(residual, with_t, seed=3)
    nparams = len(sd)
    ck.require('238 parameters with the time embedding (%d)' % nparams, nparams == 238 if with_t else nparams < 238)
    gd = _gd(unet)
    o = _oracle()
    x, t = _batch(B, 40 + B)
    x2, t2 = _batch(B, 60 + B)
    xt64 = _xt64(o, x.double(), t)
    # ---- the engine's q_sample against the oracle's float64 sequential fade; control: every sample at t - 1
    xt = gd.q_sample(x, t)
    ck('q_sample x_t (max abs)', maxabs(xt, xt64), bd['xt'],
       maxabs(xt, _xt64(o, x.double(), torch.where(t > 0, t - 1, t + 1))))
    del xt
    # ---- gradients of one micro-batch; control: the last group of images left out
    y = _engine_output(unet, gd, x, t)
    gd.p_losses(x, t).backward()
    eg = engine_grads(unet)
    unet.zero_grad(set_to_none=True)
    parts, y64 = _ref_parts(sd, xt64, t, _gy(y, x), residual)
    ref_old = _sum(parts)
    s_eng, s_ref = torch.sign(y.double() - x.double()), torch.sign(y64 - x.double())
    ck('sign(y - x0) differs from fp64 (fraction)', (s_eng != s_ref).double().mean().item(), bd['flip'],
       (torch.sign(y64.roll(1, 0) - x.double()) != s_ref).double().mean().item())
    _grad_check(ck, 'grad', eg, ref_old, _sum(parts[:-1]), bd['gmed'], bd['gworst'], nparams)
    del eg, parts, y64, s_eng, s_ref
    # ---- input gradient (L2 against a fixed target); controls: one term of dx left out, images 0 and 1 swapped
    target = torch.rand(B, 3, S, S, generator=gen(77), device=DEV) * 2 - 1
    ref, dw, res, dout = _unet_ref(unet, x, target, t, residual)
    dx = _engine_dx(unet, x, target, t)
    unet.zero_grad(set_to_none=True)
    terms = {'the depthwise path': dw, 'the res_conv path': res}
    if residual:
        terms['dout'] = dout
    _check_dx(ck, 'dx', dx, ref, terms, bd['dx'], base=dout if residual else None)
    swapped = rel(dx, ref[torch.tensor([1, 0] + list(range(2, B)), device=DEV)])
    ck('dx vs images 0 and 1 swapped', 0.0, bd['dx'], swapped)
    ck.require('dx swap control %.3e not 10x past %.1e' % (swapped, bd['dx']), swapped > 10 * bd['dx'])
    del ref, dw, res, dout, dx
    if residual:                   # the residual / no-time-embedding case stops after the two gradient checks
        ck.done()
        return
    # ---- one Trainer step over the micro-batches (x, t) and (x2, t2): what the optimizer read is snapshotted
    y2 = _engine_output(unet, gd, x2, t2)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=LR, train_num_steps=10 ** 9,
                         gradient_accumulate_every=2, ema_decay=0.995, fp16=False, results_folder=str(tmp_path),
                         dataset='synthetic')
    eng = unet.engine
    ts = iter([t, t2])
    gd.forward = lambda d: gd.p_losses(d, next(ts))          # the Trainer's micro-batches with fixed per-image t
    snap, step = {}, tr.opt.step

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
    parts2, _ = _ref_parts(sd, _xt64(o, x2.double(), t2), t2, _gy(y2, x2), False)
    ref_mb2 = _sum(parts2)
    ref_step_g = {k: (ref_old[k] + ref_mb2[k]) / 2 for k in ref_old}
    ctrl = {k: ref_step_g[k] - (parts2[-1][k] + parts2[-2][k]) / 2 for k in ref_old}     # mb 2's last two groups left out
    _grad_check(ck, 'step gradient', snap['eg'], ref_step_g, ctrl, bd['smed'], bd['sworst'], nparams)
    del parts2, ref_mb2, ref_step_g, ctrl, y2
    # Adam at step 1 in float64 (the kernel's fp32 betas) on the gradient it read; control: no bias correction
    gs = snap['kw'].get('grad_scale', 1.0)
    b1, b2 = F32(0.9), F32(0.999)
    g64 = snap['g0'].double() * gs
    m64, v64 = (1 - b1) * g64, (1 - b2) * g64 * g64
    d_r = -LR / (1 - b1) * m64 / (v64.sqrt() / math.sqrt(1 - b2) + 1e-8)
    d_k = eng.flat_param.double() - snap['p0'].double()
    wrong = -LR * m64 / (v64.sqrt() + 1e-8)
    ck('Adam update (max |err| / lr)', (d_k - d_r).abs().max().item() / LR, 8.9e-3,      # measured 2.98e-3 (fp32 rounding of p)
       (wrong - d_r).abs().max().item() / LR)
    ck.require('EMA copied the new weights at step 0', bool(torch.equal(tr._ema_unet.engine.flat_param, eng.flat_param)))
    del g64, m64, v64, d_r, d_k, wrong, snap
    # ---- gradient at the new weights; control: the reference at the old weights
    tr.opt.zero_grad()
    y = _engine_output(unet, gd, x, t)
    gd.p_losses(x, t).backward()
    torch.cuda.synchronize()
    eg = engine_grads(unet)
    tr.opt.zero_grad()
    sd1 = {k: v.detach().clone() for k, v in unet.state_dict().items()}
    gy = _gy(y, x)
    ref_new = _sum(_ref_parts(sd1, xt64, t, gy, False)[0])
    ref_old = _sum(_ref_parts(sd, xt64, t, gy, False)[0])
    _grad_check(ck, 'grad after the step', eg, ref_new, ref_old, bd['amed'], bd['aworst'], nparams)
    del ref_new, ref_old, eg, sd1
    # ---- graphed samples of the EMA model: sample(t=3), and sample(steps=10) from t = T; control: x_t in place of the sample
    ema = tr.ema_model
    eeng = ema.defade_fn.engine
    net64 = _fp64_net(ema.defade_fn.state_dict(), False)
    x64 = x.double()
    ck.require('strided levels', reverse_levels(T, 10) == SO.levels(T, 10))
    for routine in ('x0_step_down', 'default'):
        ema.sampling_routine = routine
        eeng.enable_cuda_graph(True)
        try:
            with torch.no_grad():
                xt3, dr3, img3 = ema.sample(batch_size=B, faded_recon_sample=x, t=3)
                xtK, drK, imgK = ema.sample(batch_size=B, faded_recon_sample=x, t=T, steps=10)
            torch.cuda.synchronize()
        finally:
            eeng.enable_cuda_graph(False)
        os_ = _oracle(net64, routine)
        with torch.no_grad():
            r = os_.sample(B, x64, t=3)
            D = SO.defading_D(_oracle(routine=routine))
            xT = D(x64, T)
            rdK, rK = SO.reverse(net64, xT, T, 10, SO.cold_update(D, routine), B)
        ck('%s sample(t=3) x_t' % routine, maxabs(xt3, r[0]), bd['xt'], maxabs(xt3, D(x64, 2)))
        ck('%s sample(t=3) direct' % routine, rel(dr3, r[1]), bd['direct'], rel(xt3, r[1]))
        ck('%s sample(t=3)' % routine, rel(img3, r[2]), bd['sample'][routine], rel(xt3, r[2]))
        ck('%s sample(steps=10) x_T' % routine, maxabs(xtK, xT), bd['xt'], maxabs(xtK, D(x64, T - 1)))
        ck('%s sample(steps=10) direct' % routine, rel(drK, rdK), bd['direct'], rel(xtK, rdK))
        ck('%s sample(steps=10)' % routine, rel(imgK, rK), bd['strided'][routine], rel(xtK, rK))
        del r, xT, rdK, rK
    ck.done()


@pytest.mark.parametrize('B', [100, 7])
def test_unet64_batch_independence(B):
    """the gradient of the whole batch in one pass against the sum of the same engine's gradients over B one-image passes
    (other tiles, kernels and weight-gradient splits; the same arithmetic per image).  The weight gradients accumulate with
    float atomics, whose order changes from run to run, so only the median is bounded.  Control: the passes of images 3 ..
    3 + B // 10 left out (image 3 alone at B = 7)."""
    ck = Checks('unet64 batch independence B%d' % B)
    unet, _ = _unet(seed=6)
    gd = _gd(unet)
    x, t = _batch(B, 90 + B)
    unet.zero_grad(set_to_none=True)
    gd.p_losses(x, t).backward()
    whole = engine_grads(unet)
    unet.zero_grad(set_to_none=True)
    left = range(3, 3 + max(1, B // 10))
    for i in [i for i in range(B) if i not in left] + list(left):
        if i == left[0]:
            partial = engine_grads(unet)
        (gd.p_losses(x[i:i + 1], t[i:i + 1]) / B).backward()
    split = engine_grads(unet)
    unet.zero_grad(set_to_none=True)
    errs = grad_errors(split, whole)
    med, p90, worst = stats(errs)
    cmed = stats(grad_errors(partial, whole))[0]
    _METRICS['%s::grad p90' % ck.test] = p90
    _METRICS['%s::grad worst (not bounded)' % ck.test] = worst
    bmed = {100: 2.3e-3, 7: 7.6e-3}[B]          # measured 7.9e-4 / 2.57e-3 (the L1 signs of 7 images weigh more than of 100)
    ck('grad median', med, bmed, cmed)
    ck.require('control %.3e not 10x past %.1e' % (cmed, bmed), cmed > 10 * bmed)
    ck.done()


# ==========================================================================================================================
# 2. every convolution at 16² and below, replayed
# ==========================================================================================================================
@pytest.fixture(scope='module')
def recorded():
    """every cd_conv_fwd / cd_conv_wgrad of a 64² training forward + backward at B = 100 and B = 7 whose pixel grid is at most
    16 x 16 (the 16² and 8 x 8 levels, the mid block, the 16 -> 8 downsample, the 8 -> 16 transposed convolution and the
    per-image attention weights), deduplicated"""
    unet, _ = _unet(seed=11)
    gd = _gd(unet)
    eng = unet.engine
    specs = {}
    for B in (100, 7):
        x, t = _batch(B, 500 + B)
        unet.zero_grad(set_to_none=True)
        with _record_calls() as calls:
            gd.p_losses(x, t).backward()
            torch.cuda.synchronize()
        spans = _engine_tensors(eng)
        for name, args in calls:
            if name not in ('cd_conv_fwd', 'cd_conv_wgrad'):
                continue
            d = args[0]._obj
            if d.Hg > 16 or d.Wg > 16:
                continue
            if name == 'cd_conv_fwd':
                sp = _spec('fwd', d, args[1], spans)
            else:
                sp = _spec('wgrad', d, args[5], spans, dout=(args[1].value, args[2]), db=bool(args[4].value))
            specs.setdefault(repr(sorted(sp.items())), sp)
    yield list(specs.values())
    del unet, gd


def test_16_and_8_level_convolutions_replayed_against_fp64(recorded):
    """every convolution (forward, data gradient, weight gradient) of the 16² and 8 x 8 levels and the mid block, with the
    descriptor the engine built, on TF32-rounded operands; outside every written region untouched.  Controls: the last image's
    reference replaced by the first image's (forward), the last image left out (weight gradient)."""
    from cold_diffusion_models_b200 import ops
    ck = Checks('64² small-level convolutions')
    g = gen(2064)
    seen = set()
    for sp in recorded:
        ck.require('%s: engine asked for TF32-rounded outputs' % _label(sp), not sp['rnd'])
        res, ok = _replay(sp, g)
        ck.require('%s: outside the written region untouched' % _label(sp), ok)
        for what, v, c, K in res:
            b = CONV_BOUND[what] * max(1.0, (K / 2304) ** 0.5)
            ck('%s %s' % (_label(sp), what), v, b, c)
        nt = tuple(len(s[5]) for s in sp['srcs'])
        seen.add((sp['kind'], sp['B'], sp['Hg'], nt, sp['sy'], sp['omap'][0], len(sp['srcs']), sp['impl'] == ops.CONV_TC,
                  any(s[6] for s in sp['srcs'])))
    _METRICS['64² small-level convolutions::replayed'] = len(recorded)
    for B in (100, 7):
        for kind in ('fwd', 'wgrad'):
            for H in (16, 8):
                ck.require('B%d %s 3x3 at %dx%d ran' % (B, kind, H, H), (kind, B, H, (9,), 1, 1, 1, True, False) in seen)
                ck.require('B%d %s 1x1 at %dx%d ran' % (B, kind, H, H), (kind, B, H, (1,), 1, 1, 1, True, False) in seen)
            ck.require('B%d %s parity taps 8 -> 16 ran' % (B, kind), (kind, B, 8, (4,), 1, 2, 1, True, False) in seen)
            ck.require('B%d %s 16 -> 8 stride-2 downsample ran' % (B, kind), (kind, B, 8, (16,), 2, 1, 1, True, False) in seen)
        for H in (16, 8):
            ck.require('B%d fwd [3x3 | 1x1] at %dx%d ran' % (B, H, H), ('fwd', B, H, (9, 1), 1, 1, 2, True, False) in seen)
        ck.require('B%d per-image attention weights ran' % B, any(k[1] == B and k[-1] for k in seen))
    ck.done()


def _kernel_names(fn):
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events()}


# whether the 16 x 8 shared-row kernel runs on the 8 x 8 level of a B = 100 step: what the trace shows on the H100
ROWS_AT_8X8 = False


def test_shared_row_kernels_run_in_a_64_b100_step(recorded):
    """one B = 100 training step under torch.profiler runs conv_rows256_kernel; the 8 x 8 forward convolutions of that step,
    replayed alone, run conv_rows256_kernel, and conv_rows_kernel as pinned in ROWS_AT_8X8"""
    ck = Checks('64² shared-row kernels')
    unet, _ = _unet(seed=12)
    gd = _gd(unet)
    x, t = _batch(100, 700)
    gd.p_losses(x, t).backward()                   # first step outside the trace: buffers, packs, function attributes
    torch.cuda.synchronize()
    unet.zero_grad(set_to_none=True)
    names = _kernel_names(lambda: gd.p_losses(x, t).backward())
    ck.require('conv_rows256_kernel ran in the B = 100 step', any('conv_rows256_kernel' in n for n in names))
    _METRICS['64² shared-row kernels::step runs conv_rows_kernel'] = any('conv_rows_kernel' in n for n in names)
    g = gen(2065)
    at8 = [sp for sp in recorded if sp['kind'] == 'fwd' and sp['B'] == 100 and sp['Hg'] == 8]
    names8 = _kernel_names(lambda: [_replay(sp, g) for sp in at8])
    rows8, rows256_8 = any('conv_rows_kernel' in n for n in names8), any('conv_rows256_kernel' in n for n in names8)
    _METRICS['64² shared-row kernels::8x8 runs conv_rows_kernel'] = rows8
    _METRICS['64² shared-row kernels::8x8 kernels'] = sorted(n for n in names8 if 'kernel' in n)
    ck.require('conv_rows256_kernel ran on the 8 x 8 level', rows256_8)
    ck.require('conv_rows_kernel on the 8 x 8 level: %s, expected %s' % (rows8, ROWS_AT_8X8), rows8 == ROWS_AT_8X8)
    ck.done()


# ==========================================================================================================================
# 3. the shared-row kernels forced onto grids narrower than a tile
# ==========================================================================================================================
ROWS, ROWS256, PER_TAP = 1, 4, 8          # cd_conv_tc_set_halo modes: 16 x 8 tiles, 16 x 16 tiles, the per-tap kernel
GRIDS = [(100, 8, 8), (3, 8, 8), (2, 8, 12), (2, 12, 8), (2, 4, 4)]
NARROW = [(g, co, kind) for g in GRIDS for co in (512, 256, 36) for kind in ('fwd', 'dgrad', 'dgrad-resid')]
CI = 64                   # input channels of the forward; the channels of dY for the data gradient


def _gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * math.pi) ** 0.5


def _run_mode(ops, d, mode):
    from cold_diffusion_models_b200._lib import lib
    lib.cd_conv_tc_set_halo(mode)
    try:
        ops.conv_fwd(d, ops.CONV_TC)
        torch.cuda.synchronize()
    finally:
        lib.cd_conv_tc_set_halo(0)


@pytest.mark.parametrize('case', NARROW, ids=['B%d-%dx%d-Cout%d-%s' % (g + (co, k)) for g, co, k in NARROW])
def test_shared_row_kernels_on_grids_narrower_than_a_tile(case):
    """3x3 forward (bias + resid -> out2, GELU -> out) and data gradient (GELU' with aux, and with aux and resid) written into
    a channel slice of a wider row (ld = Cout + 12) of a buffer with one extra image on each side: the 16 x 16 and 16 x 8
    shared-row kernels agree bit for bit, each matches float64 (the per-tap kernel too, on power-of-two grids), and the
    padding channels and the neighbouring images stay untouched.  Control: the last image's reference taken from the first."""
    from cold_diffusion_models_b200 import ops
    (B, H, W), Co, kind = case
    ck = Checks('narrow grid %s' % (case,))
    g = gen(3000 + B + 7 * H + 13 * W + Co + len(kind))
    ld, c0 = Co + 12, 4
    fwd = kind == 'fwd'
    Cin = CI
    w = tf32_rn(randn(Co, Cin, 3, 3, g=g, scale=(Cin * 9) ** -0.5)) if fwd else tf32_rn(randn(Cin, Co, 3, 3, g=g, scale=(Cin * 9) ** -0.5))
    x = tf32_rn(randn(B, H, W, Cin, g=g))
    xc = x.permute(0, 3, 1, 2).double()
    resid = randn(B, H, W, Co, g=g) if kind != 'dgrad' else None
    aux = randn(B, H, W, Co, g=g) if not fwd else None
    bias = randn(Co, g=g) if fwd else None
    if fwd:
        taps = ops.taps_conv(3, 1)
        pw = ops.pack_weight(w, taps, round_tf32=False)
        pre = F.conv2d(xc, w.double(), bias.double(), padding=1).permute(0, 2, 3, 1) + resid.double()
        ref = F.gelu(pre)
    else:
        taps = ops.taps_conv_dgrad(3, 1)
        pw = ops.pack_weight(w, taps, mode=1, round_tf32=False)
        pre = F.conv_transpose2d(xc, w.double(), padding=1).permute(0, 2, 3, 1)
        if resid is not None:
            pre = pre + resid.double()
        ref = pre * _gelu_grad(aux.double())
    wrong = ref.clone()
    wrong[-1] = ref[0]
    K = 9 * Cin
    # K = 576 on every case: measured at most 1.28e-6 (out, all three kernels) and 7.2e-7 (out2), well inside the 1e-5 / 1.25e-5
    # of tests/test_conv_rows256_gpu.py
    bound = 3.8e-6
    modes = [ROWS256, ROWS] + ([PER_TAP] if H & (H - 1) == 0 and W & (W - 1) == 0 and Co % 64 == 0 else [])
    outs = {}
    for mode in modes:
        obuf = sentinel(B + 2, H, W, ld)
        o2buf = sentinel(B + 2, H, W, ld) if fwd else None
        d = ops.make_conv_desc([(ops.View(x), taps, pw, False)], ops.View(obuf[1:B + 1], c0, Co), (B, H, W), Cout=Co,
                               bias=bias, resid=ops.View(resid) if resid is not None else None,
                               act=ops.ACT_GELU if fwd else ops.ACT_GELU_BWD,
                               out2=ops.View(o2buf[1:B + 1], c0, Co) if fwd else None,
                               aux=ops.View(aux) if aux is not None else None)
        _run_mode(ops, d, mode)
        outs[mode] = (obuf.clone(), o2buf.clone() if fwd else None)
        tag = {ROWS256: '16x16', ROWS: '16x8', PER_TAP: 'per-tap'}[mode]
        got = obuf[1:B + 1, ..., c0:c0 + Co]
        ck('%s out' % tag, rel(got, ref), bound, rel(got, wrong))
        if fwd:
            ck('%s out2' % tag, rel(o2buf[1:B + 1, ..., c0:c0 + Co], pre), 2.2e-6, rel(o2buf[1:B + 1, ..., c0:c0 + Co], ref))
        for nm, buf in (('out', obuf), ('out2', o2buf)):
            if buf is None:
                continue
            ck.require('%s %s: neighbouring images untouched' % (tag, nm), bool((buf[0] == 7.0).all() and (buf[B + 1] == 7.0).all()))
            ck.require('%s %s: padding channels untouched' % (tag, nm),
                       bool((buf[..., :c0] == 7.0).all() and (buf[..., c0 + Co:] == 7.0).all()))
    ck.require('16 x 16 and 16 x 8 kernels agree bit for bit (out)', bool(torch.equal(outs[ROWS256][0], outs[ROWS][0])))
    if fwd:
        ck.require('16 x 16 and 16 x 8 kernels agree bit for bit (out2)', bool(torch.equal(outs[ROWS256][1], outs[ROWS][1])))
    ck.done()


# ==========================================================================================================================
# 4. memory-bound entry points at the arguments of a B = 100 step
# ==========================================================================================================================
@pytest.fixture(scope='module')
def rec64():
    """the scalar arguments of the memory-bound entry points in a 64² B = 100 training step, by entry point (deduplicated)"""
    unet, _ = _unet(seed=13)
    gd = _gd(unet)
    x, t = _batch(100, 800)
    unet.zero_grad(set_to_none=True)
    with _record_calls() as calls:
        gd.p_losses(x, t).backward()
        torch.cuda.synchronize()
    pick = {'cd_dwconv7_fwd': (1, 2, 3, 4, 5), 'cd_dwconv7_wgrad': (1, 4, 5, 6, 7), 'cd_layernorm_fwd': (1, 2, 3),
            'cd_layernorm_bwd': (1, 6, 7), 'cd_linattn_context_det': (2, 3, 4, 5), 'cd_linattn_weff': (3, 4),
            'cd_linattn_bwd_small': (4, 5), 'cd_linattn_bwd_kv': (2, 3, 9), 'cd_colsum_batched': (1, 2, 3, 4),
            'cd_small_gemm': (1, 2, 4, 5, 7, 8, 9, 10, 11)}
    out = {k: set() for k in pick}
    for name, args in calls:
        if name in pick:
            out[name].add(tuple(int(_v(args[i])) for i in pick[name]))
    _METRICS['64² B100 entry points'] = {k: sorted(v) for k, v in out.items()}
    yield out
    del unet, gd


def _each(ck, what, cases, fn):
    """run a checking function of tests/test_unet_32_gpu.py on every case; collect its failures"""
    for c in cases:
        try:
            fn(c)
        except AssertionError as e:
            ck.require('%s %s: %s' % (what, c, e), False)


def test_depthwise_at_the_b100_arguments(rec64):
    """cd_dwconv7_fwd / _wgrad at every recorded (B, H, W, C, ld): the tile kernel at 8 x 8 x 512, the TMA kernels at 16² to
    64² (checks and controls of test_unet_32_gpu.py)"""
    ck = Checks('64² depthwise')
    fw = rec64['cd_dwconv7_fwd']
    wg = {a[1:] for a in rec64['cd_dwconv7_wgrad']}
    ck.require('the four levels recorded at B = 100: %s' % sorted(fw), {(H, Cc) for _, B, H, _, Cc in fw if B == 100} >=
               {(64, 64), (32, 128), (16, 256), (8, 512)})
    ck.require('the weight gradient at the forward arguments (but the 3-channel input block, whose forward is fused)',
               {(B, H, W, Cc) for _, B, H, W, Cc in fw} >= {k for k in wg if k[3] != 3})
    _each(ck, 'dwconv7', sorted({(B, H, Cc, ld) for ld, B, H, W, Cc in fw if H == W}), U32.test_depthwise_small_levels_against_fp64)
    ck.done()


def test_layernorm_at_the_b100_arguments(rec64):
    """cd_layernorm_fwd / _bwd at every recorded npix and C of the 16² and 8 x 8 levels (the multi-pixel kernel at npix =
    6400, C = 512), with the engine's row stride and a padded one (checks and controls of test_unet_32_gpu.py, whose bounds hold
    for up to 256 pixels per image; the larger planes are checked at 128² by test_config3_step_gpu.py)"""
    ck = Checks('64² layernorm')
    fw = rec64['cd_layernorm_fwd']
    ck.require('npix = 6400 at C = 512 recorded: %s' % sorted(fw), any(n == 6400 and Cc == 512 for _, n, Cc in fw))
    ck.require('row stride = C', all(ld == Cc for ld, _, Cc in fw))
    _each(ck, 'layernorm', sorted({(100, n // 100, Cc) for _, n, Cc in fw if n <= 100 * 256}),
          U32.test_layernorm_small_levels_against_fp64)
    ck.done()


def test_linear_attention_at_the_b100_arguments(rec64):
    """cd_linattn_context_det with the engine's plan at every recorded n (kmax exact; control: the last span's pixels dropped),
    then cd_linattn_weff, _bwd_small and _bwd_kv at n = 64 and 256 (checks and controls of test_unet_32_gpu.py)"""
    from cold_diffusion_models_b200 import ops
    ck = Checks('64² linear attention')
    ctx_calls = rec64['cd_linattn_context_det']
    ck.require('n = 64, 256, 1024 and 4096 at B = 100: %s' % sorted(ctx_calls), {n for B, n, _, _ in ctx_calls if B == 100} ==
               {64, 256, 1024, 4096})
    for B, n, nblk, ppb in sorted(ctx_calls):
        ck.require('n %d: the engine passed its plan' % n, (nblk, ppb) == ops.linattn_ctx_plan(B, n, DEV))
        g = gen(6000 + n)
        qkv = randn(B, n, 384, g=g)
        qkv[..., 128:256] *= 2.0
        k64, v64 = qkv[..., 128:256].double(), qkv[..., 256:].double()

        def ctxn(k, v):
            e = torch.exp(k - k.max(1, keepdim=True).values)
            c = torch.einsum('bnc,bne->bce', e, v).reshape(-1, 4, 32, 4, 32).diagonal(dim1=1, dim2=3).permute(0, 3, 1, 2)
            return c / e.sum(1).reshape(-1, 4, 32, 1)
        ws = torch.empty(B, nblk, 4352, device=DEV)
        kmax, ksum, ctx = sentinel(B, 128), sentinel(B, 128), sentinel(B, 4, 32, 32)
        call('cd_linattn_context_det', ptr(qkv), 384, B, n, nblk, ppb, ptr(ws), ptr(kmax), ptr(ksum), ptr(ctx), stream())
        key = 'ctx n%d (nblk %d, ppb %d)' % (n, nblk, ppb)
        ck.require(key + ': kmax exact', bool(torch.equal(kmax, qkv[..., 128:256].max(dim=1).values)))
        ksum_ref = torch.exp(k64 - kmax.double()[:, None, :]).sum(1)
        cut = (nblk - 1) * ppb if nblk > 1 else n - n // 4       # one span (n = 64): its last quarter dropped
        # ksum measured <= 8.6e-8; ctx 4.6e-7 / 6.3e-7 / 2.41e-6 / 9.35e-6 at n = 64 / 256 / 1024 / 4096: the error of the fp32
        # sums grows with the span length (64 / 96 / 352 / 1376 pixels), as test_config3_step_gpu.py measured at 1376 pixels
        ck(key + ' ksum', rel(ksum, ksum_ref), 2.5e-7, rel(torch.exp(k64[:, :cut] - kmax.double()[:, None, :]).sum(1), ksum_ref))
        ref = ctxn(k64, v64)
        ck(key + ' ctx', rel(ctx.double() / ksum.double().reshape(B, 4, 32, 1), ref),
           {64: 1.38e-6, 256: 1.9e-6, 1024: 7.2e-6, 4096: 2.8e-5}[n],
           rel(ctxn(k64[:, :cut], v64[:, :cut]), ref))
    dims = sorted(rec64['cd_linattn_weff'])
    ck.require('weff at B = 100 for dim 64 .. 512: %s' % dims, {d for B, d in dims if B == 100} == {64, 128, 256, 512})
    nd = {4096: 64, 1024: 128, 256: 256, 64: 512}
    # weff and the backward kernels with the bounds of test_unet_32_gpu.py, which hold for the short spans of the 16² and 8 x 8
    # levels; the 32² and 64² levels' spans are as long as config 3's, checked by test_config3_step_gpu.py
    _each(ck, 'linattn', sorted({(B, n, nd[n]) for B, n, _, _ in ctx_calls if n <= 256}),
          U32.test_linear_attention_small_levels_against_fp64)
    ck.done()


def test_column_sums_and_time_mlp_gemms_at_the_b100_arguments(rec64):
    """cd_colsum_batched at every recorded (B, rows, C) with rows <= 256 (the 16² and 8 x 8 levels; checks of
    test_unet_32_gpu.py) and
    cd_small_gemm at every product the time-MLP backward issues at B = 100.  Controls: the last K/8 of the contraction
    missing, and (accumulating calls) the accumulation dropped."""
    ck = Checks('64² colsum and small_gemm')
    cs = rec64['cd_colsum_batched']
    ck.require('rows 64 and 256 at B = 100: %s' % sorted(cs), {r for _, B, r, _ in cs if B == 100} >= {64, 256})
    _each(ck, 'colsum_batched', sorted({(B, r, Cc) for _, B, r, Cc in cs if r <= 256}),
          U32.test_colsum_batched_small_levels_against_fp64)
    g = gen(830)
    gm = sorted(rec64['cd_small_gemm'])
    ck.require('small_gemm products with K or M = 100 recorded: %s' % gm, any(100 in (M, K) for *_, M, N, K, acc in gm))
    for lda, ta, ldb, tb, ldc, M, N, K, acc in gm:
        Ab = randn(K if ta else M, lda, g=g)
        Bb = randn(N if tb else K, ldb, g=g)
        A = (Ab[:, :M].t() if ta else Ab[:, :K]).double()
        Bm = (Bb[:, :K].t() if tb else Bb[:, :N]).double()
        c0 = randn(M, ldc, g=g)
        cm = c0.clone()
        call('cd_small_gemm', ptr(Ab), lda, ta, ptr(Bb), ldb, tb, ptr(cm), ldc, M, N, K, acc, stream())
        base = c0[:, :N].double() if acc else 0
        ref = A @ Bm + base
        ks = K - max(1, K // 8)
        key = 'small_gemm ta%d tb%d M%d N%d K%d acc%d' % (ta, tb, M, N, K, acc)
        bound = {4676: 1.1e-6, 100: 5.5e-7, 64: 4.4e-7}[K]     # measured 3.8e-7 (K = 4676), <= 1.84e-7 (K = 100), 1.46e-7 (K = 64)
        ck(key, rel(cm[:, :N], ref), bound, rel(A[:, :ks] @ Bm[:ks] + base, ref))
        if acc:
            ck(key + ' (control: accumulation dropped)', rel(cm[:, :N], ref), bound, rel(A @ Bm, ref))
        ck.require(key + ': columns beyond N untouched', bool(torch.equal(cm[:, N:], c0[:, N:])))
    ck.done()


# ==========================================================================================================================
# 5. the defading degradation at the drivers' parameters
# ==========================================================================================================================
MASK_CASES = [('train-64', 64, 0.1, 11), ('sample-128', 128, 0.2, 1)]


def _quant_cpu(o, v):
    """the oracle's 8-bit truncation on the CPU (its division by 255 rounds as the kernel's does)"""
    return o._quant(v.cpu())


@pytest.mark.parametrize('case', MASK_CASES, ids=[c[0] for c in MASK_CASES])
def test_defading_masks_q_sample_and_step_down_against_fp64(case):
    """the cumulative mask table (fp32 cumprod) against the float64 product of the oracle's kernels, relative to each level's
    largest mask value; q_sample at every t in 0..99 (B = 100, per-sample t) against the oracle's sequential fade, also with
    discrete=True (bit for bit against the oracle's truncation of the kernel's fp32 value, within one level of the float64
    path) and, at S = 64, with the Random_Incremental windows; cd_mask_step_down for every (hi, lo) of the full loop and of
    reverse_levels(100, 10).  Controls: the mask at t - 1, the windows of another sample, the mask at lo - 1."""
    from cold_diffusion_models_b200.strided import reverse_levels
    name, Sz, kstd, init = case
    ck = Checks('defading masks %s' % name)
    kw = dict(kernel_std=kstd, initial_mask=init)
    gd = _gd(None, size=Sz, **kw)
    o = _oracle(size=Sz, **kw)
    cum64 = torch.cumprod(o.fade_kernels, 0)
    cum = gd._masks_cum
    scale = cum64.flatten(1).abs().max(1).values
    err = ((cum.double() - cum64).flatten(1).abs().max(1).values / scale)
    shifted = ((cum[1:].double() - cum64[:-1]).flatten(1).abs().max(1).values / scale[:-1])
    _METRICS['defading masks %s::table error by level (every 10th)' % name] = err[::10].tolist()
    _METRICS['defading masks %s::largest mask value by level (every 10th)' % name] = scale[::10].tolist()
    ck('masks_cum (max abs / largest value, worst level)', err.max().item(), 9e-8, shifted.max().item())      # measured 3.0e-8
    B = 100
    g = gen(9000 + Sz)
    x = torch.rand(B, 3, Sz, Sz, generator=g, device=DEV) * 2 - 1
    t = torch.randperm(T, generator=g, device=DEV)
    x64 = x.double()
    ref = _xt64(o, x64, t)
    t_lo = torch.where(t > 0, t - 1, t + 1)
    out = gd.q_sample(x, t)
    ck('q_sample every t (max abs)', maxabs(out, ref), 1.75e-7, maxabs(out, _xt64(o, x64, t_lo)))     # measured 5.9e-8
    # discrete: the fp32 value the kernel forms is x * masks_cum[t_b], one rounding
    gdq = _gd(None, size=Sz, discrete=True, **kw)
    q = gdq.q_sample(x, t)
    v32 = x * cum[t][:, None]
    ck.require('discrete: bit for bit the truncation of x * masks_cum[t]', bool(torch.equal(q.cpu(), _quant_cpu(o, v32))))
    q64 = _quant_cpu(o, ref).to(DEV)          # the float64 path, truncated
    dq = (q - q64).abs()
    ck('discrete: max abs from the float64 path', dq.max().item(), 2 / 255 + 1e-6)
    # measured 8.1e-7 (S = 64: one pixel of 1.2 M) and 2.2e-6 (S = 128: 11 of 4.9 M)
    ck('discrete: fraction of pixels off the float64 path', (dq > 1e-6).double().mean().item(), {64: 2.4e-6, 128: 6.7e-6}[Sz],
       ((_quant_cpu(o, _xt64(o, x64, t_lo)).to(DEV) - q64).abs() > 1e-6).double().mean().item())
    del gdq, q, v32, q64, dq
    if Sz == 64:
        gr = _gd(None, size=Sz, fade_routine='Random_Incremental', **kw)
        orr = _oracle(size=Sz, fade_routine='Random_Incremental', **kw)
        rx = torch.randint(0, Sz + 1, (B,), generator=g, device=DEV)
        ry = torch.randint(0, Sz + 1, (B,), generator=g, device=DEV)
        outr = gr.q_sample(x, t, _offsets=(rx, ry))
        refr = _xt64(orr, x64, t, rx=rx, ry=ry)
        ck('Random_Incremental q_sample (max abs)', maxabs(outr, refr), 1.7e-7,          # measured 5.8e-8
           maxabs(outr, _xt64(orr, x64, t, rx=rx.roll(1), ry=ry.roll(1))))
        del gr, orr, outr, refr
    # Algorithm 2: x_lo = x_hi - D(xhat, hi) + D(xhat, lo) with D(x, n) = x * prod_{i < n} K_i
    Bs = 4
    xt = torch.rand(Bs, 3, Sz, Sz, generator=g, device=DEV) * 2 - 1
    xh = torch.rand(Bs, 3, Sz, Sz, generator=g, device=DEV) * 2 - 1

    def D(v, n):
        return v if n <= 0 else v * cum64[n - 1]
    pairs = sorted(set(zip(range(T, 0, -1), range(T - 1, -1, -1))) | set(zip(reverse_levels(T, 10), reverse_levels(T, 10)[1:])))
    worst = ctrl = 0.0
    o_ = torch.empty_like(xt)
    for hi, lo in pairs:
        call('cd_mask_step_down', ptr(xt), ptr(xh), ptr(o_), ptr(cum), hi - 1, lo - 1, C.c_void_p(0), C.c_void_p(0), Bs, 3, Sz,
             Sz, stream())
        r = xt.double() - D(xh.double(), hi) + D(xh.double(), lo)
        worst = max(worst, maxabs(o_, r))
        if lo >= 1:
            ctrl = max(ctrl, maxabs(o_, xt.double() - D(xh.double(), hi) + D(xh.double(), lo - 1)))
    _METRICS['defading masks %s::step_down pairs' % name] = len(pairs)
    ck('mask_step_down, every (hi, lo) (max abs)', worst, 4.2e-7, ctrl)             # measured 1.4e-7
    ck.done()
