"""Images above 128²: the row-strip blur kernels (cd_blur_apply / cd_blur_step_down for 128 < S <= 512), the deblurring and
resolution packages at 256², and the Unet `Unet(64, (1, 2, 4, 8))` at 256² (gradients, one optimizer
step, a CUDA-graph sample) and at 512² (a forward), and the snow and decolorization packages at 256², against float64 references computed on the GPU from
oracle/.

As in tests/test_config3_step_gpu.py, every comparison also evaluates its metric on a deliberately wrong reference (a
negative control) and asserts that it exceeds the bound.  Every bound is at most 3x the value measured on an H100 80GB HBM3
(700 W), which is in the comment beside it.  Set COLDDIFF_TEST_METRICS=<file> to write all values and controls as JSON.
The file runs in about 35 s on that card; its peak device memory is 8.2 GB."""
import contextlib
import io

import pytest
import torch
from torch import nn

import deblur_oracle as DO
import resolution_oracle as RO
import unet_oracle as UO
from test_config3_step_gpu import (Checks, _metrics_file, _free_between_tests, rel, maxabs, call, ptr, stream, gen,  # noqa: F401
                                   sentinel, quantize, blur_per_image, ref_step, engine_grads, grad_errors, stats)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64


def oracle(S, routine, k, std, T, denoise_fn=None, **kw):
    o = DO.DeblurOracle(denoise_fn, image_size=S, channels=3, timesteps=T, kernel_std=std, kernel_size=k, blur_routine=routine,
                        **kw)
    o.kernels2d = [kk.double().cuda() for kk in o.kernels2d]
    return o


class Toy(nn.Module):
    """a fixed restoration "network" for the package tests: x0_hat = 0.8 x + 0.01 t (the degradation paths, not the Unet)"""

    def forward(self, x, t):
        return 0.8 * x + 0.01 * t.to(x.device, x.dtype).reshape(-1, 1, 1, 1)


# ==========================================================================================================================
# the strip kernels
# ==========================================================================================================================
@pytest.mark.parametrize('S', [256, 384, 512])
@pytest.mark.parametrize('routine,k,std', [('Exponential_reflect', 27, 0.1), ('Incremental', 27, 0.5)])
def test_strip_kernels_against_chained_fp64_convolutions(S, routine, k, std):
    """q_sample with per-sample t (incl. -1 and T-1), `discrete` collapse, 8-bit truncation, and Algorithm 2 against the
    reference's chained k = 27 convolutions in fp64"""
    from cold_diffusion_models_b200.degradation import build_blur_operators
    ck = Checks('strip[%d,%s]' % (S, routine))
    T, B = 12, 4
    o = oracle(S, routine, k, std, T)
    ops = build_blur_operators(routine, T, k, std, S)[0].to(DEV)
    g = gen(S + k)
    x = torch.rand(B, 3, S, S, generator=g, device=DEV) * 2 - 1
    x64 = x.double()
    t = torch.tensor([-1, 0, 5, T - 1], device=DEV)
    ref = blur_per_image(o, x64, t)
    ref_shift = blur_per_image(o, x64, torch.where(t < T - 1, t + 1, t - 1))        # control: every step index off by one
    ref_col = ref.clone()
    ref_col[3] = ref[3].mean(dim=(1, 2), keepdim=True).expand_as(ref[3])
    for collapse in (0, 1):
        r = ref_col if collapse else ref
        for quant in (0, 1):
            out = sentinel(B, 3, S, S)
            call('cd_blur_apply', ptr(x), ptr(out), ptr(ops), ptr(t), 0, B, 3, S, T, collapse, quant, stream())
            if quant:
                d = (out.double() - quantize(r)).abs()
                ck('q_sample c%d q1 max' % collapse, d.max().item(), 2 / 255 + 1e-6)
                ck('q_sample c%d q1 flipped fraction' % collapse, (d > 1e-6).double().mean().item(), 1.1e-5,   # measured <= 3.8e-6
                   ((quantize(ref_shift) - quantize(r)).abs() > 1e-6).double().mean().item())
            else:
                # control 2: the output shifted by one row (a strip written one row off)
                ck('q_sample c%d' % collapse, maxabs(out, r), 4.5e-7, maxabs(ref_shift, r))                  # measured <= 1.6e-7
                ck('q_sample c%d row shift' % collapse, maxabs(out, r), 4.5e-7, maxabs(out[:3].roll(1, 2), r[:3]))
    xt = torch.rand(B, 3, S, S, generator=g, device=DEV) * 2 - 1
    for hi in (T - 1, 0):
        d_hi = blur_per_image(o, x64, torch.full((B,), hi))
        d_lo = blur_per_image(o, x64, torch.full((B,), hi - 1))
        for collapse in ((0, 1) if hi == T - 1 else (0,)):
            dh = d_hi.mean(dim=(2, 3), keepdim=True).expand_as(d_hi) if collapse else d_hi
            r = xt.double() - dh + d_lo
            out = sentinel(B, 3, S, S)
            call('cd_blur_step_down', ptr(xt), ptr(x), ptr(out), ptr(ops), hi, hi - 1, B, 3, S, T, collapse, stream())
            wrong = xt.double() - d_lo + blur_per_image(o, x64, torch.full((B,), hi - 2)) if hi > 0 else xt.double()
            ck('step_down hi=%d c%d' % (hi, collapse), maxabs(out, r), 6.5e-7, maxabs(wrong, r))       # measured <= 2.3e-7
    ck.done()


# ==========================================================================================================================
# the packages at 256²
# ==========================================================================================================================
@pytest.mark.parametrize('routine,sampling,discrete', [('Exponential_reflect', 'x0_step_down', False),
                                                       ('Exponential_reflect', 'default', False),
                                                       ('Exponential_reflect', 'x0_step_down', True),
                                                       ('Exponential_reflect', 'default', True),
                                                       ('Individual_Incremental', 'default', False)])
def test_deblurring_package_at_256(routine, sampling, discrete):
    """q_sample, a 4-step sample in both routines, `discrete`, Individual_Incremental and sample_from_blur(start > 0)"""
    import cold_diffusion_models_b200 as cdm
    ck = Checks('deblur256[%s,%s,%d]' % (routine, sampling, discrete))
    S, T, B = 256, 10, 3
    kw = dict(image_size=S, channels=3, timesteps=T, kernel_std=0.1, kernel_size=11, blur_routine=routine,
              sampling_routine=sampling, discrete=discrete)
    gd = cdm.GaussianDiffusion(Toy(), device_of_kernel='cuda', loss_type='l1', **kw).to(DEV)
    o = DO.DeblurOracle(Toy(), **kw)
    o.kernels2d = [kk.double().cuda() for kk in o.kernels2d]
    g = gen(7)
    x = torch.rand(B, 3, S, S, generator=g, device=DEV) * 2 - 1
    t = torch.tensor([0, 4, T - 1], device=DEV)
    if routine != 'Individual_Incremental':
        q = gd.q_sample(x, t)
        r = o.q_sample(x.double(), t)
        if discrete:                              # 8-bit truncation: a few pixels may flip by one level at fp32 level
            ck('q_sample flipped fraction', ((q.double() - r).abs() > 1e-6).double().mean().item(), 1e-6,    # measured 0
               ((o.q_sample(x.double(), t.flip(0)) - r).abs() > 1e-6).double().mean().item())
        else:
            ck('q_sample', rel(q, r), 3e-7, rel(o.q_sample(x.double(), (t + 1).clamp(max=T - 1)), r))     # measured 1.0e-7
    tt = 4
    got = gd.sample(batch_size=B, img=x, t=tt)
    want = o.sample(B, x.double(), t=tt)
    wrong = o.sample(B, x.double(), t=tt - 1)
    # measured: x_t <= 1.4e-7, direct <= 1.3e-7, sample <= 2.9e-7 (3.2e-6 with `discrete` in x0_step_down, where x_t is a
    # plane mean and Algorithm 2 subtracts two nearly equal blurred images)
    bounds = dict(x_t=4.2e-7, direct=3.9e-7, sample=9.6e-6 if discrete and sampling == 'x0_step_down' else 8.7e-7)
    for name, a, b, w in zip(('x_t', 'direct', 'sample'), got, want, wrong):
        ck('sample %s' % name, rel(a, b), bounds[name], rel(w, b))
    if routine != 'Individual_Incremental' and not discrete:
        # sample_from_blur(start > 0): x_t is the image blurred by the steps start .. t-1 only (the one-entry range operator)
        got = gd.sample_from_blur(batch_size=B, img=x, t=tt, start=2)
        h = x.double()
        for i in range(2, tt):
            h = o.blur_step(i, h)
        ck('sample_from_blur x_t', rel(got[0], h), 3.5e-7, rel(o.blur_step(1, h), h))          # measured 1.2e-7
    ck.done()


def test_resolution_package_at_256():
    from cold_diffusion_models_b200.resolution_diffusion_pytorch import GaussianDiffusion as RSGD
    ck = Checks('resolution256')
    S, T, B = 256, 6, 3
    gd = RSGD(Toy(), image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1',
              resolution_routine='Incremental', sampling_routine='x0_step_down').to(DEV)
    o = RO.ResolutionOracle(Toy(), image_size=S, channels=3, timesteps=T, resolution_routine='Incremental',
                            sampling_routine='x0_step_down')
    x = torch.rand(B, 3, S, S, generator=gen(9), device=DEV) * 2 - 1
    t = torch.tensor([0, 3, T - 1], device=DEV)
    r = o.q_sample(x.double(), t)
    ck('q_sample', rel(gd.q_sample(x, t), r), 2e-7, rel(o.q_sample(x.double(), (t + 1).clamp(max=T - 1)), r))   # measured 6.9e-8
    ck('func[2]', rel(gd.func[2](x), o.func(2, x.double())), 1.8e-7,                     # measured 6.2e-8
       rel(o.func(3, x.double()), o.func(2, x.double())))
    got = gd.sample(batch_size=B, img=x, t=4)
    want = o.sample(B, x.double(), t=4)
    wrong = o.sample(B, x.double(), t=3)
    bounds = dict(x_t=2.6e-7, direct=2.9e-7, sample=4.7e-7)          # measured 8.9e-8, 9.9e-8, 1.6e-7
    for name, a, b, w in zip(('x_t', 'direct', 'sample'), got, want, wrong):
        ck('sample %s' % name, rel(a, b), bounds[name], rel(w, b))
    ck.done()


# ==========================================================================================================================
# the Unet at 256² and 512²
# ==========================================================================================================================
def _unet(seed=3):
    import cold_diffusion_models_b200 as cdm
    with contextlib.redirect_stdout(io.StringIO()):
        unet = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).to(DEV)
        sd = UO.make_unet_state_dict(64, (1, 2, 4, 8), 3, seed=seed)
        unet.load_state_dict(sd)
    return unet, sd


def test_unet_256_gradients_step_and_graphed_sample(tmp_path):
    import cold_diffusion_models_b200 as cdm
    ck = Checks('unet256')
    S, T, B = 256, 20, 2
    unet, sd = _unet()
    kw = dict(image_size=S, channels=3, timesteps=T, kernel_std=0.1, kernel_size=11, blur_routine='Exponential_reflect')
    gd = cdm.GaussianDiffusion(unet, device_of_kernel='cuda', loss_type='l2', sampling_routine='x0_step_down', **kw).to(DEV)
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(B, 3, S, S, generator=g) * 2 - 1).to(DEV)
    t = torch.tensor([3, T - 1], device=DEV)
    o = oracle(S, 'Exponential_reflect', 11, 0.1, T)
    xt64 = blur_per_image(o, x.double(), t)
    # gradients of one micro-batch against fp64 autograd through oracle/unet_oracle.py
    unet.zero_grad(set_to_none=True)
    gd.p_losses(x, t).backward()
    eg = engine_grads(unet)
    # the reference per image; the control leaves the second image out
    g0, _, _ = ref_step(sd, x[:1], xt64[:1], t[:1], norm=x.numel(), chunk=1)
    g1, _, _ = ref_step(sd, x[1:], xt64[1:], t[1:], norm=x.numel(), chunk=1)
    ref_g = {k: g0[k] + g1[k] for k in g0}
    med, p90, worst = stats(grad_errors(eg, ref_g))
    cmed, _, cworst = stats(grad_errors(eg, g0))
    ck('grad median', med, 3.3e-3, cmed)                  # measured 1.1e-3
    ck('grad worst', worst, 6.3e-3, cworst)               # measured 2.1e-3
    del ref_g, g0, g1
    # one optimizer step through the Trainer, then the graphed 3-step sample of the EMA model
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=1e-3, train_num_steps=10 ** 9,
                         gradient_accumulate_every=1, ema_decay=0.995, fp16=False, results_folder=str(tmp_path),
                         dataset='synthetic')
    before = {k: v.detach().clone() for k, v in unet.state_dict().items()}
    loss = tr.train_step([x]).item()
    ck.require('train_step loss finite', loss == loss and abs(loss) < 1e3)
    moved = max((unet.state_dict()[k].double() - before[k].double()).abs().max().item() for k in before)
    ck.require('train_step moved the weights (%.3e)' % moved, 1e-5 < moved < 1e-2)
    ema = tr.ema_model
    eng = ema.denoise_fn.engine
    eng.enable_cuda_graph(True)
    try:
        with torch.no_grad():
            xt, dr, img = ema.sample(batch_size=B, img=x, t=3)
        torch.cuda.synchronize()
    finally:
        eng.enable_cuda_graph(False)
    esd = {k: v.detach().to(DEV, F64) for k, v in ema.denoise_fn.state_dict().items()}
    fn = lambda a, s: UO.unet_forward(esd, a, s.to(a.device, F64))
    os_ = oracle(S, 'Exponential_reflect', 11, 0.1, T, denoise_fn=fn, sampling_routine='x0_step_down')
    r = os_.sample(B, x.double(), t=3)
    ck('graphed sample x_t', rel(xt, r[0]), 3.7e-7,               # measured 1.3e-7
       rel(xt, blur_per_image(o, x.double(), torch.full((B,), 1))))
    ck('graphed sample direct', rel(dr, r[1]), 4.3e-4, rel(dr.roll(1, 0), r[1]))   # measured 1.4e-4
    ck('graphed sample', rel(img, r[2]), 9.2e-4, rel(xt, r[2]))                 # measured 3.1e-4
    ck.done()


def test_unet_512_forward():
    ck = Checks('unet512')
    unet, sd = _unet(seed=4)
    x = torch.rand(1, 3, 512, 512, generator=gen(11), device=DEV) * 2 - 1
    t = torch.tensor([7], device=DEV)
    with torch.no_grad():
        y = unet(x, t)
        ref = UO.unet_forward({k: v.to(DEV, F64) for k, v in sd.items()}, x.double(), t.double())
        wrong = UO.unet_forward({k: v.to(DEV, F64) for k, v in sd.items()}, x.double(), t.double() + 1)
    ck('forward', rel(y, ref), 1.5e-3, rel(wrong, ref))                  # measured 5.1e-4
    ck.done()


# ==========================================================================================================================
# snow / decolor at 256² (the packages whose reference drivers take --resolution)
# ==========================================================================================================================
def _snow_package(kind, S, T, tmp_path, **kw):
    from cold_diffusion_models_b200.snowification_diffusion import GaussianDiffusion as SNGD
    with contextlib.redirect_stdout(io.StringIO()):
        return SNGD(Toy(), image_size=(S, S) if kind == 'Snow' else S, device_of_kernel='cuda', channels=3, timesteps=T,
                    loss_type='l1', forward_process_type=kind, train_routine='Final', sampling_routine='x0_step_down',
                    results_folder=str(tmp_path), **kw).to(DEV)


def test_snow_at_256(tmp_path):
    """Snow: the layers generated on the device (cd_snow_layers) against oracle/snow_oracle.py's host restatement of the
    reference generator (fixed seed 123321), then q_sample (per-sample t incl. -1) and one x0_step_down step (cd_snow)
    against SnowOracle in fp64 on those reference layers"""
    import snow_oracle as SO
    ck = Checks('snow256')
    S, T, B = 256, 8, 3
    gd = _snow_package('Snow', S, T, tmp_path, snow_level=1)
    layers = gd.forward_process.layers(DEV)
    ref_layers, br = SO.generate_snow_layers((S, S), snow_level=1, num_timesteps=T)
    ref_layers = ref_layers.to(DEV, F64)
    ck('layers', maxabs(layers, ref_layers), 1e-7, maxabs(layers[1:], ref_layers[:-1]))       # measured 0
    o = SO.SnowOracle(Toy(), SO.SnowFP(ref_layers, br), timesteps=T, sampling_routine='x0_step_down')
    x = torch.rand(B, 3, S, S, generator=gen(13), device=DEV) * 2 - 1
    for t in (torch.tensor([0, 3, T - 1], device=DEV), torch.tensor([2, -1, 5], device=DEV)):
        r = o.q_sample(x.double(), t)
        ck('q_sample t=%s' % t.tolist(), rel(gd.q_sample(x, t), r), 1.6e-7,                   # measured <= 5.5e-8
           rel(o.q_sample(x.double(), (t + 1).clamp(max=T - 1)), r))
    t = torch.tensor([1, 4, T - 1], device=DEV)
    img = gd.q_sample(x, t)
    got, _ = gd.sample_one_step(img, t)
    want, _ = o.sample_one_step(img.double(), t)
    ck('x0_step_down step', rel(got, want), 1.0e-7, rel(o.sample_one_step(img.double(), t - 1)[0], want))   # measured 3.5e-8
    ck.done()


@pytest.mark.parametrize('to_lab', [False, True])
def test_decolorization_at_256(tmp_path, to_lab):
    """Decolorization in the decolor driver's configuration ('Linear', total removal): q_sample (cd_chanmix, or cd_chanmix_lab
    with `to_lab`) and one x0_step_down step against SnowOracle in fp64 with oracle/snow_oracle.py's DecolorFP (RGB) or
    tests/lab_oracle.py's DecolorLabFP (Lab: step i = rgb2lab(M_i lab2rgb(x)), the inputs in Lab)"""
    import lab_oracle as LO
    import snow_oracle as SO
    ck = Checks('decolor256[lab=%d]' % to_lab)
    # measured: RGB q_sample <= 3.6e-8, step 2.9e-8; Lab (fp32 powf and branch thresholds) q_sample <= 6.0e-7, step 1.5e-7
    bound_q, bound_step = (1.8e-6, 4.5e-7) if to_lab else (1.1e-7, 8.7e-8)
    S, T, B = 256, 20, 3
    gd = _snow_package('Decolorization', S, T, tmp_path, decolor_routine='Linear', decolor_total_remove=True, to_lab=to_lab)
    factors = gd.forward_process.factors
    fp = LO.DecolorLabFP(factors) if to_lab else SO.DecolorFP(factors)
    fp.w = [w.to(DEV, F64) for w in fp.w]
    o = SO.SnowOracle(Toy(), fp, timesteps=T, sampling_routine='x0_step_down')
    x = torch.rand(B, 3, S, S, generator=gen(17), device=DEV) * 2 - 1
    if to_lab:
        x = LO.rgb2lab(x.double()).float()
    for t in (torch.tensor([0, 9, T - 1], device=DEV), torch.tensor([4, -1, 12], device=DEV)):
        r = o.q_sample(x.double(), t)
        ck('q_sample t=%s' % t.tolist(), rel(gd.q_sample(x, t), r), bound_q, rel(o.q_sample(x.double(), (t + 1).clamp(max=T - 1)), r))
    t = torch.tensor([1, 9, T - 1], device=DEV)
    img = gd.q_sample(x, t)
    got, _ = gd.sample_one_step(img, t)
    want, _ = o.sample_one_step(img.double(), t)
    # control: the images of the batch swapped (in RGB the mix has nearly converged by these steps, so a step index off by
    # one changes the result by only 4e-10)
    ck('x0_step_down step', rel(got, want), bound_step, rel(want.roll(1, 0), want))
    ck.done()
