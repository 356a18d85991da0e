"""`Unet(64, (1, 2, 4, 8))` trained and sampled at 512²: the parameter gradients of a 512² micro-batch, one optimizer step through
the Trainer and the gradient at the new weights, a CUDA-graph sample of the EMA model, batch independence of the gradient, and
one training step of each package that accepts 512² images (deblurring, resolution, snow, decolorization in RGB and Lab),
against float64 references computed on the GPU from oracle/.

As in tests/test_large_images_gpu.py, every comparison also evaluates its metric on a deliberately wrong reference (a
negative control) and asserts that it exceeds the bound.  Every bound is at most 3x the value measured on an H100 80GB HBM3
(700 W), which is in the comment beside it.  Set COLDDIFF_TEST_METRICS=<file> to write all values and controls as JSON.
The file runs in about 55 s on that card; its peak device memory is 55.8 GiB (the B = 8 batch-independence test)."""
import contextlib
import io
import math

import pytest
import torch

import deblur_oracle as DO
import resolution_oracle as RO
import snow_oracle as SO
import unet_oracle as UO
from test_config3_step_gpu import (Checks, _metrics_file, _free_between_tests, _METRICS, rel, gen, blur_per_image,  # noqa: F401
                                   ref_step, engine_grads, grad_errors, stats)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
S = 512


def _unet(seed=3):
    import cold_diffusion_models_b200 as cdm
    with contextlib.redirect_stdout(io.StringIO()):
        unet = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).to(DEV)
        sd = UO.make_unet_state_dict(64, (1, 2, 4, 8), 3, seed=seed)
        unet.load_state_dict(sd)
    return unet, sd


def _blur(T, denoise_fn=None, **kw):
    kw.update(image_size=S, channels=3, timesteps=T, kernel_std=0.1, kernel_size=11, blur_routine='Exponential_reflect')
    o = DO.DeblurOracle(denoise_fn, **kw)
    o.kernels2d = [k.double().cuda() for k in o.kernels2d]
    return o


def _fp64_net(sd):
    sd64 = {k: v.detach().to(DEV, F64) for k, v in sd.items()}
    return lambda a, s: UO.unet_forward(sd64, a, s.to(a.device, F64))


def _grad_check(ck, name, eg, ref, ctrl, bmed, bworst):
    errs = grad_errors(eg, ref)
    med, p90, worst = stats(errs)
    cmed, _, cworst = stats(grad_errors(eg, ctrl))
    _METRICS['%s::%s p90' % (ck.test, name)] = p90
    _METRICS['%s::%s worst parameters' % (ck.test, name)] = [(e, n) for e, n in errs[-5:]]
    ck.require('%s: %d parameter gradients' % (name, len(errs)), len(errs) == 238)
    ck('%s median' % name, med, bmed, cmed)
    ck('%s worst' % name, worst, bworst, cworst)


# ==========================================================================================================================
# gradients, one optimizer step and a graphed sample
# ==========================================================================================================================
def test_unet_512_gradients_step_and_graphed_sample(tmp_path):
    import cold_diffusion_models_b200 as cdm
    ck = Checks('unet512 train')
    T, B = 20, 2
    unet, sd = _unet()
    gd = cdm.GaussianDiffusion(unet, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, kernel_std=0.1,
                               kernel_size=11, blur_routine='Exponential_reflect', loss_type='l2',
                               sampling_routine='x0_step_down').to(DEV)
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(B, 3, S, S, generator=g) * 2 - 1).to(DEV)
    t = torch.tensor([3, T - 1], device=DEV)
    o = _blur(T)
    xt64 = blur_per_image(o, x.double(), t)
    # the gradients of one micro-batch against fp64 autograd through oracle/unet_oracle.py, one image per chunk; the control
    # leaves the second image out
    unet.zero_grad(set_to_none=True)
    gd.p_losses(x, t).backward()
    eg = engine_grads(unet)
    g0, _, _ = ref_step(sd, x[:1], xt64[:1], t[:1], norm=x.numel(), chunk=1)
    g1, _, _ = ref_step(sd, x[1:], xt64[1:], t[1:], norm=x.numel(), chunk=1)
    ref_old = {k: g0[k] + g1[k] for k in g0}
    _grad_check(ck, 'grad', eg, ref_old, g0, 3.3e-3, 6.7e-3)            # measured median 1.1e-3, worst 2.2e-3 (256²: 1.1e-3, 2.1e-3)
    del g0, g1, eg
    # one optimizer step through the Trainer (Adam at lr 1e-3, EMA), then the gradient at the new weights; the control is the
    # reference gradient at the old weights (stale forward or data-gradient packs would give that one)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=1e-3, train_num_steps=10 ** 9,
                         gradient_accumulate_every=1, ema_decay=0.995, fp16=False, results_folder=str(tmp_path),
                         dataset='synthetic')
    before = {k: v.detach().clone() for k, v in unet.state_dict().items()}
    loss = tr.train_step([x]).item()
    ck.require('train_step loss finite (%r)' % loss, math.isfinite(loss) and abs(loss) < 1e3)
    moved = max((unet.state_dict()[k].double() - before[k].double()).abs().max().item() for k in before)
    ck.require('train_step moved the weights (%.3e)' % moved, 1e-5 < moved < 1e-2)
    _METRICS['unet512 train::weights moved (max abs)'] = moved
    del before
    tr.opt.zero_grad()
    gd.p_losses(x, t).backward()
    torch.cuda.synchronize()
    eg = engine_grads(unet)
    tr.opt.zero_grad()
    sd1 = {k: v.detach().clone() for k, v in unet.state_dict().items()}
    g0, _, _ = ref_step(sd1, x[:1], xt64[:1], t[:1], norm=x.numel(), chunk=1)
    g1, _, _ = ref_step(sd1, x[1:], xt64[1:], t[1:], norm=x.numel(), chunk=1)
    ref_new = {k: g0[k] + g1[k] for k in g0}
    del g0, g1, sd1
    _grad_check(ck, 'grad after the step', eg, ref_new, ref_old, 1.5e-3, 4.8e-3)     # measured median 5.1e-4, worst 1.6e-3
    del ref_new, ref_old, eg
    # the graphed 3-step x0_step_down sample of the EMA model
    ema = tr.ema_model
    eng = ema.denoise_fn.engine
    eng.enable_cuda_graph(True)
    try:
        with torch.no_grad():
            xt, dr, img = ema.sample(batch_size=B, img=x, t=3)
        torch.cuda.synchronize()
    finally:
        eng.enable_cuda_graph(False)
    os_ = _blur(T, denoise_fn=_fp64_net(ema.denoise_fn.state_dict()), sampling_routine='x0_step_down')
    with torch.no_grad():
        r = os_.sample(B, x.double(), t=3)
    ck('graphed sample x_t', rel(xt, r[0]), 3.7e-7,                    # measured 1.3e-7
       rel(xt, blur_per_image(o, x.double(), torch.full((B,), 1))))
    ck('graphed sample direct', rel(dr, r[1]), 4.5e-4, rel(dr.roll(1, 0), r[1]))        # measured 1.5e-4
    ck('graphed sample', rel(img, r[2]), 9.7e-4, rel(xt, r[2]))                      # measured 3.3e-4
    ck.done()


@pytest.mark.parametrize('B', [2, 8])
def test_unet_512_batch_independence(B):
    """the gradient of B images in one pass against the sum of the same engine's gradients over B passes of one image (other
    grids, linear-attention spans and weight-gradient splits; the same arithmetic per image).  B = 8 is the largest batch
    that trains and samples in one process on an 80 GB card (tools/blur_shapes.py --size 512).  The control leaves the last
    one-image pass out."""
    import cold_diffusion_models_b200 as cdm
    ck = Checks('unet512 batch independence[B=%d]' % B)
    T = 20
    unet, _ = _unet(seed=6)
    gd = cdm.GaussianDiffusion(unet, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, kernel_std=0.1,
                               kernel_size=11, blur_routine='Exponential_reflect', loss_type='l2').to(DEV)
    x = torch.rand(B, 3, S, S, generator=gen(21), device=DEV) * 2 - 1
    t = torch.randint(0, T, (B,), generator=gen(22), device=DEV)
    unet.zero_grad(set_to_none=True)
    gd.p_losses(x, t).backward()
    whole = engine_grads(unet)
    unet.zero_grad(set_to_none=True)
    for i in range(B):
        if i == B - 1:
            partial = engine_grads(unet)
        (gd.p_losses(x[i:i + 1], t[i:i + 1]) / B).backward()
    split = engine_grads(unet)
    unet.zero_grad(set_to_none=True)
    # measured median 1.5e-4 (B = 2) and 1.1e-4 (B = 8), worst 3.5e-4 and 3.6e-4; one pass left out: median 0.88 and 0.16
    bmed, bworst = {2: (4.5e-4, 1.0e-3), 8: (3.3e-4, 1.0e-3)}[B]
    _grad_check(ck, 'grad', split, whole, partial, bmed, bworst)
    ck.done()


# ==========================================================================================================================
# one training step of each package that accepts 512² images
# ==========================================================================================================================
def _package(kind, unet, tmp_path):
    """-> (package, oracle/ restatement of it for a given network, the per-image t of the test batch)"""
    if kind == 'deblurring':
        import cold_diffusion_models_b200 as cdm
        T = 20
        gd = cdm.GaussianDiffusion(unet, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, kernel_std=0.1,
                                   kernel_size=11, blur_routine='Exponential_reflect', loss_type='l1').to(DEV)
        return gd, lambda fn: _blur(T, denoise_fn=fn), [3, T - 1]
    if kind == 'resolution':
        from cold_diffusion_models_b200.resolution_diffusion_pytorch import GaussianDiffusion as RSGD
        T = 4                                     # the constructor tabulates T operators on the CPU
        gd = RSGD(unet, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1',
                  resolution_routine='Incremental').to(DEV)
        return gd, lambda fn: RO.ResolutionOracle(fn, image_size=S, channels=3, timesteps=T, resolution_routine='Incremental'), [1, T - 1]
    from cold_diffusion_models_b200.snowification_diffusion import GaussianDiffusion as SNGD
    T = 8 if kind == 'snow' else 20
    kw = dict(snow_level=1) if kind == 'snow' else dict(decolor_routine='Linear', decolor_total_remove=True,
                                                        to_lab=kind == 'decolorization-lab')
    with contextlib.redirect_stdout(io.StringIO()):
        gd = SNGD(unet, image_size=(S, S) if kind == 'snow' else S, device_of_kernel='cuda', channels=3, timesteps=T,
                  loss_type='l1', forward_process_type='Snow' if kind == 'snow' else 'Decolorization', train_routine='Final',
                  sampling_routine='x0_step_down', results_folder=str(tmp_path), **kw).to(DEV)
    if kind == 'snow':
        ref_layers, br = SO.generate_snow_layers((S, S), snow_level=1, num_timesteps=T)
        fp = SO.SnowFP(ref_layers.to(DEV, F64), br)
    elif kind == 'decolorization-lab':
        import lab_oracle as LO
        fp = LO.DecolorLabFP(gd.forward_process.factors)
        fp.w = [w.to(DEV, F64) for w in fp.w]
    else:
        fp = SO.DecolorFP(gd.forward_process.factors)
        fp.w = [w.to(DEV, F64) for w in fp.w]
    return gd, lambda fn: SO.SnowOracle(fn, fp, timesteps=T, loss_type='l1'), [2, T - 1]


# relative error of the loss; measured in two runs: deblurring 7.6e-6 / 7.9e-6, resolution 8.2e-6 / 7.8e-6, snow 4.4e-7 / 2.4e-7,
# RGB decolorization 4.6e-6 / 4.2e-6, Lab 1.6e-6 / 5.2e-7 (controls 4.0e-4 to 4.1e-3)
LOSS_BOUND = {'deblurring': 2.3e-5, 'resolution': 2.4e-5, 'snow': 1.3e-6, 'decolorization-rgb': 1.3e-5, 'decolorization-lab': 4.8e-6}


@pytest.mark.parametrize('kind', list(LOSS_BOUND))
def test_package_training_step_at_512(kind, tmp_path):
    """p_losses and its backward on a 512² micro-batch of two images: the loss is finite and equal to the package's fp64
    restatement from oracle/ with the Unet of oracle/unet_oracle.py (control: the restatement with the degradation skipped),
    and every parameter gradient is finite and not all zero.  Snow also checks its device-generated layers (cd_snow_layers)
    against the host restatement of the reference generator."""
    ck = Checks('package512[%s]' % kind)
    unet, sd = _unet(seed=8)
    gd, make_oracle, tl = _package(kind, unet, tmp_path)
    x = torch.rand(2, 3, S, S, generator=gen(23), device=DEV) * 2 - 1
    if kind == 'decolorization-lab':
        import lab_oracle as LO
        x = LO.rgb2lab(x.double()).float()
    t = torch.tensor(tl, device=DEV)
    if kind == 'snow':
        layers = gd.forward_process.layers(DEV)
        ref = make_oracle(None).fp.snow
        ck('snow layers', (layers.double() - ref).abs().max().item(), 1e-7,
           (layers[1:].double() - ref[:-1]).abs().max().item())
    unet.zero_grad(set_to_none=True)
    loss = gd.p_losses(x, t)
    loss.backward()
    torch.cuda.synchronize()
    lv = loss.item()
    ck.require('loss finite (%r)' % lv, math.isfinite(lv))
    grads = engine_grads(unet)
    ck.require('every gradient finite', all(bool(torch.isfinite(v).all()) for v in grads.values()))
    ck.require('gradients not all zero', sum(float(v.abs().sum()) for v in grads.values()) > 0)
    o = make_oracle(_fp64_net(sd))
    with torch.no_grad():
        want = (x.double() - o.denoise_fn(o.q_sample(x.double(), t), t)).abs().mean().item()
        skipped = (x.double() - o.denoise_fn(x.double(), t)).abs().mean().item()
    ck('loss', abs(lv - want) / want, LOSS_BOUND[kind], abs(skipped - want) / want)
    ck.done()
