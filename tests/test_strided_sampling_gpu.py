"""Strided sampling (`sample(..., steps=K)`) on the GPU.

* identity: steps = t is the full loop bit for bit, for every package and sampling routine, eager and from the CUDA graph; the
  strided entry points at s = t - 1 are their one-step versions bit for bit;
* values: the strided loops against float64 restatements (tests/strided_oracle.py) built from the oracles' degradations and
  the oracle Unet forward with the same weights, at 32² (T = 10 - 20, K in {1, 3, T/2}) and at the config-3 shape (128²,
  T = 200, K = 20).  The Unet runs TF32 tensor-core convolutions, so each bound sits beside the error measured on an H100 SXM
  (700 W);
* controls: the restatement with the update stepping to hi - 1 instead of lo, and with the cosine table read at s instead of
  s - 1, must not match;
* a strided graphed sample replays the per-shape forward graph (no capture per stride); invalid steps and routines without a
  strided form raise ValueError naming them."""
import ctypes as C

import pytest
import torch

import strided_oracle as SO
import unet_oracle as UO
from test_unet_gpu import load, rel, make_unet

pytestmark = pytest.mark.gpu
F64 = torch.float64


@pytest.fixture(scope='module')
def small():
    g = load('unet_small')
    sd = {k[3:]: v for k, v in g.items() if k.startswith('sd:')}
    sd64 = {k: v.to(F64) for k, v in sd.items()}
    return make_unet(32, (1, 2), 3, sd), (lambda x, t: UO.unet_forward(sd64, x.cpu(), t.cpu().to(F64)))


def image(S=32, B=2, seed=0):
    return (torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(seed)) * 2 - 1).cuda()


def _pkgs(unet):
    """(name, constructor, sample call) for every package and sampling routine with a strided form"""
    from cold_diffusion_models_b200 import deblurring, resolution, defading, denoising, demixing, defading_generation, snowification
    out = []
    for r in ('default', 'x0_step_down'):
        for kw in (dict(blur_routine='Exponential_reflect', kernel_std=0.15, kernel_size=7),
                   dict(blur_routine='Incremental', kernel_std=0.3, kernel_size=5, discrete=True)):
            out.append(('deblurring %s %s' % (r, kw['blur_routine']), lambda r=r, kw=kw: deblurring.GaussianDiffusion(
                unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=10, sampling_routine=r, **kw), 'img'))
        out.append(('resolution ' + r, lambda r=r: resolution.GaussianDiffusion(
            unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=10, resolution_routine='Incremental',
            sampling_routine=r), 'img'))
        for fr in ('Incremental', 'Random_Incremental'):
            out.append(('defading %s %s' % (r, fr), lambda r=r, fr=fr: defading.GaussianDiffusion(
                unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=10, fade_routine=fr, sampling_routine=r),
                'faded_recon_sample'))
        for fpt in ('Decolorization', 'Snow'):
            out.append(('snowification %s %s' % (r, fpt), lambda r=r, fpt=fpt: snowification.GaussianDiffusion(
                unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=10, forward_process_type=fpt,
                sampling_routine=r), 'img'))
    out.append(('deblurring x0_step_down Individual_Incremental', lambda: deblurring.GaussianDiffusion(
        unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=6, blur_routine='Individual_Incremental',
        sampling_routine='x0_step_down'), 'img'))
    out.append(('denoising', lambda: denoising.GaussianDiffusion(unet, image_size=32, channels=3, timesteps=20), 'img'))
    out.append(('demixing', lambda: demixing.GaussianDiffusion(unet, image_size=32, channels=3, timesteps=20), 'img'))
    for rev in (False, True):
        out.append(('defading_generation reverse=%s' % rev, lambda rev=rev: defading_generation.GaussianDiffusion(
            unet, image_size=32, channels=3, timesteps=10, reverse=rev, kernel_std=0.6, initial_mask=3), 'img'))
    return out


_OFFSETS = (torch.tensor([3, 30]), torch.tensor([17, 0]))      # the 'Random_*' fade windows (rows, columns) of both samples


def _run(gd, key, x, **kw):
    extra = {'_offsets': tuple(o.cuda() for o in _OFFSETS)} if 'Random' in getattr(gd, 'fade_routine', '') else {}
    out = gd.sample(batch_size=x.shape[0], **{key: x}, **extra, **kw)
    out = list(out.values()) if isinstance(out, dict) else list(out)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('graphed', [False, True])
def test_steps_equal_to_t_is_the_full_loop_bit_for_bit(small, graphed):
    unet, _ = small
    x = image()
    eng = unet.engine
    eng.enable_cuda_graph(graphed)
    try:
        for name, make, key in _pkgs(unet):
            gd = make().cuda()
            full = _run(gd, key, x)
            strided = _run(gd, key, x, steps=gd.num_timesteps)
            assert all(torch.equal(a, b) for a, b in zip(full, strided)), name
    finally:
        eng.enable_cuda_graph(False)


def test_strided_entry_points_at_one_step_equal_the_one_step_kernels():
    from cold_diffusion_models_b200._lib import call, ptr, stream
    g = torch.Generator().manual_seed(5)
    T, B, S = 20, 3, 32
    sa = (torch.rand(T, generator=g) * 0.9 + 0.05).cuda()
    sb = (1 - sa * sa).sqrt()
    for n, off in ((B * 3 * S * S, 0), (B * 3 * S * S - 3, 0), (4099, 1)):
        img, x1, nz = ((torch.randn(n + off, generator=g).cuda())[off:] for _ in range(3))
        for mode in (0, 1):
            for t in (1, 2, 11, 20):
                a, b = torch.empty_like(img), torch.empty_like(img)
                call('cd_noise_step', ptr(img), ptr(x1), ptr(nz), mode, t, ptr(sa), ptr(sb), C.c_int64(n), ptr(a), stream())
                call('cd_noise_step_to', ptr(img), ptr(x1), ptr(nz), mode, t, t - 1, ptr(sa), ptr(sb), C.c_int64(n), ptr(b), stream())
                assert torch.equal(a, b), (n, off, mode, t)
    al = torch.rand(T, 1, S, S, generator=g).cuda()
    om = 1 - al
    for S_, off in ((32, 0), (30, 0), (32, 1)):
        n = B * 3 * S_ * S_
        alS, omS = al[:, :, :S_, :S_].contiguous(), om[:, :, :S_, :S_].contiguous()
        img, x1, x2 = ((torch.randn(n + off, generator=g).cuda())[off:] for _ in range(3))
        for t in (1, 2, 11, 20):
            a, b = torch.empty_like(img), torch.empty_like(img)
            call('cd_fade_step', ptr(img), ptr(x1), ptr(x2), t, ptr(alS), ptr(omS), B, 3, S_ * S_, ptr(a), stream())
            call('cd_fade_step_to', ptr(img), ptr(x1), ptr(x2), t, t - 1, ptr(alS), ptr(omS), B, 3, S_ * S_, ptr(b), stream())
            assert torch.equal(a, b), (S_, off, t)


# ---- values against float64 --------------------------------------------------------------------------------------------
def _restatements(name, gd, net64, x64):
    """-> (update, x_T) of the float64 restatement of package `gd`'s strided loop"""
    import deblur_oracle as DO, resolution_oracle as RO, defading_oracle as FO, snow_oracle as NO
    T = gd.num_timesteps
    if name.startswith('deblurring'):
        D = SO.deblur_D(DO.DeblurOracle(net64, image_size=32, channels=3, timesteps=T, kernel_std=gd.kernel_std,
                                        kernel_size=gd.kernel_size, blur_routine=gd.blur_routine))
        return SO.cold_update(D, gd.sampling_routine), D(x64, T)
    if name.startswith('resolution'):
        D = SO.resolution_D(RO.ResolutionOracle(net64, image_size=32, channels=3, timesteps=T, resolution_routine='Incremental'))
        return SO.cold_update(D, gd.sampling_routine), D(x64, T)
    if name.startswith('defading_generation'):
        return SO.fade_update(gd.alphas.cpu(), gd.one_minus_alphas.cpu(), x64), x64
    if name.startswith('defading'):
        rx, ry = _OFFSETS if 'Random' in gd.fade_routine else (None, None)
        D = SO.defading_D(FO.DefadeOracle(net64, image_size=32, channels=3, timesteps=T, fade_routine=gd.fade_routine), rx, ry)
        return SO.cold_update(D, gd.sampling_routine), D(x64, T)
    if name.startswith('denoising') or name.startswith('demixing'):
        return SO.noise_update(gd.sqrt_alphas_cumprod.cpu(), gd.sqrt_one_minus_alphas_cumprod.cpu()), x64
    fp = gd.forward_process
    if name.endswith('Decolorization'):
        o = NO.DecolorFP(fp.factors)
        o.w = [w.to(F64) for w in o.w]
    else:
        o = NO.SnowFP(fp.layers('cuda').cpu().to(F64), fp.br_t.to(F64), fp.fix_brightness)
    D = SO.snow_D(o)
    return SO.snow_update(D, gd.sampling_routine), D(x64, T)


# rel. error of the final image at K = 1 / 3 / T/2: at most 8.1e-4 measured on an H100 SXM (700 W), bound about 3x that
_BOUND = 2.5e-3


def test_strided_samples_match_float64_restatements(small):
    unet, net64 = small
    x = image()
    x64 = x.cpu().to(F64)
    errs, controls = {}, {}
    for name, make, key in _pkgs(unet):
        gd = make().cuda()
        if getattr(gd, 'discrete', False) or 'Individual' in name:
            continue             # `discrete` and Individual_Incremental: covered by the identity test
        T = gd.num_timesteps
        update, xT = _restatements(name, gd, net64, x64)
        for K in (1, 3, T // 2):
            img = _run(gd, key, x, steps=K)[2]
            _, ref = SO.reverse(net64, xT, T, K, update, 2)
            errs[name, K] = rel(img, ref)
            if K > 1:
                # controls: stepping to hi - 1 instead of lo, and the cosine table read at s instead of s - 1
                _, bad = SO.reverse(net64, xT, T, K, update, 2, lo_of=lambda hi, lo: hi - 1)
                controls[name, K, 'lo = hi - 1'] = rel(img, bad)
                if name in ('denoising', 'demixing'):
                    shifted = SO.noise_update(gd.sqrt_alphas_cumprod.cpu(), gd.sqrt_one_minus_alphas_cumprod.cpu(), table_shift=0)
                    _, bad = SO.reverse(net64, xT, T, K, shifted, 2)
                    controls[name, K, 'sqrt_ac[s]'] = rel(img, bad)
    print('strided rel. error vs float64:', {'%s K=%d' % k: '%.1e' % v for k, v in errs.items()})
    print('controls:', {'%s K=%d %s' % k: '%.1e' % v for k, v in controls.items()})
    assert max(errs.values()) < _BOUND, max(errs.items(), key=lambda kv: kv[1])
    # each control lies at least 5x farther from the package than the restatement does (measured: 9x at the closest)
    ratio = {k: v / errs[k[:2]] for k, v in controls.items()}
    assert min(ratio.values()) > 5, min(ratio.items(), key=lambda kv: kv[1])


def test_config3_strided_sample_at_128_matches_float64():
    """config 3 (Unet(64, (1, 2, 4, 8)), 128², T = 200, Exponential_reflect blur, x0_step_down), graphed, K = 20"""
    import cold_diffusion_models_b200 as cdm
    import deblur_oracle as DO
    sd = UO.make_unet_state_dict(64, (1, 2, 4, 8), 3, seed=0)
    unet = make_unet(64, (1, 2, 4, 8), 3, sd)
    kw = dict(image_size=128, channels=3, timesteps=200, kernel_std=0.01, kernel_size=15, blur_routine='Exponential_reflect')
    gd = cdm.GaussianDiffusion(unet, device_of_kernel='cuda', sampling_routine='x0_step_down', **kw).cuda()
    x = image(128, 2, seed=3)
    eng = unet.engine
    eng.enable_cuda_graph(True)
    try:
        xt, dr, img = gd.sample(batch_size=2, img=x, steps=20)
        torch.cuda.synchronize()
        assert len(eng._graphs) == 1
    finally:
        eng.enable_cuda_graph(False)
    sd64 = {k: v.to('cuda', F64) for k, v in sd.items()}
    net64 = lambda a, s: UO.unet_forward(sd64, a, s.to(a.device, F64))
    o = DO.DeblurOracle(net64, **kw)
    o.kernels2d = [k.to('cuda', F64) for k in o.kernels2d]
    D = lambda a, n: o._cum(a, n)
    x64 = x.to(F64)
    ref_dr, ref = SO.reverse(net64, D(x64, 200), 200, 20, SO.cold_update(D, 'x0_step_down'), 2)
    e_dr, e = rel(dr, ref_dr), rel(img, ref)
    print('config-3 K = 20 rel. error vs float64: direct %.2e, sample %.2e' % (e_dr, e))
    assert e_dr < 2e-3 and e < 3.5e-3, (e_dr, e)        # measured 6.5e-4 and 1.1e-3
    _, bad = SO.reverse(net64, D(x64, 200), 200, 20, SO.cold_update(D, 'x0_step_down'), 2, lo_of=lambda hi, lo: hi - 1)
    assert rel(img, bad) > 10 * e


def test_strided_graphed_sample_replays_the_per_shape_graph(small):
    unet, _ = small
    from cold_diffusion_models_b200 import deblurring
    gd = deblurring.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=10,
                                      blur_routine='Exponential_reflect', kernel_std=0.15, kernel_size=7,
                                      sampling_routine='x0_step_down').cuda()
    x = image()
    eng = unet.engine
    eager = {K: gd.sample(batch_size=2, img=x, steps=K) for K in (1, 3, 7)}
    eng.enable_cuda_graph(True)
    try:
        gd.sample(batch_size=2, img=x)
        graphs = {k: id(v[0]) for k, v in eng._graphs.items()}
        assert list(graphs) == [(2, 3, 32, 32)]
        for K in (1, 3, 7):
            graphed = gd.sample(batch_size=2, img=x, steps=K)
            assert {k: id(v[0]) for k, v in eng._graphs.items()} == graphs, K
            assert all(torch.equal(a, b) for a, b in zip(graphed, eager[K])), K
    finally:
        eng.enable_cuda_graph(False)


def test_invalid_steps_and_routines_without_a_strided_form_raise(small):
    unet, _ = small
    from cold_diffusion_models_b200 import deblurring, resolution, defading, denoising, defading_generation, snowification
    x = image()
    gd = denoising.GaussianDiffusion(unet, image_size=32, channels=3, timesteps=10).cuda()
    for bad in (0, 11, -2, 2.5, '4'):
        with pytest.raises(ValueError, match='steps'):
            gd.sample(batch_size=2, img=x, steps=bad)
    gf = defading_generation.GaussianDiffusion(unet, image_size=32, channels=3, timesteps=10).cuda()
    with pytest.raises(ValueError, match='steps'):
        gf.sample(batch_size=2, img=x, steps=11)
    cases = [
        (deblurring.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', timesteps=6, blur_routine='Individual_Incremental'),
         'img', 'Individual_Incremental'),
        (deblurring.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', timesteps=6, sampling_routine='ddim'), 'img', 'ddim'),
        (deblurring.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', timesteps=6, train_routine='Step'), 'img', 'Step'),
        (resolution.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', timesteps=6, sampling_routine='other'),
         'img', 'other'),
        (defading.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', timesteps=6, sampling_routine='other'),
         'faded_recon_sample', 'other'),
        (snowification.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', timesteps=6, train_routine='Step_Gradient'),
         'img', 'Step_Gradient'),
    ]
    for gd, key, routine in cases:
        gd = gd.cuda()
        with pytest.raises(ValueError, match=routine):
            gd.sample(batch_size=2, **{key: x}, steps=3)
        with pytest.raises(ValueError, match=routine):
            gd.sample(batch_size=2, **{key: x}, steps=gd.num_timesteps)
