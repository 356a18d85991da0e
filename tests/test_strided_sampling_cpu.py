"""Strided sampling (`sample(..., steps=K)`) without a GPU: the level schedule, the two strided entry points
(cd_noise_step_to, cd_fade_step_to) on their numpy statements (tests/strided_oracle.py) and on their CUDA sources compiled for the CPU against
a float64 restatement, and the packages' strided loops on the emulated ABI with a small deterministic network."""
import ctypes as C

import numpy as np
import pytest
import torch

import abi_emulator
import strided_oracle as SO
from cold_diffusion_models_b200.strided import reverse_levels


# ---- the schedule ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('t', [1, 2, 3, 7, 10, 50, 200, 1000])
def test_levels_run_from_t_to_zero_strictly_decreasing(t):
    for K in sorted({k for k in (1, 2, 3, t // 3, t // 2, t - 1, t) if 1 <= k <= t}):
        lv = reverse_levels(t, K)
        assert len(lv) == K + 1 and lv[0] == t and lv[-1] == 0, (t, K, lv)
        assert all(a > b for a, b in zip(lv, lv[1:])), (t, K, lv)
        # round(t (K - i) / K), halves rounded up
        assert lv == [int(np.floor(t * (K - i) / K + 0.5)) for i in range(K + 1)]
    assert reverse_levels(t, t) == list(range(t, -1, -1)) == reverse_levels(t)


def test_levels_examples():
    assert reverse_levels(200, 10) == [200, 180, 160, 140, 120, 100, 80, 60, 40, 20, 0]
    assert reverse_levels(10, 4) == [10, 8, 5, 3, 0]
    assert reverse_levels(5, 1) == [5, 0]


@pytest.mark.parametrize('bad', [0, -1, 11, 2.0, 2.5, '3', True, [3]])
def test_levels_reject_what_they_cannot_use(bad):
    with pytest.raises(ValueError):
        reverse_levels(10, bad)


def test_levels_accept_numpy_integers():
    assert reverse_levels(10, np.int64(2)) == [10, 5, 0]


# ---- the entry points --------------------------------------------------------------------------------------------------
def _p(a):
    return C.c_void_p(a.data_ptr())


def _noise_ref(img, x1, noise, mode, t, s, sa, sb):
    img, x1, sa, sb = img.double(), x1.double(), sa.double(), sb.double()
    x2 = (img - sa[t - 1] * x1) / sb[t - 1] if mode == 0 else noise.double()
    xs = x1 if s == 0 else sa[s - 1] * x1 + sb[s - 1] * x2
    return img - (sa[t - 1] * x1 + sb[t - 1] * x2) + xs


def _fade_ref(img, x1, x2, t, s, al, om):
    img, x1, x2, al, om = (a.double() for a in (img, x1, x2, al, om))
    xs = x1 if s == 0 else al[s - 1] * x1 + om[s - 1] * x2
    return img - (al[t - 1] * x1 + om[t - 1] * x2) + xs


def _backends():
    SO.install_emulator()
    return [('numpy', abi_emulator.call), ('cuda_source', abi_emulator.call_cuda_source)]


@pytest.mark.parametrize('backend', ['numpy', 'cuda_source'])
@pytest.mark.parametrize('n,offset', [(4096, 0), (4099, 0), (1024, 1)])   # float4 path, its scalar tail, misaligned operands
def test_noise_step_to_matches_float64(backend, n, offset):
    call = dict(_backends())[backend]
    g = torch.Generator().manual_seed(n + offset)
    T = 20
    sa = torch.rand(T, generator=g) * 0.9 + 0.05
    sb = (1 - sa * sa).sqrt()
    buf = [torch.randn(n + offset, generator=g) for _ in range(3)]
    img, x1, noise = (b[offset:] for b in buf)
    for mode in (0, 1):
        for t, s in ((20, 0), (20, 13), (7, 6), (1, 0), (5, 1)):
            out = torch.empty(n + offset)[offset:]
            call('cd_noise_step_to', _p(img), _p(x1), _p(noise), mode, t, s, _p(sa), _p(sb), C.c_int64(n), _p(out), None)
            ref = _noise_ref(img, x1, noise, mode, t, s, sa, sb)
            err = (out.double() - ref).abs().max().item()
            assert err < 2e-5 * (1 + ref.abs().max().item()), (mode, t, s, err)
            if s == t - 1:            # one step: cd_noise_step's bits
                one = torch.empty(n + offset)[offset:]
                call('cd_noise_step', _p(img), _p(x1), _p(noise), mode, t, _p(sa), _p(sb), C.c_int64(n), _p(one), None)
                assert torch.equal(one, out), (mode, t)


@pytest.mark.parametrize('backend', ['numpy', 'cuda_source'])
@pytest.mark.parametrize('S,offset', [(16, 0), (6, 0), (16, 1)])        # float4 path, HW % 4 != 0, misaligned operands
def test_fade_step_to_matches_float64(backend, S, offset):
    call = dict(_backends())[backend]
    g = torch.Generator().manual_seed(S + offset)
    T, B, Cc, HW = 12, 2, 3, S * S
    al = torch.rand(T, 1, S, S, generator=g)
    om = 1 - al
    n = B * Cc * HW
    buf = [torch.randn(n + offset, generator=g) for _ in range(3)]
    img, x1, x2 = (b[offset:].view(B, Cc, S, S) for b in buf)
    for t, s in ((12, 0), (12, 5), (4, 3), (1, 0)):
        out = torch.empty(n + offset)[offset:].view(B, Cc, S, S)
        call('cd_fade_step_to', _p(img), _p(x1), _p(x2), t, s, _p(al), _p(om), B, Cc, HW, _p(out), None)
        ref = _fade_ref(img, x1, x2, t, s, al, om)
        assert (out.double() - ref).abs().max().item() < 2e-6 * (1 + ref.abs().max().item()), (t, s)
        if s == t - 1:
            one = torch.empty(n + offset)[offset:].view(B, Cc, S, S)
            call('cd_fade_step', _p(img), _p(x1), _p(x2), t, _p(al), _p(om), B, Cc, HW, _p(one), None)
            assert torch.equal(one, out), t


def test_strided_entry_points_reject_bad_levels():
    x = torch.zeros(16)
    sa = torch.ones(4)
    for t, s in ((4, 4), (4, 5), (4, -1), (0, 0)):
        with pytest.raises(RuntimeError, match='cd_noise_step_to'):
            abi_emulator.call_cuda_source('cd_noise_step_to', _p(x), _p(x), None, 0, t, s, _p(sa), _p(sa), C.c_int64(16), _p(x), None)
        with pytest.raises(RuntimeError, match='cd_fade_step_to'):
            abi_emulator.call_cuda_source('cd_fade_step_to', _p(x), _p(x), _p(x), t, s, _p(sa), _p(sa), 1, 1, 16, _p(x), None)


# ---- the packages' strided loops on the emulated ABI ---------------------------------------------------------------------
def net(x, t):
    """a small deterministic stand-in for the restoration network: smooth in x, depends on t"""
    return torch.tanh(0.8 * x + 0.01 * t.to(x.dtype)[:, None, None, None]) * 0.9


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)
    SO.install_emulator()
    with abi_emulator.patched():
        yield


def _image(S=16, B=2, seed=0):
    return torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def _check(pkg_out, ref, tol):
    err = ((pkg_out.double() - ref).norm() / ref.norm()).item()
    assert err < tol, err


class _Net(torch.nn.Module):
    def forward(self, x, t):
        return net(x, t)


def test_deblurring_and_resolution_strided_loops(emulated):
    import deblur_oracle as DO
    import resolution_oracle as RO
    from cold_diffusion_models_b200 import deblurring, resolution
    x = _image()
    for routine in ('default', 'x0_step_down'):
        kw = dict(image_size=16, channels=3, timesteps=8, kernel_std=0.3, kernel_size=5, blur_routine='Incremental')
        gd = deblurring.GaussianDiffusion(_Net(), device_of_kernel='cpu', sampling_routine=routine, **kw)
        full = gd.sample(batch_size=2, img=x)
        assert all(torch.equal(a, b) for a, b in zip(full, gd.sample(batch_size=2, img=x, steps=8)))
        D = SO.deblur_D(DO.DeblurOracle(net, **kw))
        for K in (1, 3, 4):
            xt, dr, img = gd.sample(batch_size=2, img=x, steps=K)
            _, ref = SO.reverse(net, D(x.double(), 8), 8, K, SO.cold_update(D, routine), 2)
            _check(img, ref, 1e-5)
        gr = resolution.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', channels=3, timesteps=6,
                                          resolution_routine='Incremental', sampling_routine=routine)
        full = gr.sample(batch_size=2, img=x)
        assert all(torch.equal(a, b) for a, b in zip(full, gr.sample(batch_size=2, img=x, steps=6)))
        D = SO.resolution_D(RO.ResolutionOracle(net, image_size=16, channels=3, timesteps=6, resolution_routine='Incremental'))
        for K in (1, 2, 3):
            _, _, img = gr.sample(batch_size=2, img=x, steps=K)
            _, ref = SO.reverse(net, D(x.double(), 6), 6, K, SO.cold_update(D, routine), 2)
            _check(img, ref, 1e-5)


def test_noise_and_fade_strided_loops(emulated):
    from cold_diffusion_models_b200 import denoising, defading_generation
    x = _image()
    gd = denoising.GaussianDiffusion(_Net(), image_size=16, channels=3, timesteps=12)
    full = gd.sample(batch_size=2, img=x)
    assert all(torch.equal(a, b) for a, b in zip(full, gd.sample(batch_size=2, img=x, steps=12)))
    for K in (1, 3, 6):
        _, _, img = gd.sample(batch_size=2, img=x, steps=K)
        _, ref = SO.reverse(net, x.double(), 12, K, SO.noise_update(gd.sqrt_alphas_cumprod, gd.sqrt_one_minus_alphas_cumprod), 2)
        _check(img, ref, 1e-5)
    gf = defading_generation.GaussianDiffusion(_Net(), image_size=16, channels=3, timesteps=6, kernel_std=0.6, initial_mask=3)
    full = gf.sample(batch_size=2, img=x)
    assert all(torch.equal(a, b) for a, b in zip(full, gf.sample(batch_size=2, img=x, steps=6)))
    for K in (1, 3):
        _, _, img = gf.sample(batch_size=2, img=x, steps=K)
        _, ref = SO.reverse(net, x.double(), 6, K, SO.fade_update(gf.alphas, gf.one_minus_alphas, x.double()), 2)
        _check(img, ref, 1e-5)


def test_defading_and_decolor_strided_loops(emulated):
    import defading_oracle as FO
    import snow_oracle as NO
    from cold_diffusion_models_b200 import defading, snowification
    x = _image()
    for routine in ('default', 'x0_step_down'):
        kw = dict(image_size=16, channels=3, timesteps=8, kernel_std=0.1, initial_mask=11, fade_routine='Incremental')
        gd = defading.GaussianDiffusion(_Net(), device_of_kernel='cpu', sampling_routine=routine, **kw)
        full = gd.sample(batch_size=2, faded_recon_sample=x)
        assert all(torch.equal(a, b) for a, b in zip(full, gd.sample(batch_size=2, faded_recon_sample=x, steps=8)))
        D = SO.defading_D(FO.DefadeOracle(net, **kw))
        for K in (1, 3):
            _, _, img = gd.sample(batch_size=2, faded_recon_sample=x, steps=K)
            _, ref = SO.reverse(net, D(x.double(), 8), 8, K, SO.cold_update(D, routine), 2)
            _check(img, ref, 1e-5)
        gs = snowification.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', channels=3, timesteps=6,
                                             forward_process_type='Decolorization', sampling_routine=routine)
        full = gs.sample(batch_size=2, img=x)
        strided = gs.sample(batch_size=2, img=x, steps=6)
        assert all(torch.equal(full[k], strided[k]) for k in full)
        fp = NO.DecolorFP(gs.forward_process.factors)
        fp.w = [w.double() for w in fp.w]
        D = SO.snow_D(fp)
        for K in (1, 2, 3):
            img = gs.sample(batch_size=2, img=x, steps=K)['recon']
            _, ref = SO.reverse(net, D(x.double(), 6), 6, K, SO.snow_update(D, routine), 2)
            _check(img, ref, 1e-5)
