"""The Lab colour path of the snowification / decolor package (`to_lab=True`) on the CPU:
  * tests/lab_oracle.py's restatement of rgb2lab / lab2rgb / the Lab decolorization step against the vectors recorded from the
    unmodified reference (tests/golden/snow_lab_small.npz), and against an fp64 run of itself;
  * the CUDA source of cd_lab_convert / cd_chanmix_lab (csrc/degrade.cu, compiled for the CPU by tests/simt_cpu) against the oracle;
  * the package's host logic (GaussianDiffusion / Trainer with to_lab) on CPU tensors through tests/abi_emulator.py (with the two
    entry points of tests/lab_oracle.py added) against the golden;
  * get_model('UnetResNet', with_time_emb=False): the drivers' one-shot model."""
import contextlib
import ctypes as C
import io
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))
import abi_emulator as E  # noqa: E402
import lab_oracle as LO  # noqa: E402
import snow_oracle as SO  # noqa: E402

G = os.path.join(os.path.dirname(__file__), 'golden')


def load(name):
    z = np.load(os.path.join(G, name + '.npz'))
    return {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def stack(lst):
    return torch.stack([x.detach().float().cpu() for x in lst])


def P(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def parse_key(key):
    fpt, kws, T, samp = key.split('|')
    kw = {}
    for item in kws.split('-'):
        k, v = item.split('=')
        kw[k] = (v == 'True') if v in ('True', 'False') else (float(v) if '.' in v else (int(v) if v.isdigit() else v))
    return fpt, kw, int(T), samp


def decolor_keys(g):
    return sorted(k[2:] for k in g if k.startswith('q:') and k[2:].startswith('Decolorization'))


def oracle_chain(x, mats, k):
    """D(x, k) of the Lab decolorization: steps 0..k of rgb2lab(M_i lab2rgb(.)); k < 0 = x"""
    fp = LO.DecolorLabFP([])
    fp.w = [m[:, :, None, None] for m in mats]
    for i in range(k + 1):
        x = fp.forward(x, i)
    return x


# ---- oracle ---------------------------------------------------------------------------------------------------------------
def test_oracle_conversions_match_reference_golden():
    g = load('snow_lab_small')
    assert torch.allclose(LO.rgb2lab(g['conv_rgb']), g['conv_rgb2lab'], atol=1e-4)
    assert torch.allclose(LO.lab2rgb(g['conv_lab_in']), g['conv_lab2rgb'], atol=1e-6)
    assert torch.allclose(LO.lab2rgb(g['conv_lab_in'], clip=False), g['conv_lab2rgb_noclip'], atol=1e-5)
    assert torch.allclose(LO.lab2rgb(LO.rgb2lab(g['conv_rgb'].clamp(-1, 1))), g['conv_roundtrip'], atol=1e-6)
    assert torch.allclose(g['conv_roundtrip'], g['conv_rgb'].clamp(-1, 1), atol=3e-4)        # lab2rgb(rgb2lab(x)) == x
    # the out-of-gamut inputs reach the fz clamp and the clip
    lab = g['conv_lab_in']
    assert bool(((lab[:, 0] + 16) / 116 - lab[:, 2] / 200 < 0).any())
    assert bool((g['conv_lab2rgb_noclip'].abs() > 1).any()) and float(g['conv_lab2rgb'].abs().max()) <= 1.0


def test_oracle_decolor_steps_match_reference_golden():
    from cold_diffusion_models_b200.snowification import DeColorization
    g = load('snow_lab_small')
    for key in decolor_keys(g):
        fpt, kw, T, samp = parse_key(key)
        dc = DeColorization(num_timesteps=T, to_lab=True, **kw)
        fp = LO.DecolorLabFP(dc.factors)
        o = SO.SnowOracle(None, fp, timesteps=T)
        assert torch.allclose(o.q_sample(g['x'], torch.tensor([-1, 1])), g['q:' + key], atol=1e-4), key
        assert torch.allclose(fp.total_forward(g['x']), g['total:' + key], atol=1e-4), key


def test_oracle_fp32_chain_stays_close_to_fp64():
    """T = 20 'Linear' with total removal (the decolor driver's Lab configuration): fp32 within 3e-4 Lab units of fp64"""
    from cold_diffusion_models_b200.snowification import DeColorization
    torch.manual_seed(5)
    x = LO.rgb2lab(torch.rand(2, 3, 16, 16) * 2 - 1)
    fp = LO.DecolorLabFP(DeColorization(num_timesteps=20, decolor_routine='Linear', decolor_total_remove=True).factors)
    a, b = x.clone(), x.double()
    for i in range(20):
        a, b = fp.forward(a, i), fp.forward(b, i)
        assert float((a.double() - b).abs().max()) < 3e-4, i


# ---- kernel sources on the CPU --------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def cpulib():
    import build
    return C.CDLL(build.build_all())


def _lab_image(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return LO.rgb2lab(torch.rand(B, 3, H, W, generator=g) * 2 - 1).contiguous()


@pytest.mark.parametrize('to_lab,clip', [(1, 1), (0, 1), (0, 0)])
def test_lab_convert_source_against_oracle(cpulib, to_lab, clip):
    g = load('snow_lab_small')
    src = (g['conv_rgb'] if to_lab else g['conv_lab_in']).contiguous()             # 2 x 3 x 5 x 7: odd sizes
    ref = LO.rgb2lab(src) if to_lab else LO.lab2rgb(src, clip=bool(clip))
    tol = 2e-4 if to_lab else 2e-6
    for impl in (cpulib.cd_lab_convert, LO.cd_lab_convert):
        out = torch.full_like(src, 7.0)
        assert impl(P(src), P(out), 2, C.c_int64(5 * 7), to_lab, clip, None) == 0
        assert float((out - ref).abs().max()) < tol
        inplace = src.clone()                                                       # out == x
        assert impl(P(inplace), P(inplace), 2, C.c_int64(5 * 7), to_lab, clip, None) == 0
        assert torch.equal(inplace, out)


@pytest.mark.parametrize('mode', [0, 1])
def test_chanmix_lab_source_against_oracle(cpulib, mode):
    """every combination of per-sample indices (below 0, 0, middle, last) and offsets, odd image sizes; mode 1 = xt - hi + lo"""
    from cold_diffusion_models_b200.snowification import DeColorization
    T, H, W = 6, 5, 7
    mats = DeColorization(num_timesteps=T, decolor_routine='Linear', decolor_total_remove=True, to_lab=True).mats_step.contiguous()
    idx = [-1, 0, 1, 3, T - 1]
    pairs = [(h, l) for h in idx for l in idx] if mode else [(h, -1) for h in idx]
    B = len(pairs)
    xsrc = _lab_image(B, H, W, 11 + mode)
    xt = _lab_image(B, H, W, 23)
    for hi_off, lo_off in ((0, 0), (-1, -2)):
        t_hi = torch.tensor([h - hi_off for h, _ in pairs], dtype=torch.int64)
        t_lo = torch.tensor([l - lo_off for _, l in pairs], dtype=torch.int64)
        ref = torch.empty_like(xsrc)
        for b, (h, l) in enumerate(pairs):
            hv = oracle_chain(xsrc[b:b + 1], mats, h)
            ref[b] = (xt[b:b + 1] - hv + oracle_chain(xsrc[b:b + 1], mats, l))[0] if mode else hv[0]
        for impl in (cpulib.cd_chanmix_lab, LO.cd_chanmix_lab):
            out = torch.full_like(xsrc, 7.0)
            rc = impl(P(xt if mode else None), P(xsrc), P(out), P(mats), P(t_hi), P(t_lo if mode else None), hi_off, lo_off, B,
                      C.c_int64(H * W), mode, None)
            assert rc == 0
            assert float((out - ref).abs().max()) < 2e-3, (impl, hi_off)
            for b, (h, l) in enumerate(pairs):                   # index < 0: the input itself, no conversion round trip
                if h < 0 and (not mode or l < 0):
                    assert torch.equal(out[b], xt[b] - xsrc[b] + xsrc[b] if mode else xsrc[b])


# ---- package host logic through the ABI emulator --------------------------------------------------------------------------
@pytest.fixture()
def unet(monkeypatch):
    import cold_diffusion_models_b200 as cdm
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)
    g = load('unet_small')
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
    u.load_state_dict({k[3:]: v for k, v in g.items() if k.startswith('sd:')})
    LO.install_emulator()
    with E.patched():
        yield u


def test_package_conversions(unet):
    from cold_diffusion_models_b200.snowification_diffusion.utils import rgb2lab, lab2rgb
    g = load('snow_lab_small')
    assert float((rgb2lab(g['conv_rgb']) - g['conv_rgb2lab']).abs().max()) < 2e-4
    assert float((lab2rgb(g['conv_lab_in']) - g['conv_lab2rgb']).abs().max()) < 1e-5
    assert float((lab2rgb(g['conv_lab_in'], clip=False) - g['conv_lab2rgb_noclip']).abs().max()) < 1e-5
    assert rgb2lab(g['conv_rgb'][0]).shape == (3, 5, 7)
    with pytest.raises(ValueError):
        lab2rgb(torch.zeros(2, 4, 3, 3))


def test_package_lab_path_matches_reference_golden(unet):
    from cold_diffusion_models_b200.snowification_diffusion import GaussianDiffusion
    g = load('snow_lab_small')
    x = g['x']
    S = x.shape[-1]
    for key in sorted(k[4:] for k in g if k.startswith('img:')):
        fpt, kw, T, samp = parse_key(key)
        if fpt == 'Snow':
            kw['results_folder'] = '/tmp'
        with contextlib.redirect_stdout(io.StringIO()):
            gd = GaussianDiffusion(unet, image_size=(S, S) if fpt == 'Snow' else S, device_of_kernel='cpu', channels=3, timesteps=T,
                                   loss_type='l1', forward_process_type=fpt, train_routine='Final', sampling_routine=samp, to_lab=True, **kw)
        q = gd.q_sample(x, torch.tensor([-1, 1]))
        assert float((q - g['q:' + key]).abs().max()) < 2e-3, key
        with torch.no_grad():
            assert abs(gd.p_losses(x, torch.tensor([T - 1, 1])).item() - g['loss:' + key].item()) < 1e-4 * max(1.0, g['loss:' + key].item()), key
        x1, d1 = gd.sample_one_step(x, torch.tensor([T - 1, 2]))
        assert rel(d1, g['one_dr:' + key]) < 1e-5 and rel(x1, g['one_x:' + key]) < 1e-4, key
        r = gd.sample(batch_size=2, img=x)
        assert float((r['xt'] - g['xt:' + key]).abs().max()) < 1e-3, key                  # RGB in [-1, 1]
        assert rel(r['direct_recons'], g['dr:' + key]) < 1e-4 and rel(r['recon'], g['img:' + key]) < 1e-4, key
        if fpt == 'Decolorization':
            assert float((gd._total_forward(x) - g['total:' + key]).abs().max()) < 2e-3, key
        if 'all_X0:' + key in g:
            X0, Xt, ip, fl = gd.all_sample(batch_size=2, img=x)
            assert ip is None and fl == [] and len(X0) == T
            assert rel(stack(X0), g['all_X0:' + key]) < 1e-4 and rel(stack(Xt), g['all_Xt:' + key]) < 1e-4, key
            F_, B_, img = gd.forward_and_backward(batch_size=2, img=x)
            assert float((stack(F_) - g['fb_F:' + key]).abs().max()) < 2e-3, key
            assert rel(stack(B_), g['fb_B:' + key]) < 1e-4 and rel(img, g['fb_img:' + key]) < 1e-4, key


def test_lab_trainer_loop_converts_batches_and_outputs(unet, tmp_path):
    """SnowificationTrainer(to_lab=True): the training batches reach the model as Lab, `og` is saved after lab2rgb, two steps with
    a sample and a checkpoint at step 1 (SN:709-760)"""
    import copy
    from cold_diffusion_models_b200 import snowification_diffusion as snp
    gd = snp.GaussianDiffusion(copy.deepcopy(unet), image_size=32, device_of_kernel='cpu', channels=3, timesteps=4,
                               forward_process_type='Decolorization', decolor_routine='Linear', decolor_total_remove=True,
                               sampling_routine='x0_step_down', to_lab=True)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = snp.Trainer(gd, None, train_batch_size=2, train_num_steps=2, gradient_accumulate_every=1, save_and_sample_every=1,
                         results_folder=str(tmp_path), dataset='synthetic', to_lab=True)
    seen = []
    real = gd.forward
    gd.forward = lambda d, *a, **k: (seen.append(d.clone()), real(d, *a, **k))[1]
    batch = torch.rand(2, 3, 32, 32) * 2 - 1
    tr.train_step(batches=[batch])
    assert torch.allclose(seen[-1], LO.rgb2lab(batch), atol=2e-4)
    assert float(tr._eval_batch()[:, 0].min()) >= -1e-3                                  # L channel: Lab, not [-1, 1]
    with contextlib.redirect_stdout(io.StringIO()):
        tr.train()
    assert tr.step == 2
    for n in ('og', 'recon', 'direct_recons', 'xt'):
        assert (tmp_path / ('sample-%s-1.png' % n)).exists(), n
    ck = torch.load(str(tmp_path / 'model.pt'))
    assert set(ck.keys()) == {'step', 'model', 'ema'} and ck['step'] == 1


# ---- the drivers' one-shot model ----------------------------------------------------------------------------------------
def test_get_model_unet_resnet_without_time_embedding():
    from cold_diffusion_models_b200.snowification_diffusion import get_model
    from cold_diffusion_models_b200 import Model

    class Args:
        model, dataset = 'UnetResNet', 'cifar10_train'
    m0, m1 = get_model(Args(), with_time_emb=False), get_model(Args())
    assert isinstance(m0, Model) and m0.with_time_emb is False and m1.with_time_emb is True
    assert list(m0.state_dict().keys()) == list(m1.state_dict().keys())
    assert all(m0.state_dict()[k].shape == v.shape for k, v in m1.state_dict().items())
    m0.load_state_dict(m1.state_dict())                                                  # checkpoints load either way
    Args.dataset = 'celebA_train'
    assert get_model(Args(), with_time_emb=False).resolution == 128
