"""GPU checks of the Lab colour path of the snowification / decolor package (`to_lab=True`): cd_lab_convert / cd_chanmix_lab
against the CPU oracle, the package against the vectors recorded from the unmodified reference (tests/golden/snow_lab_small.npz),
the Trainer in the decolor driver's Lab configuration, and the drivers' UnetResNet one-shot model (with_time_emb=False).
The host logic of the same paths is checked on CPU by tests/test_lab_cpu.py."""
import contextlib
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import lab_oracle as LO

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), 'golden')


def load(name):
    z = np.load(os.path.join(G, name + '.npz'))
    return {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def amax(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def stack(lst):
    return torch.stack([x.detach().float().cpu() for x in lst])


def parse_key(key):
    fpt, kws, T, samp = key.split('|')
    kw = {}
    for item in kws.split('-'):
        k, v = item.split('=')
        kw[k] = (v == 'True') if v in ('True', 'False') else (float(v) if '.' in v else (int(v) if v.isdigit() else v))
    return fpt, kw, int(T), samp


@pytest.fixture(scope='module')
def small():
    import cold_diffusion_models_b200 as cdm
    g = load('unet_small')
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
    u.load_state_dict({k[3:]: v for k, v in g.items() if k.startswith('sd:')})
    return u.cuda()


def test_lab_kernels_match_oracle():
    from cold_diffusion_models_b200._lib import call, ptr, stream
    from cold_diffusion_models_b200.snowification import DeColorization
    g = load('snow_lab_small')
    for to_lab, clip, src in ((1, 1, g['conv_rgb']), (0, 1, g['conv_lab_in']), (0, 0, g['conv_lab_in'])):
        ref = LO.rgb2lab(src) if to_lab else LO.lab2rgb(src, clip=bool(clip))
        x = src.cuda().contiguous()
        out = torch.empty_like(x)
        call('cd_lab_convert', ptr(x), ptr(out), 2, C.c_int64(5 * 7), to_lab, clip, stream())
        assert amax(out, ref) < (1e-2 if to_lab else 1e-3), (to_lab, clip)
        call('cd_lab_convert', ptr(x), ptr(x), 2, C.c_int64(5 * 7), to_lab, clip, stream())          # in place
        assert torch.equal(x, out)
    # the step chain: T = 20 'Linear' with total removal (the decolor driver), every index / mode combination, odd sizes
    T, H, W = 20, 7, 9
    mats = DeColorization(num_timesteps=T, decolor_routine='Linear', decolor_total_remove=True, to_lab=True).mats_step
    fp = LO.DecolorLabFP([])
    fp.w = [m[:, :, None, None] for m in mats]
    idx = [-1, 0, 1, 9, T - 1]
    pairs = [(h, l) for h in idx for l in idx]
    B = len(pairs)
    gen = torch.Generator().manual_seed(3)
    xsrc = LO.rgb2lab(torch.rand(B, 3, H, W, generator=gen) * 2 - 1)
    xt = LO.rgb2lab(torch.rand(B, 3, H, W, generator=gen) * 2 - 1)
    chain = torch.empty(T + 1, B, 3, H, W)
    chain[0] = v = xsrc
    for i in range(T):
        v = fp.forward(v, i)
        chain[i + 1] = v                                       # chain[k + 1] = D(x, k), chain[0] = x
    t_hi = torch.tensor([h for h, _ in pairs]) + 1             # offsets -1 / -2 as in sample_one_step
    t_lo = torch.tensor([l for _, l in pairs]) + 2
    for mode in (0, 1):
        ref = torch.stack([chain[h + 1, b] if not mode else xt[b] - chain[h + 1, b] + chain[l + 1, b] for b, (h, l) in enumerate(pairs)])
        out = torch.empty(B, 3, H, W, device='cuda')
        th, tl, xs, xtt, m = t_hi.cuda(), t_lo.cuda(), xsrc.cuda(), xt.cuda(), mats.cuda()
        call('cd_chanmix_lab', ptr(xtt if mode else None), ptr(xs), ptr(out), ptr(m), ptr(th), ptr(tl if mode else None), -1, -2, B,
             C.c_int64(H * W), mode, stream())
        assert amax(out, ref) < 1e-2, mode
        assert torch.equal(out[0].cpu(), xt[0] - xsrc[0] + xsrc[0] if mode else xsrc[0])       # both indices < 0: untouched


def test_lab_package_matches_reference_golden(small):
    from cold_diffusion_models_b200.snowification_diffusion import GaussianDiffusion
    from cold_diffusion_models_b200.snowification_diffusion.utils import rgb2lab, lab2rgb
    g = load('snow_lab_small')
    assert amax(rgb2lab(g['conv_rgb'].cuda()), g['conv_rgb2lab']) < 1e-2
    assert amax(lab2rgb(g['conv_lab_in'].cuda()), g['conv_lab2rgb']) < 1e-3
    assert amax(lab2rgb(g['conv_lab_in'].cuda(), clip=False), g['conv_lab2rgb_noclip']) < 1e-3
    with pytest.raises(RuntimeError):
        rgb2lab(g['conv_rgb'])                                  # CPU tensors raise: no host fallback
    x = g['x'].cuda()
    S = x.shape[-1]
    assert amax(rgb2lab(g['x_rgb'].cuda()), g['x']) < 1e-2
    for key in sorted(k[4:] for k in g if k.startswith('img:')):
        fpt, kw, T, samp = parse_key(key)
        if fpt == 'Snow':
            kw['results_folder'] = '/tmp'
        with contextlib.redirect_stdout(io.StringIO()):
            gd = GaussianDiffusion(small, image_size=(S, S) if fpt == 'Snow' else S, device_of_kernel='cuda', channels=3, timesteps=T,
                                   loss_type='l1', forward_process_type=fpt, train_routine='Final', sampling_routine=samp, to_lab=True,
                                   **kw).cuda()
        assert amax(gd.q_sample(x, torch.tensor([-1, 1]).cuda()), g['q:' + key]) < 1e-2, key
        with torch.no_grad():
            loss = gd.p_losses(x, torch.tensor([T - 1, 1]).cuda()).item()
        # 3e-4 of the RGB tests, relative here: Lab losses are ~45 (L runs 0..100)
        assert abs(loss - g['loss:' + key].item()) < 3e-4 * max(1.0, abs(g['loss:' + key].item())), key
        x1, d1 = gd.sample_one_step(x, torch.tensor([T - 1, 2]).cuda())
        assert rel(d1, g['one_dr:' + key]) < 1e-3 and rel(x1, g['one_x:' + key]) < 2e-3, key
        r = gd.sample(batch_size=2, img=x)
        assert amax(r['xt'], g['xt:' + key]) < 1e-3, key                                     # degradation only, RGB
        assert rel(r['direct_recons'], g['dr:' + key]) < 1e-3 and rel(r['recon'], g['img:' + key]) < 3e-3, key
        if fpt == 'Decolorization':
            assert amax(gd._total_forward(x), g['total:' + key]) < 1e-2, key
        if 'all_X0:' + key in g:
            X0, Xt, _, _ = gd.all_sample(batch_size=2, img=x)
            assert rel(stack(X0), g['all_X0:' + key]) < 4e-3 and rel(stack(Xt), g['all_Xt:' + key]) < 4e-3, key
            F_, B_, img = gd.forward_and_backward(batch_size=2, img=x)
            assert amax(stack(F_), g['fb_F:' + key]) < 1e-2, key                          # degradation only, Lab
            assert rel(stack(B_), g['fb_B:' + key]) < 4e-3 and rel(img, g['fb_img:' + key]) < 4e-3, key


def _args(model, dataset):
    class Args:
        pass
    a = Args()
    a.model, a.dataset = model, dataset
    return a


def test_lab_trainer_decolor_driver_configuration(tmp_path):
    """the decolor driver with --to_lab (Decolorization, Linear, total removal, T = 20) and --model UnetResNet on CIFAR-10-shaped
    synthetic data: two optimizer steps, the periodic sample and the checkpoint at step 1"""
    from cold_diffusion_models_b200 import snowification_diffusion as snp
    args = _args('UnetResNet', 'cifar10_train')
    torch.manual_seed(0)
    model = snp.get_model(args, with_time_emb=True).cuda()
    model_one_shot = snp.get_model(args, with_time_emb=False).cuda()           # train.py:59-60 builds both
    gd = snp.GaussianDiffusion(model, image_size=32, device_of_kernel='cuda', channels=3, timesteps=20, loss_type='l1',
                               one_shot_denoise_fn=model_one_shot, forward_process_type='Decolorization', decolor_routine='Linear',
                               decolor_total_remove=True, train_routine='Final', sampling_routine='x0_step_down', to_lab=True).cuda()
    with contextlib.redirect_stdout(io.StringIO()):
        tr = snp.Trainer(gd, None, train_batch_size=4, train_num_steps=2, gradient_accumulate_every=1, save_and_sample_every=1,
                         results_folder=str(tmp_path), dataset='synthetic', to_lab=True)
    before = model.engine.flat_param.clone()
    with contextlib.redirect_stdout(io.StringIO()):
        tr.train()
    torch.cuda.synchronize()
    assert tr.step == 2 and (model.engine.flat_param - before).abs().max().item() > 0
    assert bool(torch.isfinite(model.engine.flat_param).all())
    for n in ('og', 'recon', 'direct_recons', 'xt'):
        assert (tmp_path / ('sample-%s-1.png' % n)).exists(), n
    ck = torch.load(str(tmp_path / 'model.pt'))
    assert set(ck.keys()) == {'step', 'model', 'ema'} and ck['step'] == 1
    # batches reach the model in Lab space; the periodic sample's outputs are RGB in [-1, 1]
    b = tr._eval_batch()
    assert float(b[:, 0].max()) > 1.5
    r = tr.ema_model.sample(batch_size=4, img=b)
    assert all(float(v.abs().max()) <= 1.0 for v in r.values())


def test_model_without_time_embedding_runs_at_t_zero():
    from cold_diffusion_models_b200 import snowification_diffusion as snp
    args = _args('UnetResNet', 'cifar10_train')
    torch.manual_seed(1)
    m = snp.get_model(args, with_time_emb=False).cuda().eval()
    x = torch.rand(2, 3, 32, 32, device='cuda') * 2 - 1
    with torch.no_grad():
        a = m(x)
        b = m(x, torch.zeros(2, dtype=torch.long, device='cuda'))
    assert torch.equal(a, b)
    m1 = snp.get_model(args, with_time_emb=True).cuda().eval()
    with pytest.raises(ValueError), torch.no_grad():
        m1(x)


def test_one_shot_model_optimizer_step():
    """one Adam step of the UnetResNet one-shot model at 32 x 32, called without t (the time embedding runs at t = 0)"""
    from cold_diffusion_models_b200 import snowification_diffusion as snp
    from cold_diffusion_models_b200.trainer import FusedAdamEMA
    torch.manual_seed(2)
    m = snp.get_model(_args('UnetResNet', 'cifar10_train'), with_time_emb=False).cuda()
    opt = FusedAdamEMA(m.engine, lr=1e-4)
    before = m.engine.flat_param.clone()
    x = torch.rand(2, 3, 32, 32, device='cuda') * 2 - 1
    loss = (m(x) - x).abs().mean()
    loss.backward()
    assert torch.isfinite(loss).item() and m.engine.flat_grad.abs().max().item() > 0
    opt.step()
    torch.cuda.synchronize()
    assert (m.engine.flat_param - before).abs().max().item() > 0 and bool(torch.isfinite(m.engine.flat_param).all())
