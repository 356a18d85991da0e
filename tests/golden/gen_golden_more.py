"""Golden vectors FROM THE UNMODIFIED REFERENCE for the demixing and defading-generation packages and for the deblurring
cover-figure trajectories (forward_and_backward / forward_and_backward_2).  Needs a checkout of the reference
($COLD_REF_ROOT, see oracle/ref_shim.py).  Reuses the small Unet weights stored in unet_small.npz so the existing fixtures stay untouched.

    python tests/golden/gen_golden_more.py     ->  tests/golden/{demixing_small,defading_gen_small,fb_small}.npz
"""
import os, sys
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, HERE)
import ref_shim  # noqa
from gen_golden import quiet, save  # noqa


def small_sd():
    z = np.load(os.path.join(HERE, 'unet_small.npz'))
    return {k[3:]: torch.from_numpy(np.asarray(z[k])) for k in z.files if k.startswith('sd:')}


def stack(lst):
    return torch.stack([x.detach().cpu() for x in lst])


def main():
    torch.set_num_threads(8)
    ref_shim.patch_cuda_noop()
    sd = small_sd()

    # ---- demixing ------------------------------------------------------------------------------------------
    dm = ref_shim.import_reference('demixing-diffusion-pytorch', 'demixing_diffusion_pytorch')
    unet = quiet(dm.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet.load_state_dict(sd)
    torch.manual_seed(51)
    x1 = torch.rand(2, 3, 32, 32) * 2 - 1
    x2 = torch.rand(2, 3, 32, 32) * 2 - 1
    gd = dm.GaussianDiffusion(unet, image_size=32, channels=3, timesteps=5, loss_type='l1')
    out = {}
    tt = torch.tensor([4, 1])
    out['q'] = gd.q_sample(x1, x2, tt)
    with torch.no_grad():
        out['loss'] = gd.p_losses(x1, x2, tt)
    _, out['gen_dr'], out['gen_img'] = quiet(gd.gen_sample, batch_size=2, img=x2, noise_level=0)
    _, out['sample_dr'], out['sample_img'] = quiet(gd.sample, batch_size=2, img=x2)
    F_, B_, img = quiet(gd.forward_and_backward, batch_size=2, img1=x1, img2=x2)
    out['fb_F'], out['fb_B'], out['fb_img'] = stack(F_), stack(B_), img
    X1, Xt = quiet(gd.all_sample, batch_size=2, img=x2)
    out['all_X1'], out['all_Xt'] = stack(X1), stack(Xt)
    save('demixing_small', x1=x1, x2=x2, **out)

    # ---- defading generation -------------------------------------------------------------------------------
    dg = ref_shim.import_reference('defading-generation-diffusion-pytorch', 'defading_diffusion_pytorch')
    unet = quiet(dg.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet.load_state_dict(sd)
    torch.manual_seed(61)
    x1 = torch.rand(2, 3, 32, 32) * 2 - 1
    col = (torch.rand(2, 3) - 0.5)[:, :, None, None].expand(2, 3, 32, 32).contiguous()
    out = {}
    for rev in (False, True):
        gd = dg.GaussianDiffusion(unet, image_size=32, channels=3, timesteps=4, loss_type='l1', reverse=rev, kernel_std=0.6,
                                  initial_mask=3)
        k = 'rev%d:' % int(rev)
        tt = torch.tensor([3, 0])
        out[k + 'alphas'], out[k + 'one_minus_alphas'] = gd.alphas, gd.one_minus_alphas
        out[k + 'q'] = gd.q_sample(x1, col, tt)
        with torch.no_grad():
            out[k + 'loss'] = gd.p_losses(x1, col, tt)
        _, out[k + 'sample_dr'], out[k + 'sample_img'] = quiet(gd.sample, batch_size=2, img=col)
        _, out[k + 'gen_dr'], out[k + 'gen_img'] = quiet(gd.gen_sample, batch_size=2, img=col, noise_level=0)
        F_, B_, img = quiet(gd.forward_and_backward, batch_size=2, img1=x1, img2=col)
        out[k + 'fb_F'], out[k + 'fb_B'], out[k + 'fb_img'] = stack(F_), stack(B_), img
        X1, Xt = quiet(gd.all_sample, batch_size=2, img=col)
        out[k + 'all_X1'], out[k + 'all_Xt'] = stack(X1), stack(Xt)
    save('defading_gen_small', x1=x1, col=col, **out)

    # ---- deblurring cover-figure trajectories --------------------------------------------------------------
    db = ref_shim.import_reference('deblurring-diffusion-pytorch', 'deblurring_diffusion_pytorch')
    unet = quiet(db.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet.load_state_dict(sd)
    torch.manual_seed(71)
    x = torch.rand(2, 3, 32, 32) * 2 - 1
    out = {}
    for routine, ks, std, T, samp in [('Exponential_reflect', 7, 0.15, 4, 'x0_step_down'), ('Constant', 5, 1.0, 3, 'default')]:
        gd = db.GaussianDiffusion(unet, image_size=32, device_of_kernel='cpu', channels=3, timesteps=T, kernel_std=std,
                                  kernel_size=ks, blur_routine=routine, sampling_routine=samp)
        key = '%s|%d|%g|%d|%s' % (routine, ks, std, T, samp)
        F_, B_, img = quiet(gd.forward_and_backward, batch_size=2, img=x)
        out['F:' + key], out['B:' + key], out['img:' + key] = stack(F_), stack(B_), img
        F2, B1, B2, i1, i2 = quiet(gd.forward_and_backward_2, batch_size=2, img=x)
        out['F2:' + key], out['B1:' + key], out['B2:' + key], out['i1:' + key], out['i2:' + key] = stack(F2), stack(B1), stack(B2), i1, i2
        for start in (0, 1):
            xt, dr, img2 = quiet(gd.sample_from_blur, batch_size=2, img=x, start=start)
            out['sfb_xt:%d:' % start + key], out['sfb_dr:%d:' % start + key], out['sfb_img:%d:' % start + key] = xt, dr, img2
        X0s, Xts = quiet(gd.all_sample, batch_size=2, img=x)
        out['all_X0:' + key], out['all_Xt:' + key] = stack(X0s), stack(Xts)
        torch.manual_seed(17)
        xt, dr, img3 = quiet(gd.gen_sample, batch_size=2, img=x, noise_level=0.05)
        out['gen_xt:' + key], out['gen_img:' + key] = xt, img3
    save('fb_small', x=x, **out)

    # ---- the seventh blur routine, 'Individual_Incremental' (kernel size 2i+1, sigma 2k, DB:379-383): q_sample + sample ----
    torch.manual_seed(91)
    xi = torch.rand(2, 3, 32, 32) * 2 - 1
    out = {}
    for samp in ('default', 'x0_step_down'):
        gd = db.GaussianDiffusion(unet, image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, kernel_std=0.1, kernel_size=3,
                                  blur_routine='Individual_Incremental', sampling_routine=samp)
        if samp == 'default':
            for i, kconv in enumerate(gd.gaussian_kernels):
                out['w%d' % i] = kconv.weight[0, 0]
            out['q'] = gd.q_sample(xi, torch.tensor([3, 1]))
            with torch.no_grad():
                out['loss'] = gd.p_losses(xi, torch.tensor([3, 1]))
        xt, dr, img = quiet(gd.sample, batch_size=2, img=xi)
        out['xt:' + samp], out['dr:' + samp], out['img:' + samp] = xt, dr, img
    save('individual_small', x=xi, **out)

    # ---- resolution package: the six train routines of p_losses (RS:655-761), incl. the t = 0 row of 'Step' (RS:645 quirk) ----
    rs = ref_shim.import_reference('resolution-diffusion-pytorch', 'resolution_diffusion_pytorch')
    unet_rs = quiet(rs.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet_rs.load_state_dict(sd)
    torch.manual_seed(95)
    xr = torch.rand(3, 3, 32, 32) * 2 - 1
    out = {}
    # ('Gradient_norm' raises inside torch.linalg.norm(dim=(1,2,3)) in the reference: no golden)
    for routine in ('Final', 'Final_small_noise', 'Final_random_mean', 'Final_random_mean_and_actual', 'Step'):
        for lt in ('l1', 'l2'):
            gd = rs.GaussianDiffusion(unet_rs, image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, loss_type=lt,
                                      resolution_routine='Incremental_factor_2', train_routine=routine, sampling_routine='x0_step_down')
            torch.manual_seed(7)
            with torch.no_grad():
                out['loss:%s|%s' % (routine, lt)] = gd.p_losses(xr, torch.tensor([3, 0, 2]))
    out['q_neg'] = gd.q_sample(xr, torch.tensor([2, -1, 1]))
    out['func1'] = gd.func[1](xr); out['func2of1'] = gd.func[2](out['func1'])
    out['tf_bilinear5'] = gd.transform_func(xr, 5, 'bilinear'); out['tf_area16_blur'] = gd.transform_func(xr, 16, 'area', do_blur=True)
    for samp in ('x0_step_down', 'default'):
        gd = rs.GaussianDiffusion(unet_rs, image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, loss_type='l1',
                                  resolution_routine='Incremental_factor_2', train_routine='Final', sampling_routine=samp)
        xdeg = gd.opt(xr)
        torch.manual_seed(23)
        xt, dr, img = quiet(gd.gen_sample, batch_size=3, img=xdeg, noise_level=0.02)
        out['gen_xt:' + samp], out['gen_dr:' + samp], out['gen_img:' + samp] = xt, dr, img
        X0s, Xts = quiet(gd.all_sample, batch_size=3, img=xr)
        out['all_X0:' + samp], out['all_Xt:' + samp] = stack(X0s), stack(Xts)
        F_, B_, img = quiet(gd.forward_and_backward, batch_size=3, img=xr)
        out['fb_F:' + samp], out['fb_B:' + samp], out['fb_img:' + samp] = stack(F_), stack(B_), img
    save('resolution_train_small', x=xr, **out)

    # ---- Unet constructor options used by the drivers' flags (--residual, --remove_time_embed) and out_dim (DB:192-200) ----
    out = {}
    torch.manual_seed(103)
    xo = torch.rand(2, 3, 32, 32) * 2 - 1
    to = torch.tensor([1, 6])
    tgt5 = torch.rand(2, 5, 32, 32) * 2 - 1
    for tag, kw in (('residual', dict(residual=True)), ('notime', dict(with_time_emb=False)), ('outdim', dict(out_dim=5))):
        torch.manual_seed(0)
        uo = quiet(db.Unet, dim=32, dim_mults=(1, 2), channels=3, **kw)
        own = uo.state_dict()                      # weights: unet_small.npz wherever the key and shape exist there
        uo.load_state_dict({k: (sd[k] if k in sd and sd[k].shape == v.shape else v) for k, v in own.items()})
        y = uo(xo, to)
        target = tgt5 if tag == 'outdim' else xo.flip(0)
        loss = ((target - y) ** 2).mean()
        loss.backward()
        out[tag + ':y'], out[tag + ':loss'] = y.detach(), loss.detach()
        for n, p_ in uo.state_dict().items():
            if n not in sd or sd[n].shape != p_.shape:
                out[tag + ':sd:' + n] = p_.clone()         # only what unet_small.npz does not hold (the out_dim = 5 projection)
        for n, p_ in uo.named_parameters():
            g_ = p_.grad.reshape(-1)
            out[tag + ':gnorm:' + n] = g_.double().norm().float()
            out[tag + ':gsub:' + n] = g_[::max(1, g_.numel() // 256)].clone()
    save('unet_options_small', x=xo, t=to, tgt5=tgt5, **out)

    # ---- denoising baseline: all_sample (DN:474-515) and forward_and_backward (DN:437-472; noise drawn inside: seeded) -------
    dn = ref_shim.import_reference('denoising-diffusion-pytorch', 'denoising_diffusion_pytorch')
    unet_dn = quiet(dn.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet_dn.load_state_dict(sd)
    torch.manual_seed(101)
    xd = torch.rand(2, 3, 32, 32) * 2 - 1
    nd = torch.randn(2, 3, 32, 32)
    gd = dn.GaussianDiffusion(unet_dn, image_size=32, channels=3, timesteps=5, loss_type='l1')
    out = {}
    X1, X2, Xt = quiet(gd.all_sample, batch_size=2, img=nd)
    out['all_X1'], out['all_X2'], out['all_Xt'] = stack(X1), stack(X2), stack(Xt)
    torch.manual_seed(29)
    F_, B_, img = quiet(gd.forward_and_backward, batch_size=2, img=xd)
    out['fb_F'], out['fb_B'], out['fb_img'] = stack(F_), stack(B_), img
    save('denoise_more_small', x=xd, noise=nd, **out)

    # ---- defading all_sample (DFG:428-494) and snowification all_sample / forward_and_backward (SN:299-339, 450-490) -----------
    df = ref_shim.import_reference('defading-diffusion-pytorch', 'defading_diffusion_pytorch')
    unet_df = quiet(df.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet_df.load_state_dict(sd)
    torch.manual_seed(97)
    xf = torch.rand(2, 3, 32, 32) * 2 - 1
    out = {}
    for routine, T, samp in [('Incremental', 4, 'x0_step_down'), ('Constant', 3, 'default'), ('Random_Incremental', 4, 'x0_step_down')]:
        gd = df.GaussianDiffusion(unet_df, image_size=32, device_of_kernel='cpu', channels=3, timesteps=T, loss_type='l1',
                                  kernel_std=0.6, initial_mask=3, fade_routine=routine, sampling_routine=samp)
        key = '%s|%d|%s' % (routine, T, samp)
        torch.manual_seed(78)
        out['rx:' + key] = torch.randint(0, 33, (2,)); out['ry:' + key] = torch.randint(0, 33, (2,))
        torch.manual_seed(78)
        x0l, xtl = quiet(gd.all_sample, batch_size=2, faded_recon_sample=xf)
        out['x0:' + key], out['xt:' + key] = stack(x0l), stack(xtl)
    save('defading_all_small', x=xf, **out)

    sn = ref_shim.import_reference('snowification', 'diffusion')
    unet_sn = quiet(db.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet_sn.load_state_dict(sd)
    torch.manual_seed(99)
    xs = torch.rand(3, 3, 32, 32) * 2 - 1
    out = {}
    for fpt, kw, T, samp in [('Decolorization', dict(decolor_routine='Linear', decolor_total_remove=True), 5, 'x0_step_down'),
                             ('Decolorization', dict(decolor_routine='Constant', decolor_ema_factor=0.8, decolor_total_remove=False), 4, 'default'),
                             ('Snow', dict(snow_level=1, results_folder='/tmp'), 4, 'x0_step_down')]:
        gd = quiet(sn.GaussianDiffusion, unet_sn, image_size=(32, 32) if fpt == 'Snow' else 32, device_of_kernel='cpu', channels=3,
                   timesteps=T, loss_type='l1', forward_process_type=fpt, train_routine='Final', sampling_routine=samp, **kw)
        key = '%s|%s|%d|%s' % (fpt, '-'.join('%s=%s' % (k, v) for k, v in sorted(kw.items()) if k != 'results_folder'), T, samp)
        if fpt == 'Decolorization':
            X0, Xt, _, _ = quiet(gd.all_sample, batch_size=3, img=xs)
            out['all_X0:' + key], out['all_Xt:' + key] = stack(X0), stack(Xt)
        F_, B_, img = quiet(gd.forward_and_backward, batch_size=3, img=xs)
        out['fb_F:' + key], out['fb_B:' + key], out['fb_img:' + key] = stack(F_), stack(B_), img
        if fpt == 'Decolorization':
            xq = gd.q_sample(xs, torch.tensor([T - 1, 1, 2]))
            out['ms:' + key] = quiet(gd.sample_multi_step, xq, torch.tensor([T - 1, 1, 2]), torch.tensor([1, 1, 0]))
    save('snow_more_small', x=xs, **out)

    # ---- checkpoint wire format: state_dict keys and shapes of every package's GaussianDiffusion (+ Model) ------------------
    import json
    fmt = {}

    def record(tag, module):
        fmt[tag] = {k: list(v.shape) for k, v in module.state_dict().items()}
    mk = lambda mod: quiet(mod.Unet, dim=32, dim_mults=(1, 2), channels=3)
    record('deblurring', db.GaussianDiffusion(mk(db), image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, kernel_std=0.15,
                                              kernel_size=7, blur_routine='Exponential_reflect'))
    record('deblurring_model', db.GaussianDiffusion(db.Model(resolution=16, in_channels=3, out_ch=3, ch=32, ch_mult=(1, 2), num_res_blocks=2,
                                                             attn_resolutions=(8,), dropout=0.1), image_size=16, device_of_kernel='cpu',
                                                    channels=3, timesteps=3, kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine'))
    record('resolution', rs.GaussianDiffusion(mk(rs), image_size=32, device_of_kernel='cpu', channels=3, timesteps=4,
                                              resolution_routine='Incremental_factor_2'))
    record('defading', df.GaussianDiffusion(mk(df), image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, kernel_std=0.6,
                                            initial_mask=3, fade_routine='Incremental'))
    record('denoising', dn.GaussianDiffusion(mk(dn), image_size=32, channels=3, timesteps=5))
    record('demixing', dm.GaussianDiffusion(mk(dm), image_size=32, channels=3, timesteps=5))
    record('defading_generation', dg.GaussianDiffusion(mk(dg), image_size=32, channels=3, timesteps=4, kernel_std=0.6, initial_mask=3))
    record('decolor', quiet(sn.GaussianDiffusion, mk(db), image_size=32, device_of_kernel='cpu', channels=3, timesteps=4,
                            forward_process_type='Decolorization', decolor_routine='Linear'))
    with open(os.path.join(HERE, 'state_dict_format.json'), 'w') as f:
        json.dump(fmt, f, indent=0, sort_keys=True)
    print('wrote state_dict_format.json', sum(len(v) for v in fmt.values()), 'keys')

    # ---- API surface: constructor / method signatures of every exported class ---------------------------------------------
    import inspect

    def sig(fn):
        out_ = []
        for n, p_ in inspect.signature(fn).parameters.items():
            if n == 'self':
                continue
            d = None if p_.default is inspect._empty else repr(p_.default)
            out_.append([n, str(p_.kind), d])
        return out_
    api = {}
    for tag, mod, names in (('deblurring', db, ('Unet', 'GaussianDiffusion', 'Trainer', 'Model')), ('resolution', rs, ('Unet', 'GaussianDiffusion', 'Trainer')),
                            ('defading', df, ('Unet', 'GaussianDiffusion', 'Trainer')), ('denoising', dn, ('Unet', 'GaussianDiffusion', 'Trainer')),
                            ('demixing', dm, ('Unet', 'GaussianDiffusion', 'Trainer')), ('defading_generation', dg, ('Unet', 'GaussianDiffusion', 'Trainer')),
                            ('snowification', sn, ('GaussianDiffusion', 'Trainer'))):
        for cn in names:
            cls = getattr(mod, cn)
            entry = {'__init__': sig(cls.__init__)}
            if cn == 'GaussianDiffusion':
                for mn, fn in inspect.getmembers(cls, predicate=inspect.isfunction):
                    if not mn.startswith('_'):
                        entry[mn] = sig(fn)
            api[tag + '.' + cn] = entry
    with open(os.path.join(HERE, 'api_surface.json'), 'w') as f:
        json.dump(api, f, indent=0, sort_keys=True)
    print('wrote api_surface.json', len(api), 'classes')

    # ---- DDPM-style `Model` (Model2.py): L1-loss gradients of every parameter (dropout inactive: eval mode) -----------
    z = np.load(os.path.join(HERE, 'model2_small.npz'))
    msd = {k[3:]: torch.from_numpy(np.asarray(z[k])) for k in z.files if k.startswith('sd:')}
    model = db.Model(resolution=16, in_channels=3, out_ch=3, ch=32, ch_mult=(1, 2), num_res_blocks=2, attn_resolutions=(8,),
                     dropout=0.1).eval()
    model.load_state_dict(msd)
    xm, tm = torch.from_numpy(np.asarray(z['x'])), torch.from_numpy(np.asarray(z['t']))
    torch.manual_seed(81)
    target = torch.rand(3, 3, 16, 16) * 2 - 1
    y = model(xm, tm)
    loss = (target - y).abs().mean()
    loss.backward()
    grads = {}
    for n, p_ in model.named_parameters():
        g = p_.grad.reshape(-1)
        if g.numel() <= 4096:
            grads['grad:' + n] = p_.grad.clone()
        else:
            stride = g.numel() // 2048
            grads['gsub:' + n] = g[::stride].clone()
            grads['gnorm:' + n] = g.double().norm().float()
    loss2 = ((target - y) ** 2).mean()
    save('model2_grads_small', target=target, loss=loss.detach(), loss_l2=loss2.detach(), **grads)


if __name__ == '__main__':
    main()
