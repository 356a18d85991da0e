"""Generate golden vectors FROM THE UNMODIFIED REFERENCE (needs a checkout of the reference, found by oracle/ref_shim.py via
$COLD_REF_ROOT).  Output: tests/golden/*.npz (committed).

    python tests/golden/gen_golden.py            # every golden of this script
    python tests/golden/gen_golden.py config1    # config1_mnist_loss.npz only
"""
import os, sys, io, contextlib
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import ref_shim  # noqa


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def save(name, **arrs):
    out = {}
    for k, v in arrs.items():
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().numpy()
        out[k] = v
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print('wrote', name, sum(np.asarray(v).nbytes for v in out.values()) // 1024, 'KiB')


def gen_config1_mnist_loss():
    """BASELINE config 1 (MNIST-shaped 1x32x32, T=20, k=11, sigma=7, Constant, B=4, full-size Unet): the reference's p_losses on
    its Unet initialised under torch.manual_seed(0).  tests/test_oracle_golden.py rebuilds those weights with the package's Unet
    under the same seed; that both draw identical parameters is asserted here."""
    m = ref_shim.import_reference('deblurring-diffusion-pytorch', 'deblurring_diffusion_pytorch')
    torch.manual_seed(0)
    unet = quiet(m.Unet, dim=64, dim_mults=(1, 2, 4, 8), channels=1)
    gd = m.GaussianDiffusion(unet, image_size=32, device_of_kernel='cpu', channels=1, timesteps=20,
                             kernel_std=7.0, kernel_size=11, blur_routine='Constant', loss_type='l1')
    torch.manual_seed(1234)
    x = torch.rand(4, 1, 32, 32) * 2 - 1
    t = torch.randint(0, 20, (4,))
    with torch.no_grad():
        ref_loss = gd.p_losses(x, t)
    sys.path.insert(0, ROOT)
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(0)
    ours = quiet(cdm.Unet, dim=64, dim_mults=(1, 2, 4, 8), channels=1).state_dict()
    theirs = unet.state_dict()
    assert set(ours) == set(theirs) and all(torch.equal(ours[k], theirs[k]) for k in theirs), "Unet initialisations differ"
    save('config1_mnist_loss', x=x, t=t, ref_loss=np.float64(ref_loss.item()))


def main():
    torch.set_num_threads(8)
    ref_shim.patch_cuda_noop()
    m = ref_shim.import_reference('deblurring-diffusion-pytorch', 'deblurring_diffusion_pytorch')

    # ---- (1) small ConvNeXt Unet: forward, L1 loss, gradients -------------------------
    torch.manual_seed(0)
    unet = quiet(m.Unet, dim=32, dim_mults=(1, 2), channels=3)
    # make LayerNorm affine / biases non-trivial so every term is exercised
    with torch.no_grad():
        for n, p in unet.named_parameters():
            if n.endswith('.g'):
                p.add_(0.1 * torch.randn_like(p))
            if n.endswith('.b'):
                p.add_(0.1 * torch.randn_like(p))
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    torch.manual_seed(1234)
    x = torch.rand(2, 3, 32, 32) * 2 - 1
    t = torch.tensor([0, 7], dtype=torch.long)
    target = torch.rand(2, 3, 32, 32) * 2 - 1
    y = unet(x, t)
    loss = (target - y).abs().mean()
    loss.backward()
    # full gradient for small tensors; strided subsample + norm for large ones (keeps the fixture small)
    grads = {}
    for n, p in unet.named_parameters():
        g = p.grad.reshape(-1)
        if g.numel() <= 4096:
            grads['grad:' + n] = p.grad.clone()
        else:
            stride = g.numel() // 2048
            grads['gsub:' + n] = g[::stride].clone()
            grads['gnorm:' + n] = g.double().norm().float()
    save('unet_small', x=x, t=t, target=target, y=y, loss=loss,
         **{'sd:' + k: v for k, v in sd.items()}, **grads)

    # ---- (2) q_sample for every blur routine (+discrete) ------------------------------
    ident = torch.nn.Identity()
    cases = [
        ('Incremental', 5, 0.4, 6), ('Constant', 11, 7.0, 6), ('Constant_reflect', 5, 1.5, 6),
        ('Exponential_reflect', 7, 0.1, 8), ('Exponential', 7, 0.1, 8),
        ('Special_6_routine', 11, 0.0, 6),
    ]
    out = {}
    torch.manual_seed(7)
    xq = torch.rand(4, 3, 16, 16) * 2 - 1
    for routine, ks, std, T in cases:
        for discrete in (False, True):
            gd = m.GaussianDiffusion(ident, image_size=16, device_of_kernel='cpu', channels=3,
                                     timesteps=T, kernel_std=std, kernel_size=ks,
                                     blur_routine=routine, discrete=discrete)
            tt = torch.tensor([0, T - 1, 2, 1], dtype=torch.long)
            q = gd.q_sample(xq, tt)
            key = '%s|%d|%g|%d|%d' % (routine, ks, std, T, int(discrete))
            out['q:' + key] = q
            out['t:' + key] = tt
            out['w:' + key] = torch.stack([k.weight[0, 0] for k in gd.gaussian_kernels]) \
                if routine != 'Individual_Incremental' else torch.zeros(1)
    save('qsample', x=xq, **out)

    # ---- (3) sample(): Algorithm 1 ('default') and Algorithm 2 ('x0_step_down') -------
    torch.manual_seed(3)
    out = {}
    xs = torch.rand(2, 3, 32, 32) * 2 - 1
    for routine, ks, std, T, samp, discrete in [
        ('Exponential_reflect', 7, 0.15, 4, 'x0_step_down', False),
        ('Constant', 5, 1.0, 3, 'default', False),
        ('Incremental', 5, 0.5, 3, 'x0_step_down', True),
    ]:
        gd = m.GaussianDiffusion(unet, image_size=32, device_of_kernel='cpu', channels=3,
                                 timesteps=T, kernel_std=std, kernel_size=ks, blur_routine=routine,
                                 sampling_routine=samp, discrete=discrete)
        xt, dr, img = quiet(gd.sample, batch_size=2, img=xs)
        key = '%s|%d|%g|%d|%s|%d' % (routine, ks, std, T, samp, int(discrete))
        out['xt:' + key], out['dr:' + key], out['img:' + key] = xt, dr, img
        tt = torch.tensor([T - 1, 0])
        with torch.no_grad():
            out['loss:' + key] = gd.p_losses(xs, tt)
    save('sample_small', x=xs, **out)

    # ---- (4) Gaussian-noise baseline (denoising-diffusion-pytorch): q_sample, p_losses, gen_sample ----
    dn = ref_shim.import_reference('denoising-diffusion-pytorch', 'denoising_diffusion_pytorch')
    torch.manual_seed(11)
    out = {}
    x1 = torch.rand(2, 3, 32, 32) * 2 - 1
    x2 = torch.randn(2, 3, 32, 32)
    unet_dn = quiet(dn.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet_dn.load_state_dict(sd)          # same small network as (1): identical architecture and keys
    for samp in ('ddim', 'x0_step_down'):
        gd = dn.GaussianDiffusion(unet_dn, image_size=32, channels=3, timesteps=5, loss_type='l1', sampling_routine=samp)
        tt = torch.tensor([4, 0])
        out['q:' + samp] = gd.q_sample(x1, x2, tt)
        with torch.no_grad():
            out['loss:' + samp] = gd.p_losses(x1, x2, tt)
        n, dr, img = quiet(gd.gen_sample, batch_size=2, img=x2)
        out['dr:' + samp], out['img:' + samp] = dr, img
    gd = dn.GaussianDiffusion(unet_dn, image_size=32, channels=3, timesteps=5)
    xt, dr, img = quiet(gd.sample, batch_size=2, img=x2)
    out['sample_dr'], out['sample_img'] = dr, img
    out['sqrt_ac'], out['sqrt_1mac'] = gd.sqrt_alphas_cumprod, gd.sqrt_one_minus_alphas_cumprod
    save('denoise_small', x1=x1, x2=x2, **out)

    # ---- (5) resolution (super-resolution) package: q_sample, p_losses, sample ----------------------------
    rs = ref_shim.import_reference('resolution-diffusion-pytorch', 'resolution_diffusion_pytorch')
    torch.manual_seed(21)
    out = {}
    xr = torch.rand(2, 3, 32, 32) * 2 - 1
    unet_rs = quiet(rs.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet_rs.load_state_dict(sd)
    for routine, T, samp in [('Incremental_factor_2', 4, 'x0_step_down'), ('Incremental_area_factor_2', 5, 'default'),
                             ('Incremental_bilinear', 6, 'x0_step_down'), ('Incremental_bicubic_with_blur', 3, 'x0_step_down')]:
        gd = rs.GaussianDiffusion(unet_rs, image_size=32, device_of_kernel='cpu', channels=3, timesteps=T, loss_type='l1',
                                  resolution_routine=routine, train_routine='Final', sampling_routine=samp)
        tt = torch.tensor([T - 1, 1])
        key = '%s|%d|%s' % (routine, T, samp)
        out['q:' + key] = gd.q_sample(xr, tt)
        with torch.no_grad():
            out['loss:' + key] = gd.p_losses(xr, tt)
        xt, dr, img = quiet(gd.sample, batch_size=2, img=xr)
        out['xt:' + key], out['dr:' + key], out['img:' + key] = xt, dr, img
    save('resolution_small', x=xr, **out)

    # ---- (6) defading (Gaussian mask) package ---------------------------------------------------------------
    df = ref_shim.import_reference('defading-diffusion-pytorch', 'defading_diffusion_pytorch')
    torch.manual_seed(31)
    out = {}
    xf = torch.rand(2, 3, 32, 32) * 2 - 1
    unet_df = quiet(df.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet_df.load_state_dict(sd)
    for routine, T, samp, disc in [('Incremental', 4, 'x0_step_down', False), ('Constant', 3, 'default', False),
                                   ('Random_Incremental', 4, 'x0_step_down', False), ('Incremental', 3, 'x0_step_down', True)]:
        gd = df.GaussianDiffusion(unet_df, image_size=32, device_of_kernel='cpu', channels=3, timesteps=T, loss_type='l1',
                                  kernel_std=0.6, initial_mask=3, fade_routine=routine, sampling_routine=samp, discrete=disc)
        key = '%s|%d|%s|%d' % (routine, T, samp, int(disc))
        tt = torch.tensor([T - 1, 0])
        torch.manual_seed(77)                       # the reference draws the window offsets inside q_sample / sample
        rx = torch.randint(0, 33, (2,)); ry = torch.randint(0, 33, (2,))
        torch.manual_seed(77)
        out['q:' + key] = gd.q_sample(xf, tt)
        torch.manual_seed(77)
        with torch.no_grad():
            out['loss:' + key] = gd.p_losses(xf, tt)
        torch.manual_seed(77)
        xt, dr, img = quiet(gd.sample, batch_size=2, faded_recon_sample=xf)
        out['xt:' + key], out['dr:' + key], out['img:' + key] = xt, dr, img
        out['rx:' + key], out['ry:' + key] = rx, ry
        out['k:' + key] = gd.fade_kernels
    save('defading_small', x=xf, **out)

    # ---- (7) snowification / decolor package (masked per-sample stepping) ----------------------------------
    sn = ref_shim.import_reference('snowification', 'diffusion')
    torch.manual_seed(41)
    out = {}
    xs2 = torch.rand(3, 3, 32, 32) * 2 - 1
    for fpt, kw, T, samp in [('Decolorization', dict(decolor_routine='Linear', decolor_total_remove=True), 5, 'x0_step_down'),
                             ('Decolorization', dict(decolor_routine='Constant', decolor_ema_factor=0.8, decolor_total_remove=False), 4, 'default'),
                             ('Snow', dict(snow_level=1, results_folder='/tmp'), 4, 'x0_step_down'),
                             ('Snow', dict(snow_level=3, fix_brightness=True, results_folder='/tmp'), 3, 'default')]:
        gd = quiet(sn.GaussianDiffusion, unet, image_size=(32, 32) if fpt == 'Snow' else 32, device_of_kernel='cpu', channels=3,
                   timesteps=T, loss_type='l1', forward_process_type=fpt, train_routine='Final', sampling_routine=samp, **kw)
        key = '%s|%s|%d|%s' % (fpt, '-'.join('%s=%s' % (k, v) for k, v in sorted(kw.items()) if k != 'results_folder'), T, samp)
        tt = torch.tensor([T - 1, -1, 1])
        out['q:' + key] = gd.q_sample(xs2, tt)
        with torch.no_grad():
            out['loss:' + key] = gd.p_losses(xs2, torch.tensor([T - 1, 0, 1]))
        tmix = torch.tensor([T - 1, 1, 2])
        x1, d1 = quiet(gd.sample_one_step, xs2, tmix)
        out['one_x:' + key], out['one_dr:' + key] = x1, d1
        r = quiet(gd.sample, batch_size=3, img=xs2)
        out['xt:' + key], out['dr:' + key], out['img:' + key] = r['xt'], r['direct_recons'], r['recon']
        if fpt == 'Snow':
            out['snow:' + key] = torch.stack(gd.forward_process.snow)
            out['br:' + key] = torch.tensor(gd.forward_process.br_coef_list)
    save('snow_small', x=xs2, **out)

    # ---- (8) DDPM-style `Model` (Model2.py), eval mode, + Special_6_routine sampling (BASELINE config 2 shape) ----
    torch.manual_seed(51)
    mkw = dict(resolution=16, in_channels=3, out_ch=3, ch=32, ch_mult=(1, 2), num_res_blocks=2, attn_resolutions=(8,), dropout=0.1)
    model = m.Model(**mkw).eval()
    with torch.no_grad():
        for n, p in model.named_parameters():
            if 'norm' in n:
                p.add_(0.1 * torch.randn_like(p))
    msd = {k: v.clone() for k, v in model.state_dict().items()}
    xm = torch.rand(3, 3, 16, 16) * 2 - 1
    tm = torch.tensor([0, 3, 5])
    with torch.no_grad():
        ym = model(xm, tm)
    gdm = m.GaussianDiffusion(model, image_size=16, device_of_kernel='cpu', channels=3, timesteps=6, loss_type='l1', kernel_std=0.1,
                              kernel_size=3, blur_routine='Special_6_routine', train_routine='Final', sampling_routine='x0_step_down')
    xt, dr, img = quiet(gdm.sample, batch_size=3, img=xm)
    model.eval()
    save('model2_small', x=xm, t=tm, y=ym, s_xt=xt, s_dr=dr, s_img=img, **{'sd:' + k: v for k, v in msd.items()})


if __name__ == '__main__':
    if sys.argv[1:] == ['config1']:
        gen_config1_mnist_loss()
    else:
        main()
        gen_config1_mnist_loss()
