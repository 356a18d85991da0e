"""Golden vectors FROM THE UNMODIFIED REFERENCE for the Lab colour path (`to_lab=True`) of the snowification / decolor package
(SN:287-336, FP:189-218, diffusion/utils.py:113-222).  Needs a checkout of the reference ($COLD_REF_ROOT, see oracle/ref_shim.py);
kornia's four colour stages come from the restatement in tests/lab_oracle.py.  Reuses the small Unet weights of unet_small.npz.

    python tests/golden/gen_golden_lab.py     ->  tests/golden/snow_lab_small.npz

Records rgb2lab / lab2rgb of seeded images (with out-of-gamut Lab inputs that hit the fz clamp and the clip), and q_sample (t
with -1), p_losses, sample_one_step, sample, all_sample and forward_and_backward of Lab decolorization for both sampling
routines (the trajectories of all_sample / forward_and_backward for x0_step_down), plus Snow with to_lab (only its outputs
are converted).  q_sample's t = [-1, 1] hits the reference quirk of SN:373-378 (the kept row is indexed with the unfiltered -1,
i.e. it gets the fully degraded image).  The inputs are rgb2lab of seeded RGB images, as the reference's training loop feeds
them (SN:613-625).  2 images of 16 x 16 keep the file small.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
import lab_oracle  # noqa: E402
from gen_golden import quiet, save  # noqa: E402
from gen_golden_more import small_sd, stack  # noqa: E402


def main():
    torch.set_num_threads(8)
    ref_shim.patch_cuda_noop()
    sd = small_sd()
    db = ref_shim.import_reference('deblurring-diffusion-pytorch', 'deblurring_diffusion_pytorch')   # installs the shim's stubs
    lab_oracle.install_kornia()                                                                    # ... then the colour stages
    sn = ref_shim.import_reference('snowification', 'diffusion')
    ut = sys.modules['diffusion.utils']
    assert ut.rgb_to_linear_rgb is lab_oracle.rgb_to_linear_rgb and ut.xyz_to_rgb is lab_oracle.xyz_to_rgb
    unet = quiet(db.Unet, dim=32, dim_mults=(1, 2), channels=3)
    unet.load_state_dict(sd)
    out = {}
    torch.manual_seed(131)
    rgb = torch.rand(2, 3, 5, 7) * 2.2 - 1.1                      # a little outside [-1, 1] as well
    lab_in = torch.stack([torch.rand(2, 5, 7) * 140 - 20, torch.rand(2, 5, 7) * 300 - 150, torch.rand(2, 5, 7) * 300 - 150], 1)
    out['conv_rgb'], out['conv_lab_in'] = rgb, lab_in
    out['conv_rgb2lab'] = ut.rgb2lab(rgb)
    out['conv_lab2rgb'] = ut.lab2rgb(lab_in)
    out['conv_lab2rgb_noclip'] = ut.lab2rgb(lab_in, clip=False)
    out['conv_roundtrip'] = ut.lab2rgb(ut.rgb2lab(rgb.clamp(-1, 1)))
    torch.manual_seed(137)
    S = 16
    x_rgb = torch.rand(2, 3, S, S) * 2 - 1
    x = ut.rgb2lab(x_rgb)
    for fpt, kw, T, samp in [('Decolorization', dict(decolor_routine='Linear', decolor_total_remove=True), 3, 'x0_step_down'),
                             ('Decolorization', dict(decolor_routine='Constant', decolor_ema_factor=0.8, decolor_total_remove=False), 3, 'default'),
                             ('Snow', dict(snow_level=1, results_folder='/tmp'), 3, 'x0_step_down')]:
        gd = quiet(sn.GaussianDiffusion, unet, image_size=(S, S) if fpt == 'Snow' else S, device_of_kernel='cpu', channels=3,
                   timesteps=T, loss_type='l1', forward_process_type=fpt, train_routine='Final', sampling_routine=samp, to_lab=True, **kw)
        key = '%s|%s|%d|%s' % (fpt, '-'.join('%s=%s' % (k, v) for k, v in sorted(kw.items()) if k != 'results_folder'), T, samp)
        out['q:' + key] = gd.q_sample(x, torch.tensor([-1, 1]))
        with torch.no_grad():
            out['loss:' + key] = gd.p_losses(x, torch.tensor([T - 1, 1]))
        x1, d1 = gd.sample_one_step(x, torch.tensor([T - 1, 2]))
        out['one_x:' + key], out['one_dr:' + key] = x1, d1
        r = quiet(gd.sample, batch_size=2, img=x)
        out['xt:' + key], out['dr:' + key], out['img:' + key] = r['xt'], r['direct_recons'], r['recon']
        if fpt == 'Decolorization':
            out['total:' + key] = gd.forward_process.total_forward(x)
        if samp == 'x0_step_down' and fpt == 'Decolorization':     # the trajectories once (all_sample is decolorization-only)
            X0, Xt, _, _ = quiet(gd.all_sample, batch_size=2, img=x)
            out['all_X0:' + key], out['all_Xt:' + key] = stack(X0), stack(Xt)
            F_, B_, img = quiet(gd.forward_and_backward, batch_size=2, img=x)
            out['fb_F:' + key], out['fb_B:' + key], out['fb_img:' + key] = stack(F_), stack(B_), img
    save('snow_lab_small', x_rgb=x_rgb, x=x, **out)


if __name__ == '__main__':
    main()
