"""Trainer hot loop on the GPU: one optimizer step (2 micro-batches + fused Adam + EMA) against the same step
done with the CPU oracle + torch.optim.Adam, and checkpoint round trip with reference-format keys."""
import io
import contextlib
import os
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def build(sd, T=4):
    import cold_diffusion_models_b200 as cdm
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
        u.load_state_dict(sd)
        gd = cdm.GaussianDiffusion(u, image_size=32, device_of_kernel='cuda', channels=3, timesteps=T, kernel_std=0.15,
                                   kernel_size=7, blur_routine='Exponential_reflect', sampling_routine='x0_step_down').cuda()
    return gd


def test_train_step_matches_oracle_adam(tmp_path):
    import unet_oracle as UO
    import deblur_oracle as DO
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.ops import CONV_SIMT
    sd = UO.make_unet_state_dict(32, (1, 2), 3, seed=3)
    gd = build(sd)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=32, train_batch_size=2, train_lr=1e-3, gradient_accumulate_every=2,
                         results_folder=str(tmp_path), dataset='synthetic', step_start_ema=0, update_ema_every=1, ema_decay=0.9)
    gd.denoise_fn.engine.conv_impl = CONV_SIMT         # fp32 path: isolates the optimizer/EMA/accumulation logic
    g = torch.Generator().manual_seed(5)
    xs = [torch.rand(2, 3, 32, 32, generator=g) * 2 - 1 for _ in range(2)]
    ts = [torch.tensor([3, 0]), torch.tensor([1, 2])]
    # oracle: same two micro-batches, loss/2 each, torch Adam, EMA lerp
    ref = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    orc = DO.DeblurOracle(lambda a, b: UO.unet_forward(ref, a, b), image_size=32, channels=3, timesteps=4, kernel_std=0.15,
                          kernel_size=7, blur_routine='Exponential_reflect')
    opt = torch.optim.Adam(list(ref.values()), lr=1e-3)
    for x, t in zip(xs, ts):
        (orc.p_losses(x, t) / 2).backward()
    opt.step()
    # engine: drive p_losses with the same t (forward() would draw its own)
    for x, t in zip(xs, ts):
        (gd.p_losses(x.cuda(), t.cuda()) / 2).backward()
    tr.opt.step(ema_mode=2, ema_beta=0.9)
    tr.opt.zero_grad()
    torch.cuda.synchronize()
    new = gd.denoise_fn.state_dict()
    ema = tr.ema_model.denoise_fn.state_dict()
    for k in sd:
        assert rel(new[k], ref[k].detach()) < 2e-4, k
        exp_ema = sd[k] * 0.9 + 0.1 * ref[k].detach()
        assert rel(ema[k], exp_ema) < 2e-4, k
    assert float(gd.denoise_fn.engine.flat_grad.abs().max()) == 0.0


def test_gradients_follow_the_weights_across_fused_optimizer_steps(tmp_path):
    """the fused Adam kernel updates the flat parameter buffer through raw pointers (torch's version counters do not move): after
    every optimizer step BOTH pack generations (forward operands and the transposed data-gradient operands) must be rebuilt.
    Two optimizer steps at a large learning rate, then every parameter gradient at the NEW weights against the oracle's
    autograd at the same weights (stale data-gradient packs from step 0 would be several per cent off from step 2 on)."""
    import unet_oracle as UO
    import deblur_oracle as DO
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.ops import CONV_SIMT
    sd = UO.make_unet_state_dict(32, (1, 2), 3, seed=11)
    gd = build(sd)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=32, train_batch_size=2, train_lr=1e-2, gradient_accumulate_every=2,
                         results_folder=str(tmp_path), dataset='synthetic')
    gd.denoise_fn.engine.conv_impl = CONV_SIMT         # fp32 path: tight comparison
    g = torch.Generator().manual_seed(6)
    for _ in range(2):
        tr.train_step(batches=[torch.rand(2, 3, 32, 32, generator=g) * 2 - 1 for _ in range(2)])
        tr.step += 1
    torch.cuda.synchronize()
    now = {k: v.detach().cpu().clone() for k, v in gd.denoise_fn.state_dict().items()}
    assert max(rel(now[k], sd[k]) for k in sd) > 1e-2                      # the weights really moved
    ref = {k: v.clone().requires_grad_(True) for k, v in now.items()}
    orc = DO.DeblurOracle(lambda a, b: UO.unet_forward(ref, a, b), image_size=32, channels=3, timesteps=4, kernel_std=0.15,
                          kernel_size=7, blur_routine='Exponential_reflect', loss_type='l2')
    x = torch.rand(2, 3, 32, 32, generator=g) * 2 - 1
    t = torch.tensor([2, 1])
    orc.p_losses(x, t).backward()
    gd.loss_type = 'l2'
    gd.p_losses(x.cuda(), t.cuda()).backward()
    torch.cuda.synchronize()
    worst = max((rel(p.grad, ref[n].grad), n) for n, p in gd.denoise_fn.named_parameters())
    assert worst[0] < 2e-4, worst


def test_checkpoint_roundtrip_and_train_loop(tmp_path):
    import unet_oracle as UO
    import cold_diffusion_models_b200 as cdm
    sd = UO.make_unet_state_dict(32, (1, 2), 3, seed=4)
    gd = build(sd)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=32, train_batch_size=4, train_lr=2e-5, train_num_steps=3,
                         gradient_accumulate_every=2, results_folder=str(tmp_path), dataset='synthetic')
        tr.train()
    assert tr.step == 3
    tr.save()
    ck = torch.load(os.path.join(str(tmp_path), 'model.pt'), map_location='cpu')
    assert set(ck.keys()) == {'step', 'model', 'ema'}
    # reference key names: denoise_fn.* and gaussian_kernels.{i}.weight (C,1,k,k)
    assert 'denoise_fn.downs.0.0.ds_conv.weight' in ck['model'] and 'gaussian_kernels.3.weight' in ck['model']
    assert tuple(ck['model']['gaussian_kernels.0.weight'].shape) == (3, 1, 7, 7)
    gd2 = build(UO.make_unet_state_dict(32, (1, 2), 3, seed=9))
    with contextlib.redirect_stdout(io.StringIO()):
        tr2 = cdm.Trainer(gd2, None, image_size=32, train_batch_size=4, results_folder=str(tmp_path), dataset='synthetic',
                          load_path=os.path.join(str(tmp_path), 'model.pt'))
    assert tr2.step == 3
    x = torch.rand(2, 3, 32, 32).cuda()
    t = torch.tensor([1, 2]).cuda()
    with torch.no_grad():
        assert torch.equal(gd2.denoise_fn(x, t), gd.denoise_fn(x, t))      # same weights, same inputs: bit-identical (deterministic forward)
    # DataParallel-prefixed checkpoints load too
    pref = {'step': 1, 'model': {'module.' + k: v for k, v in ck['model'].items()}, 'ema': {'module.' + k: v for k, v in ck['ema'].items()}}
    torch.save(pref, os.path.join(str(tmp_path), 'dp.pt'))
    tr2.load(os.path.join(str(tmp_path), 'dp.pt'))
    assert tr2.step == 1


def test_device_resident_input_pipeline_on_the_gpu(tmp_path):
    """SURVEY 8f rank 2: DeviceImageDataset keeps the decoded, resized uint8 images in HBM and builds every batch with one gather
    kernel (cd_augment_u8): bit-exact against the reference's torchvision pipeline (DB:990-996: Resize 1.12 x S, CenterCrop,
    ToTensor()*2-1), explicit crop windows / flips against crop + hflip of the resized image, and a Trainer that trains from it
    (`dataset='device_aug'`) without a DataLoader or an H2D copy of fp32 images."""
    import numpy as np
    from PIL import Image
    from torchvision import transforms
    import unet_oracle as UO
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.trainer import DeviceImageDataset
    rng = np.random.RandomState(0)
    folder = tmp_path / 'imgs'
    folder.mkdir()
    for i in range(7):
        Image.fromarray(rng.randint(0, 256, (40 + i, 44, 3), dtype=np.uint8)).save(str(folder / ('im%d.png' % i)))
    S = 32
    ds = DeviceImageDataset(str(folder), S, augment=False, device='cuda')
    assert ds.src.is_cuda and ds.src.dtype == torch.uint8
    ref_tf = transforms.Compose([transforms.Resize((int(S * 1.12), int(S * 1.12))), transforms.CenterCrop(S), transforms.ToTensor(),
                                 transforms.Lambda(lambda t: (t * 2) - 1)])
    idx = torch.tensor([3, 0, 6, 4])
    got = ds.batch(4, index=idx)
    assert got.is_cuda
    ref = torch.stack([ref_tf(Image.open(ds.paths[int(i)]).convert('RGB')) for i in idx])
    assert torch.equal(got.cpu(), ref)
    resized = [transforms.Resize((ds.rs, ds.rs))(Image.open(p).convert('RGB')) for p in ds.paths]
    oy, ox, fl = torch.tensor([0, 2, 3, 1]), torch.tensor([3, 1, 0, 2]), torch.tensor([True, False, True, False])
    got = ds.batch(4, index=idx, oy=oy, ox=ox, flip=fl).cpu()
    for b in range(4):
        im = transforms.functional.crop(resized[int(idx[b])], int(oy[b]), int(ox[b]), S, S)
        if fl[b]:
            im = transforms.functional.hflip(im)
        assert torch.equal(got[b], transforms.ToTensor()(im) * 2 - 1)
    gd = build(UO.make_unet_state_dict(32, (1, 2), 3, seed=2))
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, str(folder), image_size=S, train_batch_size=4, train_lr=2e-5, train_num_steps=2,
                         gradient_accumulate_every=2, results_folder=str(tmp_path / 'res'), dataset='device_aug')
        b = tr._next()
        assert b.is_cuda and tuple(b.shape) == (4, 3, S, S) and float(b.min()) >= -1.0 and float(b.max()) <= 1.0
        tr.train()
    assert tr.step == 2
