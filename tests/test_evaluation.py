"""Evaluation path: metrics against the reference-generated goldens / the oracle, the mixture model
statistically, and the Trainer's evaluation methods end to end on CPU tensors through tests/abi_emulator.py (files written,
index conventions, metric dictionary)."""
import contextlib
import io
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..', 'oracle'))
G = os.path.join(os.path.dirname(__file__), 'golden')


def _cpu_mode(monkeypatch):
    """CPU tensors pose as CUDA tensors for the host logic; data loaders run in-process (no worker forks in the test suite)"""
    from torch.utils import data
    real = data.DataLoader
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)
    monkeypatch.setattr(data, 'DataLoader', lambda *a, **k: real(*a, **{**k, 'num_workers': 0, 'pin_memory': False}))


def test_frechet_distance_matches_the_reference():
    """symmetric-eigenvalue formulation of the product vs the reference's sqrtm formulation, incl. rank-deficient covariances"""
    from cold_diffusion_models_b200.evaluation import calculate_frechet_distance
    import eval_oracle
    g = np.load(os.path.join(G, 'eval_small.npz'))
    for name in ('d8', 'd64', 'd32_rankdef', 'd16_same'):
        a1, a2, want = g[name + ':a1'], g[name + ':a2'], float(g[name + ':fid'])
        m1, s1, m2, s2 = a1.mean(0), np.cov(a1, rowvar=False), a2.mean(0), np.cov(a2, rowvar=False)
        got = calculate_frechet_distance(m1, s1, m2, s2)
        ora = float(eval_oracle.frechet_distance_sqrtm(m1, s1, m2, s2))
        # the rank-deficient case is where sqrtm itself is ill-conditioned: the reference's value carries ~1e-6 of noise
        tol = 1e-5 if 'rankdef' in name else 1e-9
        assert abs(got - want) <= tol * max(1.0, abs(want)), (name, got, want)
        assert abs(ora - want) <= tol * max(1.0, abs(want)), (name, ora, want)
    assert calculate_frechet_distance(0.0, 2.0, 1.0, 8.0) == pytest.approx(1 + 2 + 8 - 2 * 4)        # scalars: atleast_1d / 2d


def test_activation_statistics_match_the_reference():
    from cold_diffusion_models_b200.evaluation import calculate_activation_statistics, get_activations, calculate_fid_given_samples
    g = np.load(os.path.join(G, 'eval_small.npz'))
    net = torch.nn.Conv2d(3, 12, 3, stride=2)
    net.weight.data.copy_(torch.from_numpy(g['acts:w'])); net.bias.data.copy_(torch.from_numpy(g['acts:b']))
    imgs = torch.from_numpy(g['acts:imgs'])
    mu, sigma = calculate_activation_statistics(imgs[:20], lambda x: [net(x)], batch_size=5, dims=12, device='cpu')
    assert np.allclose(mu, g['acts:mu'], atol=1e-7) and np.allclose(sigma, g['acts:sigma'], atol=1e-7)
    # 23 images at batch 5: the trailing 3 are not evaluated (the reference leaves their rows uninitialised; here they are dropped)
    assert get_activations(imgs, net, batch_size=5, dims=12).shape == (20, 12)
    assert calculate_fid_given_samples([imgs[:20], imgs[:20]], batch_size=5, device='cpu', dims=12, model=net) < 1e-9
    with pytest.raises(RuntimeError, match='feature extractor'):
        calculate_fid_given_samples([imgs, imgs])


def test_ssim_matches_the_direct_restatement():
    from cold_diffusion_models_b200.evaluation import ssim, rmse
    import eval_oracle
    rng = np.random.RandomState(3)
    for shape in ((3, 3, 32, 32), (2, 1, 17, 40), (2, 3, 11, 11), (1, 3, 8, 24)):
        x = rng.rand(*shape).astype(np.float32)
        y = np.clip(x + 0.1 * rng.randn(*shape), 0, 1).astype(np.float32)
        for size_average in (True, False):
            got = ssim(torch.from_numpy(x), torch.from_numpy(y), data_range=1, size_average=size_average).numpy()
            want = eval_oracle.ssim_direct(x, y, data_range=1.0, size_average=size_average)
            assert np.allclose(got, want, atol=2e-5), (shape, got, want)
    x = torch.rand(4, 3, 20, 20)
    assert float(ssim(x, x, data_range=1)) == pytest.approx(1.0, abs=1e-6)
    assert float(ssim(x, x, data_range=1, chunk=3)) == pytest.approx(1.0, abs=1e-6)
    assert float(ssim(x, 1 - x, data_range=1)) < 0.1 < float(ssim(x, 1 - x, data_range=1, nonnegative_ssim=True)) + 0.1001
    assert float(rmse(x, x + 0.5)) == pytest.approx(0.5, abs=1e-6)
    with pytest.raises(ValueError):
        ssim(x, x[:, :, :10], data_range=1)
    with pytest.raises(ValueError):
        ssim(x[0], x[0], data_range=1)
    with pytest.raises(ValueError):
        ssim(x, x, win_size=10)


def test_gaussian_mixture_recovers_a_known_mixture():
    from cold_diffusion_models_b200.evaluation import GaussianMixture
    torch.manual_seed(0)
    means = torch.tensor([[-4.0, 0.0, 1.0], [3.0, 3.0, -2.0], [0.0, -5.0, 4.0]])
    A = torch.tensor([[1.0, 0.3, 0.0], [0.0, 0.7, 0.2], [0.0, 0.0, 0.5]])
    comp = torch.multinomial(torch.tensor([0.5, 0.3, 0.2]), 6000, replacement=True)
    X = means[comp] + torch.randn(6000, 3) @ A
    # the call the reference's drivers make (DB:1410-1411)
    gm = GaussianMixture(num_components=3, trainer_params=dict(gpus=1), covariance_type='full', convergence_tolerance=0.001,
                         batch_size=100, seed=1)
    assert gm.fit(X) is gm and gm.converged_
    order = torch.cdist(means.double(), gm.means_).argmin(1)
    assert sorted(order.tolist()) == [0, 1, 2]
    assert torch.allclose(gm.means_[order].float(), means, atol=0.1)
    assert torch.allclose(gm.weights_[order].float(), torch.tensor([0.5, 0.3, 0.2]), atol=0.03)
    assert torch.allclose(gm.covariances_[order[0]].float(), A.T @ A, atol=0.08)
    s = gm.sample(num_datapoints=20000)
    assert s.shape == (20000, 3) and s.dtype == torch.float32
    assert torch.allclose(s.mean(0), X.mean(0), atol=0.12) and torch.allclose(torch.cov(s.T), torch.cov(X.T), atol=0.5)
    assert abs(gm.score(X) - gm.nll_) < 1e-2
    assert (gm.predict(means) == order).all()
    assert gm.get_params()['num_components'] == 3 and 'GaussianMixture' in repr(gm)
    for ct in ('diag', 'spherical'):
        g2 = GaussianMixture(num_components=3, covariance_type=ct, seed=2).fit(X)
        assert g2.score(X) >= gm.score(X) - 1e-6            # fewer covariance parameters cannot fit better than 'full'
        assert g2.sample(5).shape == (5, 3)
    with pytest.raises(ValueError):
        GaussianMixture(2, covariance_type='tied')
    with pytest.raises(RuntimeError):
        GaussianMixture(2).sample(3)


@pytest.fixture()
def trainer(monkeypatch, tmp_path):
    """deblurring Trainer over a folder of 14 PNG files, on CPU tensors through the emulated C ABI"""
    import abi_emulator
    import cold_diffusion_models_b200 as cdm
    from PIL import Image
    _cpu_mode(monkeypatch)
    monkeypatch.chdir(tmp_path)
    z = np.load(os.path.join(G, 'unet_small.npz'))
    rng = np.random.RandomState(0)
    data_dir = tmp_path / 'data'
    data_dir.mkdir()
    for i in range(14):
        Image.fromarray(rng.randint(0, 256, (32, 32, 3), dtype=np.uint8)).save(str(data_dir / f'{i:03d}.png'))
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
        u.load_state_dict({k[3:]: torch.from_numpy(np.asarray(z[k])) for k in z.files if k.startswith('sd:')})
        gd = cdm.GaussianDiffusion(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=3, kernel_std=0.15, kernel_size=5,
                                   blur_routine='Exponential_reflect', sampling_routine='x0_step_down')
    with abi_emulator.patched():
        with contextlib.redirect_stdout(io.StringIO()):
            tr = cdm.Trainer(gd, str(data_dir), image_size=32, train_batch_size=4, results_folder=str(tmp_path / 'res'), shuffle=False)
            from cold_diffusion_models_b200.trainer import cycle
            tr.dl = cycle(torch.utils.data.DataLoader(tr.ds, batch_size=4, shuffle=False, num_workers=0, drop_last=True))
        yield tr, tmp_path / 'res'


def test_trainer_figure_dumps(trainer):
    """test_from_data / save_training_data / paper_* write the reference's file names (DB:1238-1388, 1712-1722)"""
    import cv2
    tr, res = trainer
    with contextlib.redirect_stdout(io.StringIO()):
        X0s, Xts = tr.test_from_data('test', s_times=None)
    assert len(X0s) == 4 and len(Xts) == 3
    for i in range(4):
        assert (res / f'sample-{i}-test-x0.png').exists()
    for i in range(3):
        assert (res / f'sample-{i}-test-xt.png').exists()
    assert (res / 'og-test.png').exists() and (res / 'Gif-test-x0.gif').exists() and (res / 'Gif-test-xt.gif').exists()
    grid = cv2.imread(str(res / 'og-test.png'))
    titled = cv2.imread(str(res / 'sample-0-test-x0.png'))
    assert titled.shape[0] == grid.shape[0] + 40 and titled.shape[1] == grid.shape[1] + 20      # 10 px frame + 20 px title bar
    assert tuple(titled[5, 5]) == (255, 0, 180)

    with contextlib.redirect_stdout(io.StringIO()):
        tr.paper_showing_diffusion_images_cover_page(n_batches=1)
        tr.paper_showing_diffusion_images_cover_page_both_sampling(n_batches=1)
    # timesteps = 3: of the shown indices only 2 exists -> original, forward[2], backward[len - 2], final = 4 tiles of 32 px
    strip = cv2.imread(str(res / 'all_0.png'))
    assert strip.shape == (32, 4 * 32, 3)
    for k in range(4):
        for n in (f'all_{k}.png', f'all_1_{k}.png', f'all_2_{k}.png', f'og_img_{k}.png', f'final_{k}.png', f'final_1_{k}.png'):
            assert (res / n).exists(), n
    with contextlib.redirect_stdout(io.StringIO()):
        tr.paper_invert_section_images(n_batches=1)
    assert cv2.imread(str(res / 'all_0.png')).shape == (52, 4 * 52, 3)                           # 4 framed 32 px tiles
    out = res / 'train_png'
    tr.results_folder = out
    with contextlib.redirect_stdout(io.StringIO()):
        tr.save_training_data()
    assert len(list(out.glob('*.png'))) == 14


def test_trainer_metrics_over_the_manifold(trainer):
    """fid_distance_decrease_from_manifold: skips image `start`, includes `end`, batches of `bs`, the three comparisons"""
    from cold_diffusion_models_b200.evaluation import ssim, rmse
    tr, res = trainer
    seen = []

    def fake_fid(samples):
        seen.append((tuple(samples[0].shape), tuple(samples[1].shape)))
        return float((samples[0] - samples[1]).abs().mean())
    with contextlib.redirect_stdout(io.StringIO()) as log:
        out = tr.fid_distance_decrease_from_manifold(fake_fid, start=0, end=9, bs=4)
    assert seen == [((9, 3, 32, 32), (9, 3, 32, 32))] * 3                    # images 1..9
    assert set(out) == {'blurred', 'deblurred', 'direct'}
    assert all(0 <= v['rmse'] <= 1 and -1 <= v['ssim'] <= 1 for v in out.values())
    for n in ('og', 'xt', 'recons', 'direct-recons'):
        assert os.path.exists(f'./sanity_check/sample-{n}.png')
    text = log.getvalue()
    assert 'The FID of blurry images with original image is' in text and 'Hence the improvement in FID using direct sampling is' in text
    # the numbers are those of the images the diffusion produces for the same batches
    og = torch.stack([tr.ds[i] for i in range(1, 10)])
    X0s, Xts = tr.ema_model.all_sample(batch_size=4, img=og[:4])
    u = lambda t: (t + 1) * 0.5
    with contextlib.redirect_stdout(io.StringIO()):
        out4 = tr.fid_distance_decrease_from_manifold(None, start=0, end=4, bs=4, sanity_check=0)
    assert out4['blurred']['fid'] is None
    assert out4['blurred']['rmse'] == pytest.approx(float(rmse(u(og[:4]), u(Xts[0]))), abs=1e-6)
    assert out4['deblurred']['ssim'] == pytest.approx(float(ssim(u(og[:4]), u(X0s[-1]), data_range=1)), abs=1e-5)


def test_trainer_generation_from_fitted_mixtures(trainer):
    """sample_as_a_*_gmm*: features gathered over the data set in order, mixture fitted, samples restored and written"""
    from cold_diffusion_models_b200.evaluation import GaussianMixture
    tr, res = trainer
    fitted = {}

    class Spy(GaussianMixture):
        def fit(self, X):
            fitted['X'] = X.clone()
            return super().fit(X)
    feats = torch.stack([tr.ds[i] for i in range(12)]).mean((2, 3))
    orig = tr._dataset_features
    tr._dataset_features = lambda fn, batch_size=100: orig(fn, batch_size=4)          # 14 images: 3 full batches of 4
    with contextlib.redirect_stdout(io.StringIO()):
        m = tr.sample_as_a_mean_blur_torch_gmm_ablation(Spy, clusters=2, num_samples=4, bs=2)
    assert isinstance(m, Spy) and torch.allclose(fitted['X'], feats, atol=1e-6)
    for k in ('xt', 'out', 'dir_recons'):
        assert len(os.listdir(f'{res}_{k}')) == 4
    with contextlib.redirect_stdout(io.StringIO()):
        tr.sample_as_a_mean_blur_torch_gmm(None, clusters=2, num_samples=3, noise_levels=(0.001,), repeats=2)
        tr.sample_as_a_blur_torch_gmm(Spy, siz=2, clusters=1, sample_at=1, num_samples=3)
    assert fitted['X'].shape == (12, 3 * 2 * 2)
    for n in ('sample-og-0.001-0-0.png', 'sample-recon-0.001-0-1.png', 'sample-xt-1-2-1.png', 'sample-direct_recons-1-2-1.png'):
        assert (res / n).exists(), n


def test_package_trainers_use_their_own_evaluation_inputs(monkeypatch, tmp_path):
    """the hooks behind the shared evaluation routines: demixing starts from the second folder and runs forward_and_backward on a
    pair (DM:776, 848-852), defading-generation starts from a constant colour (DFGEN:833-839, 917-928), denoising has no
    noise_level keyword, resolution fits its mixture to area-shrunk step-t images (RS:1117-1183)"""
    import abi_emulator
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200 import (demixing_diffusion_pytorch as dm, defading_generation_diffusion_pytorch as dg,
                                            denoising_diffusion_pytorch as dn, resolution_diffusion_pytorch as rs)
    from cold_diffusion_models_b200.trainer import cycle
    from PIL import Image
    _cpu_mode(monkeypatch)
    monkeypatch.chdir(tmp_path)
    real_rand, real_randn = torch.rand, torch.randn
    monkeypatch.setattr(torch, 'rand', lambda *a, **k: real_rand(*a, **{x: y for x, y in k.items() if x != 'device'}))
    monkeypatch.setattr(torch, 'randn', lambda *a, **k: real_randn(*a, **{x: y for x, y in k.items() if x != 'device'}))
    z = np.load(os.path.join(G, 'unet_small.npz'))
    sd = {k[3:]: torch.from_numpy(np.asarray(z[k])) for k in z.files if k.startswith('sd:')}
    rng = np.random.RandomState(1)
    for d in ('a', 'b'):
        (tmp_path / d).mkdir()
        for i in range(6):
            Image.fromarray(rng.randint(0, 256, (32, 32, 3), dtype=np.uint8)).save(str(tmp_path / d / f'{i}.png'))

    def unet():
        with contextlib.redirect_stdout(io.StringIO()):
            u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
        u.load_state_dict(sd)
        return u
    quiet = lambda: contextlib.redirect_stdout(io.StringIO())
    common = dict(image_size=32, train_batch_size=2)
    with abi_emulator.patched():
        # demixing
        with quiet():
            tr = dm.Trainer(dm.GaussianDiffusion(unet(), image_size=32, channels=3, timesteps=3), str(tmp_path / 'a'), str(tmp_path / 'b'),
                            results_folder=str(tmp_path / 'dm'), shuffle=False, **common)
            first_b = tr.ds2[0]
            assert torch.equal(tr._eval_batch()[0], first_b)
            tr.paper_showing_diffusion_images_cover_page(n_batches=1)
            tr.test_from_data('t')
        assert tr._cover_batches == 5 and (tmp_path / 'dm' / 'all_1.png').exists() and (tmp_path / 'dm' / 'Gif-t-x0.gif').exists()
        # defading-generation
        with quiet():
            tr = dg.Trainer(dg.GaussianDiffusion(unet(), image_size=32, channels=3, timesteps=3), str(tmp_path / 'a'),
                            results_folder=str(tmp_path / 'dg'), **common)
            b = tr._eval_batch()
            assert b.shape == (2, 3, 32, 32) and float(b.std((2, 3)).max()) < 1e-4 and float(b.abs().max()) <= 0.51
            tr.paper_showing_diffusion_images_cover_page(n_batches=1)
            tr.sample_and_save_for_fid(num_samples=2, bs=2)
        assert (tmp_path / 'dg' / 'all_0.png').exists() and len(os.listdir(str(tmp_path / 'dg') + '_out')) == 2
        # denoising: forward_and_backward has no noise_level keyword
        with quiet():
            tr = dn.Trainer(dn.GaussianDiffusion(unet(), image_size=32, channels=3, timesteps=3), str(tmp_path / 'a'),
                            results_folder=str(tmp_path / 'dn'), **common)
            tr.paper_showing_diffusion_images_cover_page(n_batches=1)
            tr.paper_showing_diffusion_images(n_batches=1, to_show=(0, 2))
        assert (tmp_path / 'dn' / 'x_best_1.png').exists() and (tmp_path / 'dn' / 'x_3_0.png').exists()
        # resolution
        with quiet():
            gd = rs.GaussianDiffusion(unet(), image_size=32, device_of_kernel='cpu', channels=3, timesteps=3,
                                      resolution_routine='Incremental_factor_2', sampling_routine='x0_step_down')
            tr = rs.Trainer(gd, str(tmp_path / 'a'), results_folder=str(tmp_path / 'rs'), shuffle=False, **common)
            orig = tr._dataset_features
            tr._dataset_features = lambda fn, batch_size=100: orig(fn, batch_size=3)
            m = tr.sample_as_a_mean_blur_torch_gmm_ablation(None, siz=2, clusters=1, sample_at=2, num_samples=4, bs=2)
        want = torch.nn.functional.interpolate(gd.opt(torch.stack([tr.ds[i] for i in range(6)]), t=2), size=2, mode='area').flatten(1)
        assert torch.allclose(m.means_[0].float(), want.mean(0), atol=1e-5)
        assert len(os.listdir(str(tmp_path / 'rs') + '_out')) == 4
        import inspect
        assert inspect.signature(tr.fid_distance_decrease_from_manifold).parameters['bs'].default == 200


def test_snowification_trainer_evaluation_helpers(monkeypatch, tmp_path):
    """the decolor / snow Trainer's own helpers (SN:682-1200): multi-title bars, og dictionary grids, composite GIF frames,
    PSNR / SSIM running metrics, permuted manifold walk with 16-image batches"""
    import abi_emulator
    import cv2
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200 import snowification_diffusion as sn
    from cold_diffusion_models_b200.evaluation import PSNR, SSIM
    from PIL import Image
    _cpu_mode(monkeypatch)
    monkeypatch.chdir(tmp_path)
    z = np.load(os.path.join(G, 'unet_small.npz'))
    rng = np.random.RandomState(2)
    (tmp_path / 'a').mkdir()
    for i in range(6):
        Image.fromarray(rng.randint(0, 256, (32, 32, 3), dtype=np.uint8)).save(str(tmp_path / 'a' / f'{i}.png'))
    quiet = lambda: contextlib.redirect_stdout(io.StringIO())
    with quiet():
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
        u.load_state_dict({k[3:]: torch.from_numpy(np.asarray(z[k])) for k in z.files if k.startswith('sd:')})
        gd = sn.GaussianDiffusion(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=4, forward_process_type='Decolorization',
                                  decolor_routine='Linear', sampling_routine='x0_step_down')
    with abi_emulator.patched():
        with quiet():
            tr = sn.Trainer(gd, str(tmp_path / 'a'), train_batch_size=3, results_folder=str(tmp_path / 'sn'))
        res = tmp_path / 'sn'
        assert tr.data_loader is not None and tr._to_show == (0, 1, 2, 3, 3)
        with quiet():
            tr.test_from_data('t')
            tr.test_with_mixup('m')
            tr.test_from_random('r')
        for n in ('og-t.png', 'sample-0-t-x0.png', 'sample-3-t-xt.png', 'Gif-t-x0.gif', 'og1-m.png', 'og2-m.png', 'og-m.png',
                  'Gif-m-xt.gif', 'og-r.png', 'sample-3-r-x0.png'):
            assert (res / n).exists(), n
        og = cv2.imread(str(res / 'og-t.png'))
        frame = cv2.imread(str(res / 'sample-0-t-x0.png'))
        # frame = [step grid | og grid] side by side (make_grid of two grids, padding 2) inside the 10 px frame + 20 px bar
        grid_h, grid_w = og.shape[0] - 40, og.shape[1] - 20
        assert frame.shape[0] == (grid_h + 4) + 40 and frame.shape[1] == (2 * grid_w + 6) + 20
        with quiet():
            tr.paper_invert_section_images(n_batches=1, group=3)
            tr.paper_showing_diffusion_images(n_batches=1)
            tr.paper_showing_diffusion_images_cover_page(n_batches=1)
        assert (res / 'blurry_image_0.png').exists() and (res / 'x_best_2.png').exists() and (res / 'all_2.png').exists()
        md = tr.create_metric_dict()
        assert set(md) == {'PSNR', 'SSIM'} and len(md['PSNR']) == 4
        a = torch.rand(3, 3, 32, 32)
        for m in md['PSNR'] + md['SSIM']:
            m.update((a, a))
        md['PSNR'][0].update(((a + 0.1).clamp(0, 1), a))
        tr.save_metric(md, prefix='x')
        lines = open(str(res / 'x-SSIM.txt')).read().split()
        assert len(lines) == 4 and abs(float(lines[0]) - 1.0) < 1e-5
        assert float(open(str(res / 'x-PSNR.txt')).read().split()[0]) < float(open(str(res / 'x-PSNR.txt')).read().split()[1])
        p = PSNR(data_range=1.0); p.update((torch.zeros(2, 3, 8, 8), torch.full((2, 3, 8, 8), 0.1)))
        assert float(p.compute()) == pytest.approx(20.0, abs=1e-3)
        assert torch.equal(tr.shift_data_range(torch.tensor([-1.0, 1.0])), torch.tensor([0.0, 1.0]))
        seen = []
        with quiet():
            out = tr.fid_distance_decrease_from_manifold(lambda samples: seen.append(samples[0].shape[0]) or 0.0, start=0, end=None)
        assert seen == [5, 5, 5] and not os.path.exists('./sanity_check') and set(out) == {'blurred', 'deblurred', 'direct'}
        assert tr._score_view(torch.zeros(1, 3, 300, 300)).shape[-1] == 64 and tr._score_view(torch.zeros(1, 3, 128, 128)).shape[-1] == 128


def test_defading_trainer_evaluation_calls(monkeypatch, tmp_path):
    """defading names the start image `faded_recon_sample` (DFG:817); mixup / off-manifold / seeded-sample / per-image dumps"""
    import abi_emulator
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200 import defading_diffusion_pytorch as df
    from PIL import Image
    _cpu_mode(monkeypatch)
    monkeypatch.chdir(tmp_path)
    z = np.load(os.path.join(G, 'unet_small.npz'))
    rng = np.random.RandomState(3)
    (tmp_path / 'a').mkdir()
    for i in range(7):
        Image.fromarray(rng.randint(0, 256, (32, 32, 3), dtype=np.uint8)).save(str(tmp_path / 'a' / f'{i}.png'))
    quiet = lambda: contextlib.redirect_stdout(io.StringIO())
    with quiet():
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
        u.load_state_dict({k[3:]: torch.from_numpy(np.asarray(z[k])) for k in z.files if k.startswith('sd:')})
        gd = df.GaussianDiffusion(u, image_size=32, device_of_kernel='cpu', channels=3, timesteps=3, kernel_std=0.6, initial_mask=3,
                                  fade_routine='Incremental', sampling_routine='x0_step_down')
    with abi_emulator.patched():
        with quiet():
            tr = df.Trainer(gd, str(tmp_path / 'a'), image_size=32, train_batch_size=2, results_folder=str(tmp_path / 'df'))
            tr.test_from_data('t')
            tr.test_with_mixup('m')
            tr.test_from_random('r')
            tr.controlled_direct_reconstruct('c')
            orig = tr._dataset_features
            tr._dataset_features = lambda fn, batch_size=100: orig(fn, batch_size=3)
            n = tr.test_from_data_save_results(bs=4)
            out = tr.fid_distance_decrease_from_manifold(None, start=0, end=4, bs=2, sanity_check=0)
    res = tmp_path / 'df'
    for name in ('og-t.png', 'Gif-t-xt.gif', 'og1-m.png', 'og2-m.png', 'sample-2-m-x0.png', 'og-r.png', 'sample-og-c.png', 'sample-recon-c.png',
                 'sample-direct_recons-c.png', 'sample-xt-c.png', 'model.pt'):
        assert (res / name).exists(), name
    assert n == 6 and all(len(os.listdir(f'{res}_{k}')) == 6 for k in ('orig', 'blur', 'deblur', 'd_deblur'))
    assert out['direct']['fid'] is None and 0 < out['blurred']['rmse'] < 1


# Trainer methods of the reference that no driver script calls and that cannot run there either: they call
# `GaussianDiffusion.all_sample_both_sample`, which no package defines (DN:1004, 1056), or fit sklearn mixtures to 64 x 64 x 3
# vectors and unpack a pair from denoising's three-list `all_sample` (DN:1128).  Not carried over.
_UNCALLED_LEFTOVERS = {'paper_showing_diffusion_images_diff', 'paper_showing_sampling_diff_images', 'sample_as_a_vector_gmm',
                       'sample_as_a_vector_gmm_and_save', 'sample_as_a_vector_pytorch_gmm_and_save',
                       'sample_as_a_vector_from_blur_pytorch_gmm_and_save'}


def test_trainer_method_surface_matches_the_reference():
    """every public method of every package's reference Trainer (tests/golden/trainer_api.json, recorded from the unmodified
    reference) exists with the same parameter names in the same order; ours may add keyword parameters with defaults"""
    import inspect
    import json
    from cold_diffusion_models_b200 import (deblurring_diffusion_pytorch as db, resolution_diffusion_pytorch as rs,
                                            defading_diffusion_pytorch as df, denoising_diffusion_pytorch as dn,
                                            demixing_diffusion_pytorch as dm, defading_generation_diffusion_pytorch as dg,
                                            snowification_diffusion as sn)
    mods = dict(deblurring=db, resolution=rs, defading=df, denoising=dn, demixing=dm, defading_generation=dg, snowification=sn)
    api = json.load(open(os.path.join(G, 'trainer_api.json')))
    problems, skipped = [], set()
    for tag, entry in api.items():
        T = mods[tag].Trainer
        for mn, names in entry.items():
            fn = getattr(T, mn, None)
            if fn is None:
                if mn in _UNCALLED_LEFTOVERS and tag in ('denoising', 'demixing', 'defading_generation'):
                    skipped.add(mn)
                else:
                    problems.append((tag, mn, 'missing'))
                continue
            params = inspect.signature(fn).parameters
            mine = [n for n in params if n != 'self']
            if [n for n in mine if n in names] != names:
                problems.append((tag, mn, names, mine))
            extras = [n for n in mine if n not in names and params[n].default is inspect._empty
                      and params[n].kind not in (inspect.Parameter.VAR_KEYWORD, inspect.Parameter.VAR_POSITIONAL)]
            if extras:
                problems.append((tag, mn, 'extra parameter without default', extras))
    assert not problems, problems
    assert skipped == _UNCALLED_LEFTOVERS


def test_fid_inception_matches_the_reference_network():
    """`evaluation.InceptionV3` (torchvision blocks + pooling hooks) against the reference's Fid/inception.py network, both loaded
    with the same synthetic weight file (tests/golden/fid_weights.py); the border row of block 2 is where counting the padding
    in the average pooling would show"""
    import tempfile
    import torchvision
    from cold_diffusion_models_b200.evaluation import InceptionV3, calculate_fid_given_samples
    sys.path.insert(0, G)
    from fid_weights import synthetic_state
    g = np.load(os.path.join(G, 'eval_small.npz'))
    shapes = {k: v.shape for k, v in torchvision.models.inception_v3(weights=None, aux_logits=False, num_classes=1008,
                                                                       init_weights=False).state_dict().items()}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'pt_inception.pth')
        torch.save(synthetic_state(shapes), path)
        net = InceptionV3([0, 1, 2, 3], weights_path=path).eval()
        small = InceptionV3([2], resize_input=False, normalize_input=False, weights_path=path).eval()
        os.environ['COLDDIFF_FID_WEIGHTS'] = path
        try:
            imgs = torch.from_numpy(g['fid:imgs'])
            fid = calculate_fid_given_samples([imgs, imgs.flip(0)], batch_size=2, device='cpu', dims=64)
        finally:
            del os.environ['COLDDIFF_FID_WEIGHTS']
    assert abs(fid) < 1e-6                                             # same set in another order
    assert not any(p.requires_grad for p in net.parameters())
    with torch.no_grad():
        feats = net(torch.from_numpy(g['fid:imgs']))
        sb2 = small(torch.from_numpy(g['fid:small_in']))[0]
    rel = lambda a, b: float(np.linalg.norm(a - b) / np.linalg.norm(b))
    for i, f in enumerate(feats):
        got = (f if i == 3 else f.mean((2, 3))).numpy()
        assert got.shape == g[f'fid:block{i}'].shape and rel(got, g[f'fid:block{i}']) < 1e-5, i
    assert rel(feats[2][:, :16, 0, :].numpy(), g['fid:block2_edge']) < 1e-5
    assert rel(sb2.numpy(), g['fid:small_block2']) < 1e-5
    with pytest.raises(RuntimeError, match='weights_path'):
        InceptionV3()
    assert InceptionV3.BLOCK_INDEX_BY_DIM[2048] == 3
