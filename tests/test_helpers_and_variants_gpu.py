"""GPU parity of the API helpers (Individual_Incremental, resolution Step routine / t = -1 rows, sample_from_blur, all_sample /
forward_and_backward of every package, Unet constructor options, the evaluation routines) against the reference goldens, and of
the kernel variants behind library switches against the kernels they replace."""
import io
import contextlib
import pytest
import torch

from test_unet_gpu import load, rel, make_unet

pytestmark = pytest.mark.gpu

OPT_IN = lambda f: f          # kernel-variant tests (switch on / off comparisons)


@pytest.fixture(scope='module')
def small():
    g = load('unet_small')
    sd = {k[3:]: v for k, v in g.items() if k.startswith('sd:')}
    return g, sd, make_unet(32, (1, 2), 3, sd)


@pytest.fixture(scope='module')
def unet(small):
    return small[2]


def stack(lst):
    return torch.stack([x.detach().float().cpu() for x in lst])


def test_individual_incremental_routine_matches_reference_golden(small):
    """the seventh blur routine (kernel size 2i+1, sigma 2k; `sample` starts from the single step-t kernel, DB:379-383, 401-402)"""
    import cold_diffusion_models_b200 as cdm
    g = load('individual_small')
    _, sd, u = small
    x = g['x'].cuda()
    for samp in ('default', 'x0_step_down'):
        gd = cdm.GaussianDiffusion(u, image_size=32, device_of_kernel='cuda', channels=3, timesteps=4, kernel_std=0.1, kernel_size=3,
                                   blur_routine='Individual_Incremental', sampling_routine=samp).cuda()
        for i, kconv in enumerate(gd.gaussian_kernels):
            assert torch.equal(kconv.weight[0, 0].cpu(), g['w%d' % i])
        tt = torch.tensor([3, 1]).cuda()
        assert torch.allclose(gd.q_sample(x, tt).cpu(), g['q'], atol=3e-6)
        with torch.no_grad():
            assert abs(gd.p_losses(x, tt).item() - g['loss'].item()) < 3e-4
        xt, dr, img = gd.sample(batch_size=2, img=x)
        assert rel(xt, g['xt:' + samp]) < 1e-5 and rel(dr, g['dr:' + samp]) < 1e-3 and rel(img, g['img:' + samp]) < 2e-3, samp


def test_resolution_step_routine_and_negative_t_rows_match_reference_golden(small):
    """'Step' train routine (RS:742-755; no random draws) and the t = -1 rows of q_sample, which take the level max(t) of the
    batch in the reference (RS:645 tests the loop index instead of t)"""
    from cold_diffusion_models_b200.resolution_diffusion_pytorch import GaussianDiffusion
    g = load('resolution_train_small')
    _, sd, u = small
    x = g['x'].cuda()
    for lt in ('l1', 'l2'):
        gd = GaussianDiffusion(u, image_size=32, device_of_kernel='cuda', channels=3, timesteps=4, loss_type=lt,
                               resolution_routine='Incremental_factor_2', train_routine='Step', sampling_routine='x0_step_down').cuda()
        with torch.no_grad():
            assert abs(gd.p_losses(x, torch.tensor([3, 0, 2]).cuda()).item() - g['loss:Step|' + lt].item()) < 3e-4, lt
    assert torch.allclose(gd.q_sample(x, torch.tensor([2, -1, 1]).cuda()).cpu(), g['q_neg'], atol=3e-6)


def test_deblur_sample_from_blur_and_all_sample_match_reference_golden(unet):
    """sample_from_blur with a partial blur (start .. t-1, DB:863-925) and the all_sample lists (DB:609-689).  Multi-step
    trajectories on the TF32 path: 4e-3 (the single-forward tolerance is 1e-3; errors compound over the reverse steps)"""
    import cold_diffusion_models_b200 as cdm
    g = load('fb_small')
    x = g['x'].cuda()
    for key in sorted(k[4:] for k in g if k.startswith('img:')):
        routine, ks, std, T, samp = key.split('|')
        gd = cdm.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=int(T), kernel_std=float(std),
                                   kernel_size=int(ks), blur_routine=routine, sampling_routine=samp).cuda()
        for start in (0, 1):
            xt, dr, img = gd.sample_from_blur(batch_size=2, img=x, start=start)
            pre = ':%d:' % start + key
            assert rel(xt, g['sfb_xt' + pre]) < 1e-5 and rel(dr, g['sfb_dr' + pre]) < 1e-3 and rel(img, g['sfb_img' + pre]) < 4e-3, pre
        X0s, Xts = gd.all_sample(batch_size=2, img=x)
        assert rel(stack(X0s), g['all_X0:' + key]) < 4e-3 and rel(stack(Xts), g['all_Xt:' + key]) < 4e-3, key


def test_sampling_helpers_of_the_other_packages_match_reference_golden(unet):
    """resolution all_sample / forward_and_backward / func[i] (RS:505-616, 389-414), defading all_sample (DFG:428-494),
    snowification / decolor all_sample and forward_and_backward (SN:299-339, 450-490)"""
    import io
    import contextlib
    from cold_diffusion_models_b200.resolution_diffusion_pytorch import GaussianDiffusion as RSGD
    from cold_diffusion_models_b200.defading_diffusion_pytorch import GaussianDiffusion as DFGD
    from cold_diffusion_models_b200.snowification_diffusion import GaussianDiffusion as SNGD
    g = load('resolution_train_small')
    x = g['x'].cuda()
    for samp in ('x0_step_down', 'default'):
        gd = RSGD(unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=4, loss_type='l1',
                  resolution_routine='Incremental_factor_2', train_routine='Final', sampling_routine=samp).cuda()
        X0s, Xts = gd.all_sample(batch_size=3, img=x)
        assert rel(stack(X0s), g['all_X0:' + samp]) < 4e-3 and rel(stack(Xts), g['all_Xt:' + samp]) < 4e-3, samp
        F_, B_, img = gd.forward_and_backward(batch_size=3, img=x)
        assert rel(stack(F_), g['fb_F:' + samp]) < 1e-5 and rel(stack(B_), g['fb_B:' + samp]) < 4e-3 and rel(img, g['fb_img:' + samp]) < 4e-3, samp
    f1 = gd.func[1](x)
    assert torch.allclose(f1.cpu(), g['func1'], atol=3e-6) and torch.allclose(gd.func[2](f1).cpu(), g['func2of1'], atol=3e-6)

    g = load('defading_all_small')
    x = g['x'].cuda()
    for key in sorted(k[3:] for k in g if k.startswith('x0:')):
        routine, T, samp = key.split('|')
        gd = DFGD(unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=int(T), loss_type='l1', kernel_std=0.6, initial_mask=3,
                  fade_routine=routine, sampling_routine=samp).cuda()
        off = (g['rx:' + key].cuda(), g['ry:' + key].cuda()) if 'Random' in routine else (None, None)
        x0l, xtl = gd.all_sample(batch_size=2, faded_recon_sample=x, _offsets=off)
        assert rel(stack(x0l), g['x0:' + key]) < 4e-3 and rel(stack(xtl), g['xt:' + key]) < 4e-3, key

    g = load('snow_more_small')
    x = g['x'].cuda()
    for key in sorted(k[5:] for k in g if k.startswith('fb_F:')):
        fpt, kws, T, samp = key.split('|')
        kw = {}
        for item in kws.split('-'):
            k, v = item.split('=')
            kw[k] = (v == 'True') if v in ('True', 'False') else (float(v) if '.' in v else (int(v) if v.isdigit() else v))
        if fpt == 'Snow':
            kw['results_folder'] = '/tmp'
        with contextlib.redirect_stdout(io.StringIO()):
            gd = SNGD(unet, image_size=(32, 32) if fpt == 'Snow' else 32, device_of_kernel='cuda', channels=3, timesteps=int(T),
                      loss_type='l1', forward_process_type=fpt, train_routine='Final', sampling_routine=samp, **kw).cuda()
        if fpt == 'Decolorization':
            X0, Xt, _, _ = gd.all_sample(batch_size=3, img=x)
            assert rel(stack(X0), g['all_X0:' + key]) < 4e-3 and rel(stack(Xt), g['all_Xt:' + key]) < 4e-3, key
        F_, B_, img = gd.forward_and_backward(batch_size=3, img=x)
        assert rel(stack(F_), g['fb_F:' + key]) < 1e-5 and rel(stack(B_), g['fb_B:' + key]) < 4e-3 and rel(img, g['fb_img:' + key]) < 4e-3, key


@pytest.mark.parametrize('tag,kw', [('residual', dict(residual=True)), ('notime', dict(with_time_emb=False)), ('outdim', dict(out_dim=5))])
def test_unet_constructor_options_match_reference_golden(tag, kw):
    """Unet(residual=True) / Unet(with_time_emb=False) (the drivers' --residual / --remove_time_embed flags) / out_dim:
    forward on the TF32 path (1e-3), forward + every gradient on the fp32 CUDA-core path against the reference"""
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.ops import CONV_SIMT
    g = load('unet_options_small')
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3, **kw)
    pre = tag + ':sd:'
    base = {k[3:]: v for k, v in load('unet_small').items() if k.startswith('sd:')}
    extra = {k[len(pre):]: v for k, v in g.items() if k.startswith(pre)}
    u.load_state_dict({k: extra.get(k, base.get(k)) for k in u.state_dict()})
    u = u.cuda()
    x, t = g['x'].cuda(), g['t'].cuda()
    with torch.no_grad():
        assert rel(u(x, t), g[tag + ':y']) < 1e-3
    u.engine.conv_impl = CONV_SIMT
    y = u(x, t)
    assert rel(y.detach(), g[tag + ':y']) < 2e-5
    target = (g['tgt5'] if tag == 'outdim' else g['x'].flip(0)).cuda()
    loss = ((target - y) ** 2).mean()
    assert abs(loss.item() - g[tag + ':loss'].item()) < 2e-5
    loss.backward()
    torch.cuda.synchronize()
    worst = (-1.0, '')
    for n, p_ in u.named_parameters():
        gr = p_.grad.reshape(-1).cpu()
        worst = max(worst, (rel(gr[::max(1, gr.numel() // 256)], g[tag + ':gsub:' + n]), n))
    assert worst[0] < 5e-4, worst


def test_evaluation_routines_on_the_gpu(unet, tmp_path, monkeypatch):
    """the Trainer's evaluation methods (evaluation.py) over the real engine: files of `test_from_data`, the metric dictionary of
    `fid_distance_decrease_from_manifold` equal to metrics recomputed from `all_sample`, SSIM on CUDA tensors equal to the CPU
    value"""
    import os
    import numpy as np
    from PIL import Image
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.evaluation import ssim, rmse
    monkeypatch.chdir(tmp_path)
    rng = np.random.RandomState(0)
    (tmp_path / 'data').mkdir()
    for i in range(9):
        Image.fromarray(rng.randint(0, 256, (32, 32, 3), dtype=np.uint8)).save(str(tmp_path / 'data' / f'{i:02d}.png'))
    gd = cdm.GaussianDiffusion(unet, image_size=32, device_of_kernel='cuda', channels=3, timesteps=3, kernel_std=0.15, kernel_size=5,
                               blur_routine='Exponential_reflect', sampling_routine='x0_step_down').cuda()
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, str(tmp_path / 'data'), image_size=32, train_batch_size=4, results_folder=str(tmp_path / 'res'), shuffle=False)
        X0s, Xts = tr.test_from_data('t')
        out = tr.fid_distance_decrease_from_manifold(None, start=0, end=4, bs=4, sanity_check=0)
    assert len(X0s) == 4 and len(Xts) == 3
    for n in ('og-t.png', 'sample-0-t-x0.png', 'sample-2-t-xt.png', 'Gif-t-x0.gif'):
        assert (tmp_path / 'res' / n).exists(), n
    og = torch.stack([tr.ds[i] for i in range(1, 5)]).cuda()
    A0, At = tr.ema_model.all_sample(batch_size=4, img=og)
    u = lambda t: (t.float().cpu() + 1) * 0.5
    assert out['blurred']['rmse'] == pytest.approx(float(rmse(u(og), u(At[0]))), abs=1e-5)       # the degradation is exact
    assert out['deblurred']['ssim'] == pytest.approx(float(ssim(u(og), u(A0[-1]), data_range=1)), abs=5e-3)   # two TF32 runs
    a, b = torch.rand(3, 3, 40, 40), torch.rand(3, 3, 40, 40)
    assert float(ssim(a.cuda(), b.cuda(), data_range=1)) == pytest.approx(float(ssim(a, b, data_range=1)), abs=1e-5)


@OPT_IN
def test_batched_repack_matches_the_single_launches():
    """csrc/repack.cu (one launch for all weight repacks / packed-gradient unpacks, COLDDIFF_BATCHED_REPACK): bit-exact against the single-weight entry points on a job table that takes every branch,
    then the same Unet gradients with the switch on and off (float atomics in the weight-gradient kernels: TF32-level tolerance)"""
    from cold_diffusion_models_b200 import ops, engine
    from test_repack_batched import _job_set
    from test_grads_gpu import _grads
    for kind in ('pack', 'unpack'):
        res = []
        for batched in (False, True):
            gen = torch.Generator().manual_seed(11)
            batch, bufs = ops.RepackBatch(kind), []
            for shape, taps, mode, tr, rnd in _job_set(kind):
                O, I = (shape[1], shape[0]) if tr else (shape[0], shape[1])
                w = torch.randn(shape, generator=gen).cuda()
                n, k = (O, I) if mode == 0 else (I, O)
                packed = torch.randn(len(taps), n, k, generator=gen).cuda()
                if kind == 'pack':
                    if batched:
                        batch.add(w, taps, packed, shape=shape, mode=mode, transposed_conv=tr, round_tf32=rnd)
                    else:
                        ops.pack_weight(w, taps, mode=mode, transposed_conv=tr, round_tf32=bool(rnd), out=packed)
                else:
                    if batched:
                        batch.add(packed, taps, w, shape=shape, transposed_conv=tr)
                    else:
                        ops.unpack_wgrad(packed, taps, w, transposed_conv=tr, accumulate=True)
                bufs.append((w, packed))
            batch.run(accumulate=True, clear_src=False)
            torch.cuda.synchronize()
            res.append(bufs)
        for j, ((w0, p0), (w1, p1)) in enumerate(zip(*res)):
            assert torch.equal(w0, w1) and torch.equal(p0, p1), (kind, j)
    g = load('unet_small')
    sd = {k[3:]: v for k, v in g.items() if k.startswith('sd:')}
    grads = []
    try:
        for batched in (False, True):
            engine.batched_repack(batched)
            u = make_unet(32, (1, 2), 3, sd)
            for _ in range(2):                                  # the second pass relies on the buffers the first unpack cleared
                _grads(u, g['x'], g['t'], g['target'], 1)
            grads.append({n: p.grad.detach().clone() for n, p in u.named_parameters()})
    finally:
        engine.batched_repack(False)
    for n in grads[0]:
        assert rel(grads[1][n], grads[0][n]) < 2e-3, n


@OPT_IN
def test_linattn_staged_kernels_match_the_default_ones():
    """csrc/linattn_small.cu (cd_linattn_set_staged / COLDDIFF_LINATTN_STAGED): same arithmetic order as the default kernels, so weff / dctxn / rowdot are bit-identical and dW_out (float atomics over
    the batch) agrees to rounding"""
    import ctypes as C
    from cold_diffusion_models_b200._lib import lib, ptr, stream, _check
    gen = torch.Generator().manual_seed(3)
    for B, dim in ((32, 64), (8, 512), (3, 100)):
        ctx, ksum = torch.randn(B, 4, 32, 32, generator=gen).cuda(), (1 + 30 * torch.rand(B, 128, generator=gen)).cuda()
        w_out, dweff = (torch.randn(dim, 128, generator=gen) / 11).cuda(), torch.randn(B, dim, 128, generator=gen).cuda()
        res = []
        try:
            for staged in (0, 1):
                lib.cd_linattn_set_staged(staged)
                weff = [torch.full((B, dim, 128), 7.0).cuda() for _ in range(2)]
                for rnd in (0, 1):
                    _check(lib.cd_linattn_weff(ptr(ctx), ptr(ksum), ptr(w_out), B, dim, C.c_float(0.17), rnd, ptr(weff[rnd]), stream()), 'weff')
                dw_out, dctxn, rowdot = torch.zeros(dim, 128).cuda(), torch.full((B, 4, 32, 32), 7.0).cuda(), torch.full((B, 128), 7.0).cuda()
                _check(lib.cd_linattn_bwd_small(ptr(dweff), ptr(ctx), ptr(ksum), ptr(w_out), B, dim, C.c_float(0.17), ptr(dw_out), ptr(dctxn),
                                                ptr(rowdot), stream()), 'bwd_small')
                torch.cuda.synchronize()
                res.append((weff[0], weff[1], dctxn, rowdot, dw_out))
        finally:
            lib.cd_linattn_set_staged(0)
        for i in range(4):
            assert torch.equal(res[0][i], res[1][i]), (B, dim, i)
        assert rel(res[1][4], res[0][4]) < 1e-5, (B, dim)
    # attn_bwd_kv_kernel<REMAP>: one head and four pixel quads per warp; same sums in the same order
    for B, n in ((4, 4096), (2, 1000), (3, 40)):
        qkv = torch.randn(B, n, 384, generator=gen).cuda()
        kmax = qkv[:, :, 128:256].max(dim=1).values.contiguous()
        ksum = torch.exp(qkv[:, :, 128:256] - kmax[:, None, :]).sum(dim=1).contiguous()
        dctxn, rowdot = torch.randn(B, 4, 32, 32, generator=gen).cuda(), torch.randn(B, 128, generator=gen).cuda()
        outs = []
        try:
            for staged in (0, 1):
                lib.cd_linattn_set_staged(staged)
                dqkv = torch.full((B, n, 384), 7.0, device='cuda')
                _check(lib.cd_linattn_bwd_kv(ptr(qkv), 384, B, n, ptr(kmax), ptr(ksum), ptr(dctxn), ptr(rowdot), ptr(dqkv), 384, stream()), 'bwd_kv')
                torch.cuda.synchronize()
                outs.append(dqkv)
        finally:
            lib.cd_linattn_set_staged(0)
        assert torch.equal(outs[0], outs[1]), (B, n)
        # context_kernel<PRELOAD>: same values and partial sums; float atomics across blocks -> agreement to rounding
        cres = []
        try:
            for staged in (0, 1):
                lib.cd_linattn_set_staged(staged)
                km, ks, cx = torch.empty(B, 128, device='cuda'), torch.empty(B, 128, device='cuda'), torch.empty(B, 4, 32, 32, device='cuda')
                _check(lib.cd_linattn_context(ptr(qkv), 384, B, n, ptr(km), ptr(ks), ptr(cx), stream()), 'context')
                torch.cuda.synchronize()
                cres.append((km, ks, cx))
        finally:
            lib.cd_linattn_set_staged(0)
        assert torch.equal(cres[0][0], cres[1][0]) and rel(cres[1][1], cres[0][1]) < 1e-5 and rel(cres[1][2], cres[0][2]) < 1e-5, (B, n)


@OPT_IN
def test_layernorm_multi_pixel_forward_matches_the_default_kernel():
    """csrc/layernorm_multi.cu (cd_layernorm_set_multi): same per-pixel
    arithmetic as layernorm_kernel<1> -> bit-identical output and statistics"""
    import ctypes as C
    from cold_diffusion_models_b200._lib import lib, ptr, stream, _check
    gen = torch.Generator().manual_seed(4)
    for npix, Cc, pad in ((32 * 128 * 128, 64, 0), (32 * 64 * 64 + 3, 128, 8), (5000, 32, 4)):
        ld = Cc + pad
        x = (torch.randn(npix, ld, generator=gen) * 3 + 0.5).cuda()
        gam, bet = (1 + 0.2 * torch.randn(Cc, generator=gen)).cuda(), (0.1 * torch.randn(Cc, generator=gen)).cuda()
        res = []
        try:
            for pp in (0, 2, 4):
                lib.cd_layernorm_set_multi(pp)
                y, st = torch.full((npix, ld), 7.0, device='cuda'), torch.full((npix, 2), 7.0, device='cuda')
                _check(lib.cd_layernorm_fwd(ptr(x), ld, C.c_int64(npix), Cc, ptr(gam), ptr(bet), C.c_float(1e-5), ptr(y), ld, ptr(st), 1, stream()), 'ln')
                torch.cuda.synchronize()
                res.append((y, st))
        finally:
            lib.cd_layernorm_set_multi(0)
        for y, st in res[1:]:
            assert torch.equal(y, res[0][0]) and torch.equal(st, res[0][1]), (npix, Cc)


@OPT_IN
def test_image_edge_kernels_with_preloaded_staging_match_the_default():
    """cd_conv_simt_set_preload: the 3-channel image-edge convolution and its
    weight gradient with all receptive-field loads of a chunk in flight; outputs bit-identical, weight gradients (float atomics over
    blocks) to rounding"""
    from cold_diffusion_models_b200 import ops
    from cold_diffusion_models_b200._lib import lib
    gen = torch.Generator().manual_seed(8)
    for Cout, k, B, H in ((128, 3, 8, 128), (64, 1, 8, 128), (128, 3, 3, 32)):
        x = torch.zeros(B, H, H, 4)
        x[..., :3] = torch.randn(B, H, H, 3, generator=gen)
        x = x.cuda()
        taps = ops.taps_conv(k, k // 2)
        wp, bias = (torch.randn(len(taps), Cout, 3, generator=gen) / 3).cuda(), torch.randn(Cout, generator=gen).cuda()
        dy = torch.randn(B, H, H, Cout, generator=gen).cuda()
        res = []
        try:
            for pre in (0, 1):
                lib.cd_conv_simt_set_preload(pre)
                out, pa = torch.full((B, H, H, Cout), 7.0, device='cuda'), torch.full((B, H, H, Cout), 7.0, device='cuda')
                d = ops.make_conv_desc([(ops.View(x, 0, 3), taps, wp, False)], ops.View(out), (B, H, H), Cout=Cout, bias=bias, act=ops.ACT_GELU,
                                       out2=ops.View(pa))
                ops.conv_fwd(d, ops.CONV_SIMT)
                dw, db = torch.zeros(len(taps), Cout, 3, device='cuda'), torch.zeros(Cout, device='cuda')
                dd = ops.make_conv_desc([(ops.View(x, 0, 3), taps, dw, False)], ops.View(dy), (B, H, H), Cout=Cout)
                ops.conv_wgrad(dd, ops.View(dy), dw, db, impl=ops.CONV_SIMT)
                torch.cuda.synchronize()
                res.append((out, pa, dw, db))
        finally:
            lib.cd_conv_simt_set_preload(0)
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), (Cout, k)
        assert rel(res[1][2], res[0][2]) < 1e-5 and rel(res[1][3], res[0][3]) < 1e-5, (Cout, k)
    # the same switch: final 1x1 projection NHWC -> NCHW through a shared-memory tile (csrc/final_proj.cu), bit-identical
    import ctypes as C
    from cold_diffusion_models_b200._lib import ptr, stream, _check
    for B, H, Cc, Co in ((32, 128, 64, 3), (3, 17, 64, 3), (2, 16, 32, 1)):
        x = torch.randn(B, H, H, Cc, generator=gen).cuda()
        w, bias = (torch.randn(Co, Cc, generator=gen) / 8).cuda(), torch.randn(Co, generator=gen).cuda()
        r = torch.randn(B, Co, H, H, generator=gen).cuda()
        outs = []
        try:
            for pre in (0, 1):
                lib.cd_conv_simt_set_preload(pre)
                o = torch.full((B, Co, H, H), 7.0, device='cuda')
                _check(lib.cd_conv1x1_to_nchw(ptr(x), Cc, B, H, H, Cc, ptr(w), ptr(bias), Co, ptr(r), ptr(o), stream()), 'final projection')
                torch.cuda.synchronize()
                outs.append(o)
        finally:
            lib.cd_conv_simt_set_preload(0)
        assert torch.equal(outs[0], outs[1]), (B, H, Cc, Co)
        # ... and its backward with four pixels per trip in flight: same order of every sum per thread; dW / db go through float atomics
        bres = []
        try:
            for pre in (0, 1):
                lib.cd_conv_simt_set_preload(pre)
                dx, dw, db = torch.full((B, H, H, Cc), 7.0, device='cuda'), torch.zeros(Co, Cc, device='cuda'), torch.zeros(Co, device='cuda')
                _check(lib.cd_conv1x1_to_nchw_bwd(ptr(r), ptr(x), Cc, B, H, H, Cc, ptr(w), Co, ptr(dx), Cc, ptr(dw), ptr(db), stream()), 'final projection bwd')
                torch.cuda.synchronize()
                bres.append((dx, dw, db))
        finally:
            lib.cd_conv_simt_set_preload(0)
        assert torch.equal(bres[0][0], bres[1][0]) and rel(bres[1][1], bres[0][1]) < 1e-5 and rel(bres[1][2], bres[0][2]) < 1e-5, (B, H, Cc, Co)
    # ... and the float4 variant of the batched column sums (time-conditioning gradient): another summation order, fp32 rounding
    for B, rows, Cc in ((32, 16384, 64), (3, 300, 128), (2, 256, 512)):
        x = torch.randn(B, rows, Cc, generator=gen).cuda()
        cres = []
        try:
            for pre in (0, 1):
                lib.cd_conv_simt_set_preload(pre)
                o = torch.full((B, Cc + 16), 0.5, device='cuda')
                _check(lib.cd_colsum_batched(ptr(x), Cc, B, C.c_int64(rows), Cc, ptr(o), Cc + 16, stream()), 'colsum_batched')
                torch.cuda.synchronize()
                cres.append(o)
        finally:
            lib.cd_conv_simt_set_preload(0)
        assert rel(cres[1], cres[0]) < 1e-5 and bool((cres[1][:, Cc:] == 0.5).all()), (B, rows, Cc)


@OPT_IN
def test_conv_staged_epilogue_matches_the_row_epilogue():
    """runs _conv_staged_epilogue_body in a child process with a time limit: a wgmma / mbarrier pipeline that went wrong would spin instead of failing -- that must not take the session's
    CUDA context (and the tests after it) with it"""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r, %r]; import test_helpers_and_variants_gpu as t; t._conv_staged_epilogue_body(); print('STAGED_OK')"
            % (os.path.dirname(here), os.path.join(os.path.dirname(here), 'oracle'), here))
    try:
        r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=600)
    except subprocess.TimeoutExpired as e:
        pytest.fail('staged-epilogue child process hung (killed after 600 s): %s' % str(e.stdout)[-500:])
    assert r.returncode == 0 and 'STAGED_OK' in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])


def _conv_staged_epilogue_body():
    """csrc/conv_epilogue.cuh (cd_conv_tc_set_staged_epilogue): every tensor-core
    convolution case of tests/test_conv_gpu.py again with the line-coalesced epilogue forced on all launches (mode 2: 3/4/6-stage
    kernels with the per-warp staging tiles), then bit-exact against the row epilogue on the store-bound 1x1 shapes in mode 1"""
    import test_conv_gpu as T
    from cold_diffusion_models_b200 import ops
    from cold_diffusion_models_b200._lib import lib
    try:
        lib.cd_conv_tc_set_staged_epilogue(2)
        for case in T.CASES:
            T.test_conv_stride1(ops, case, 'tc')
        T.test_conv_two_sources_channel_slices(ops, 'tc')
        T.test_conv_4x4_stride2_and_transpose(ops, 'tc')
        T.test_conv_per_batch_weights(ops, 'tc')
        gen = torch.Generator().manual_seed(9)
        for (B, Ci, Co, H, W) in ((2, 64, 384, 64, 64), (1, 128, 384, 32, 32), (3, 256, 64, 16, 16), (2, 512, 384, 16, 16)):
            x = torch.randn(B, H, W, Ci, generator=gen).cuda()
            w = (torch.randn(Co, Ci, 1, 1, generator=gen) / Ci ** 0.5).cuda()
            b, r = torch.randn(Co, generator=gen).cuda(), torch.randn(B, H, W, Co, generator=gen).cuda()
            taps = ops.taps_conv(1, 0)
            pw = ops.pack_weight(w, taps, round_tf32=False)
            outs = []
            for mode in (0, 1):
                lib.cd_conv_tc_set_staged_epilogue(mode)
                out, pre = torch.full((B, H, W, Co), 7.0, device='cuda'), torch.full((B, H, W, Co), 7.0, device='cuda')
                d = ops.make_conv_desc([(ops.View(x), taps, pw, False)], ops.View(out), (B, H, W), Cout=Co, bias=b, resid=ops.View(r),
                                       act=ops.ACT_GELU, out2=ops.View(pre), round_tf32=True)
                T.run_conv(ops, d, 'tc')
                outs.append((out, pre))
            assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), (B, Ci, Co, H, W)
    finally:
        lib.cd_conv_tc_set_staged_epilogue(0)


@OPT_IN
def test_fp16_operand_probe_agrees_with_the_tf32_kernel():
    """cd_conv_fwd_f16_probe (experimental, not used by the engine; tools/conv_f16_probe.py): kind::f16 MMAs on FP16 operands give
    the TF32 kernel's result when both multiply the same (FP16-representable) values.  Child process with a time limit: tensor-core
    code that has never run."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, os.path.join(root, 'tools', 'conv_f16_probe.py'), '--check'], capture_output=True, text=True, timeout=600)
    except subprocess.TimeoutExpired as e:
        pytest.fail('fp16 probe hung (killed after 600 s): %s' % str(e.stdout)[-500:])
    assert r.returncode == 0 and 'F16_PROBE_OK' in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])


def test_depthwise_kernels_with_tma_staged_tiles_match_the_ldgsts_kernels_and_torch():
    """csrc/dwconv_tma.cu (cd_dwconv7_set_tma, the default): the depthwise 7x7 forward / data gradient (flip) / weight gradient
    with tiles staged by one bulk tensor copy (border zero fill by the tensor map) against the LDGSTS kernels of elementwise.cu
    (same per-thread arithmetic: forward bit-identical) and against torch's depthwise convolution (DB:145) in fp32"""
    import torch.nn.functional as F
    from cold_diffusion_models_b200._lib import lib, ptr, stream, _check
    gen = torch.Generator().manual_seed(11)
    for (B, H, W, Cc, pad) in ((2, 32, 32, 64, 0), (3, 16, 48, 32, 4), (1, 128, 128, 64, 0), (2, 16, 16, 96, 32),
                               (32, 64, 64, 128, 0), (32, 32, 32, 256, 0), (32, 16, 16, 512, 0)):     # the config-3 levels at B = 32
        ld = Cc + pad
        x = torch.randn(B, H, W, ld, generator=gen).cuda()
        dh = torch.randn(B, H, W, ld, generator=gen).cuda()
        add = torch.randn(B, H, W, ld, generator=gen).cuda()
        w = (torch.randn(Cc, 1, 7, 7, generator=gen) / 7).cuda()
        bias, cond = torch.randn(Cc, generator=gen).cuda(), torch.randn(B, Cc, generator=gen).cuda()
        xc = x[..., :Cc].permute(0, 3, 1, 2).contiguous()
        ref_f = (F.conv2d(xc, w, bias, padding=3, groups=Cc) + cond[:, :, None, None]).permute(0, 2, 3, 1) + add[..., :Cc]
        ref_d = F.conv_transpose2d(dh[..., :Cc].permute(0, 3, 1, 2).contiguous(), w, padding=3, groups=Cc).permute(0, 2, 3, 1)
        xg = xc.clone().requires_grad_(True); wg = w.clone().requires_grad_(True)
        F.conv2d(xg, wg, None, padding=3, groups=Cc).backward(dh[..., :Cc].permute(0, 3, 1, 2).contiguous())
        ref_w = wg.grad.reshape(Cc, 49)
        res = []
        try:
            for tma in (1, 0):
                lib.cd_dwconv7_set_tma(tma)
                out = torch.full((B, H, W, ld), 7.0, device='cuda'); dx = torch.full((B, H, W, ld), 7.0, device='cuda')
                dw = torch.zeros(Cc, 49, device='cuda')
                _check(lib.cd_dwconv7_fwd(ptr(x), ld, B, H, W, Cc, ptr(w), ptr(bias), ptr(cond), Cc, ptr(out), ld, 0, ptr(add), ld, stream()), 'dw')
                _check(lib.cd_dwconv7_fwd(ptr(dh), ld, B, H, W, Cc, ptr(w), ptr(None), ptr(None), 0, ptr(dx), ld, 1, ptr(None), 0, stream()), 'dw flip')
                for _ in range(2):                      # accumulates (+=)
                    _check(lib.cd_dwconv7_wgrad(ptr(dh), ld, ptr(x), ld, B, H, W, Cc, ptr(dw), stream()), 'dw wgrad')
                torch.cuda.synchronize()
                res.append((out, dx, dw))
        finally:
            lib.cd_dwconv7_set_tma(1)
        case = (B, H, W, Cc, pad)
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), case
        assert torch.all(res[0][0][..., Cc:] == 7.0) and torch.all(res[0][1][..., Cc:] == 7.0), case     # padding columns untouched
        assert rel(res[0][0][..., :Cc], ref_f) < 2e-6 and rel(res[0][1][..., :Cc], ref_d) < 2e-6, case
        assert rel(res[0][2], 2 * ref_w) < 1e-5 and rel(res[1][2], 2 * ref_w) < 1e-5, case
