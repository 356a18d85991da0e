"""CUDA-graph training (`Trainer.enable_cuda_graph`): from one saved state and seeds, K optimizer steps replayed from a graph
compute what K eager steps compute, for one Trainer per package.

The backward's float-atomic reductions make eager runs differ in the last bits, so the graphed run is held to the spread of
the eager runs: its relative L2 distance from a first eager run (per-step losses, parameters, EMA weights, Adam m and v) is at
most max(3 x the larger distance of two more eager runs, 1e-6) (one such distance alone is a noisy estimate of the spread, and
falls short of it by more than 3x now and then), and its first loss is bit-identical (16² images, B = 2: the loss kernel
adds two block partials, an order-free sum).  Two negative controls (dropout seeds
frozen at the capture; t draws shifted by one step) land at least 10x past that bound."""
import contextlib
import io

import numpy as np
import pytest
import torch

import cold_diffusion_models_b200 as cdm
from cold_diffusion_models_b200 import _lib, train_graph

pytestmark = pytest.mark.gpu

K, A, B = 4, 2, 2
SEED = 1234


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


def small_unet(seed=0):
    torch.manual_seed(seed)
    with quiet():
        return cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)


def small_model(seed=0):
    torch.manual_seed(seed)
    return cdm.Model(resolution=16, in_channels=3, out_ch=3, ch=32, ch_mult=(1, 2), num_res_blocks=2, attn_resolutions=(8,),
                     dropout=0.1)


def make(case, tmp_path):
    """-> (trainer, image size, two-input batches?)"""
    from cold_diffusion_models_b200 import (deblurring_diffusion_pytorch as db, denoising_diffusion_pytorch as dn,
                                            resolution_diffusion_pytorch as rs, defading_diffusion_pytorch as df,
                                            defading_generation_diffusion_pytorch as dg, demixing_diffusion_pytorch as dm,
                                            snowification_diffusion as sn)
    kw = dict(train_batch_size=B, train_lr=1e-3, gradient_accumulate_every=A, step_start_ema=0, update_ema_every=1,
              results_folder=str(tmp_path), dataset='synthetic')
    S, extra, pair = 16, (), False
    if case == 'deblur_unet':
        gd = db.GaussianDiffusion(small_unet(), image_size=16, device_of_kernel='cuda', channels=3, timesteps=4, kernel_std=0.15,
                                  kernel_size=7, blur_routine='Exponential_reflect')
        T = db.Trainer
    elif case == 'deblur_model':
        gd = db.GaussianDiffusion(small_model(), image_size=16, device_of_kernel='cuda', channels=3, timesteps=6, kernel_std=0.1,
                                  kernel_size=3, blur_routine='Special_6_routine')
        T = db.Trainer
    elif case == 'denoise':
        gd, T = dn.GaussianDiffusion(small_unet(), image_size=16, channels=3, timesteps=5), dn.Trainer
    elif case == 'resolution':
        gd, T = rs.GaussianDiffusion(small_unet(), image_size=16, device_of_kernel='cuda', channels=3, timesteps=4), rs.Trainer
    elif case == 'defading':
        gd = df.GaussianDiffusion(small_unet(), image_size=16, device_of_kernel='cuda', channels=3, timesteps=4, kernel_std=0.1,
                                  fade_routine='Random_Incremental')
        T = df.Trainer
    elif case == 'defading_generation':
        gd, T = dg.GaussianDiffusion(small_unet(), image_size=16, channels=3, timesteps=4, kernel_std=0.6, initial_mask=3), dg.Trainer
    elif case == 'demixing':
        gd, T, extra, pair = dm.GaussianDiffusion(small_unet(), image_size=16, channels=3, timesteps=4), dm.Trainer, (None,), True
    elif case in ('decolor', 'decolor_lab'):
        lab = case == 'decolor_lab'
        gd = sn.GaussianDiffusion(small_unet(), image_size=16, device_of_kernel='cuda', channels=3, timesteps=4,
                                  forward_process_type='Decolorization', decolor_routine='Linear', decolor_total_remove=True,
                                  to_lab=lab)
        T = sn.Trainer
        kw['to_lab'] = lab
    elif case == 'snow':
        gd = sn.GaussianDiffusion(small_unet(), image_size=(16, 16), device_of_kernel='cuda', channels=3, timesteps=4,
                                  forward_process_type='Snow', random_snow=True, single_snow=True, batch_size=B)
        T = sn.Trainer
    else:
        raise KeyError(case)
    gd = gd.cuda()
    if T is not sn.Trainer:
        kw['image_size'] = S
    with quiet():
        tr = T(gd, None, *extra, **kw)
    # Adam's first steps are lr * sign(g) for every element whose |g| is far above eps, including elements whose gradient is
    # as small as the rounding of the float-atomic reductions: their sign differs from run to run, and so two eager runs fall
    # apart by chance, by far more than the rounding.  eps = 1e-3 makes the step of those elements proportional to their
    # gradient, so that runs differ by what the rounding explains, and keeps every kernel of the step in use.
    tr.opt.param_groups[0]['eps'] = 1e-3
    # and the L2 loss (every package has it): the L1 loss's gradient sign(x_recon - x_start) jumps for the residuals the
    # rounding moves across zero
    gd.loss_type = 'l2'
    return tr, S, pair


def batches(S, pair, n, seed=5):
    g = torch.Generator().manual_seed(seed)
    mk = lambda: torch.rand(B, 3, S, S, generator=g) * 2 - 1
    return [(mk(), mk()) if pair else mk() for _ in range(n)]


def snapshot(tr):
    e, ee = tr._unet.engine, tr._ema_unet.engine
    return dict(p=e.flat_param.clone(), ema=ee.flat_param.clone(), m=tr.opt.m.clone(), v=tr.opt.v.clone(), t=tr.opt.t,
                g=e.flat_grad.clone(), step=tr.step)


def restore(tr, s):
    e, ee = tr._unet.engine, tr._ema_unet.engine
    e.flat_param.copy_(s['p']); ee.flat_param.copy_(s['ema'])
    tr.opt.m.copy_(s['m']); tr.opt.v.copy_(s['v']); tr.opt.t = s['t']
    e.flat_grad.copy_(s['g']); tr.step = s['step']
    e.mark_weights_dirty(); ee.mark_weights_dirty()


def run(tr, s0, data, graphed, shift_t=False):
    """K optimizer steps from state s0 and the seeds -> (per-step losses, params, EMA, m, v)"""
    restore(tr, s0)
    torch.manual_seed(SEED)
    np.random.seed(SEED)
    if shift_t:          # the draws of one step's t (one per micro-batch) are skipped: every later draw moves
        for _ in range(A):
            torch.randint(0, 4, (B,), device='cuda')
    tr.enable_cuda_graph(graphed)
    losses = []
    for k in range(K):
        losses.append(tr.train_step(batches=data[k * A:(k + 1) * A]).clone())
        tr.step += 1
    tr.enable_cuda_graph(False)
    torch.cuda.synchronize()
    e, ee = tr._unet.engine, tr._ema_unet.engine
    return dict(loss=torch.stack(losses), p=e.flat_param.clone(), ema=ee.flat_param.clone(), m=tr.opt.m.clone(), v=tr.opt.v.clone())


def dist(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def distances(r, ref):
    return {k: dist(r[k], ref[k]) for k in ref}


CASES = ['deblur_unet', 'deblur_model', 'denoise', 'resolution', 'defading', 'defading_generation', 'demixing', 'decolor',
         'decolor_lab', 'snow']


@pytest.mark.parametrize('case', CASES)
def test_graphed_steps_compute_what_eager_steps_compute(case, tmp_path):
    tr, S, pair = make(case, tmp_path)
    data = batches(S, pair, K * A)
    s0 = snapshot(tr)
    e1 = run(tr, s0, data, False)
    eager = [distances(run(tr, s0, data, False), e1) for _ in range(2)]
    gr = run(tr, s0, data, True)
    assert bool(torch.isfinite(e1['loss']).all())
    assert torch.equal(gr['loss'][0], e1['loss'][0]), (case, gr['loss'][0].item(), e1['loss'][0].item())
    d2 = {k: max(d[k] for d in eager) for k in eager[0]}
    dg = distances(gr, e1)
    bound = {k: max(3 * d2[k], 1e-6) for k in d2}
    for k in bound:
        assert dg[k] <= bound[k], (case, k, dg[k], bound[k], d2[k])
    controls = []
    if case == 'deblur_unet':
        controls.append(('t shifted by one step', run(tr, s0, data, True, shift_t=True)))
    if case == 'deblur_model':
        stage = train_graph.HostDraws.stage

        def stage_once(self):                       # the seeds staged for the first replay are kept: the masks stay frozen
            if not getattr(self, '_frozen', False):
                self._frozen = True
                stage(self)
        train_graph.HostDraws.stage = stage_once
        try:
            controls.append(('dropout seeds frozen at capture', run(tr, s0, data, True)))
        finally:
            train_graph.HostDraws.stage = stage
    for name, r in controls:
        dc = distances(r, e1)
        assert dc['p'] >= 10 * bound['p'] and dc['loss'] >= 10 * bound['loss'], (case, name, dc, bound)


def test_replays_draw_new_dropout_masks_equal_to_the_eager_masks(tmp_path):
    """lr = 0 keeps the weights: each step's loss is then a function of its batch, t and dropout masks only, and the graphed
    losses equal the eager ones bit for bit.  The seeds staged for two consecutive replays differ and are the host draws the
    eager steps make."""
    tr, S, pair = make('deblur_model', tmp_path)
    tr.opt.param_groups[0]['lr'] = 0.0
    data = batches(S, pair, 3 * A)
    s0 = snapshot(tr)
    losses = {}
    for graphed in (False, True):
        restore(tr, s0)
        torch.manual_seed(SEED)
        tr.enable_cuda_graph(graphed)
        out, seeds = [], []
        for k in range(3):
            out.append(tr.train_step(batches=data[k * A:(k + 1) * A]).item())
            if graphed:
                d = next(iter(tr._step_graphs.values())).draws
                seeds.append(d.seeds[:d.nseeds].cpu())
        losses[graphed] = out
    tr.enable_cuda_graph(False)
    assert losses[True] == losses[False], losses
    n = seeds[0].numel()
    assert n == A * 12 and not torch.equal(seeds[0], seeds[1])          # 12 ResnetBlocks with dropout per micro-batch
    torch.manual_seed(SEED)
    expect = [int(torch.randint(0, 2 ** 62, (1,)).item()) for _ in range(3 * n)]
    for k in range(3):
        assert seeds[k].tolist() == expect[k * n:(k + 1) * n]


def test_load_keeps_the_graph_and_the_next_step_equals_the_eager_step(tmp_path):
    tr, S, pair = make('deblur_unet', tmp_path)
    data = batches(S, pair, 3 * A)
    tr.save()
    path = str(tmp_path / 'model.pt')
    tr.enable_cuda_graph(True)
    for k in range(2):
        tr.train_step(batches=data[k * A:(k + 1) * A])
    graph = next(iter(tr._step_graphs.values()))
    with quiet():
        tr.load(path)
    torch.manual_seed(SEED)
    lg = tr.train_step(batches=data[2 * A:]).item()
    assert len(tr._step_graphs) == 1 and next(iter(tr._step_graphs.values())) is graph
    tr.enable_cuda_graph(False)
    with quiet():
        tr.load(path)
    torch.manual_seed(SEED)
    le = tr.train_step(batches=data[2 * A:]).item()
    assert lg == le, (lg, le)


def test_a_new_micro_batch_shape_captures_a_second_graph(tmp_path):
    tr, S, pair = make('deblur_unet', tmp_path)
    tr.enable_cuda_graph(True)
    tr.train_step(batches=batches(S, pair, A))
    assert len(tr._step_graphs) == 1
    g = torch.Generator().manual_seed(9)
    loss = tr.train_step(batches=[torch.rand(3, 3, S, S, generator=g) * 2 - 1 for _ in range(A)])
    assert len(tr._step_graphs) == 2 and bool(torch.isfinite(loss))
    tr.train_step(batches=batches(S, pair, A))
    assert len(tr._step_graphs) == 2


def test_disabling_returns_to_eager_launches(tmp_path):
    tr, S, pair = make('deblur_unet', tmp_path)
    data = batches(S, pair, A)
    counts = []
    for switch in (None, True, None, False):        # eager, capture, replay, eager again
        if switch is not None:
            tr.enable_cuda_graph(switch)
        torch.cuda.synchronize()
        _lib.reset_launch_count()
        tr.train_step(batches=data)
        counts.append(_lib.launch_count())
    eager, capture, replay, eager_again = counts
    assert tr._step_graphs is None
    assert replay < eager // 4 and eager_again == eager, counts


def test_changing_requires_grad_after_the_first_step_still_raises(tmp_path):
    tr, S, pair = make('deblur_unet', tmp_path)
    data = batches(S, pair, A)
    tr.enable_cuda_graph(True)
    tr.train_step(batches=data)
    next(tr._unet.parameters()).requires_grad_(False)
    with pytest.raises(ValueError, match='requires_grad'):
        tr.train_step(batches=data)


def test_world_size_two_is_refused(tmp_path):
    tr, S, pair = make('deblur_unet', tmp_path)
    tr._world = 2
    with pytest.raises(ValueError, match='single process'):
        tr.enable_cuda_graph(True)
    assert tr._step_graphs is None


@pytest.mark.parametrize('case', ['deblur_unet', 'deblur_model'])
def test_peak_memory_of_the_graphed_step(case, tmp_path):
    """the graph keeps the activations of all A micro-batches in its private pool: its peak is reported beside the eager
    step's (each over two steps, the first one of the graphed run being the capture)"""
    tr, S, pair = make(case, tmp_path)
    data = batches(S, pair, A)
    peaks = {}
    for graphed in (False, True):
        tr.enable_cuda_graph(graphed)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        for _ in range(2):
            tr.train_step(batches=data)
        torch.cuda.synchronize()
        peaks[graphed] = torch.cuda.max_memory_allocated()
    tr.enable_cuda_graph(False)
    print('\n%s, B = %d, A = %d: peak device memory allocated, eager %.1f MiB, graphed %.1f MiB'
          % (case, B, A, peaks[False] / 2 ** 20, peaks[True] / 2 ** 20))
    assert peaks[True] >= peaks[False] > 0
