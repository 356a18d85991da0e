"""The DDPM `Model` (BASELINE config 2's network: ch = 128, ch_mult = (1, 2, 2, 2), two ResNet blocks per level, attention at
16², dropout 0.1) replayed as a CUDA graph, `Model.engine.enable_cuda_graph(True)`:

- bit equality with the eager inference forward at 32² (B = 1, 4, 128) and 256² (B = 2, the split GroupNorm), per-sample t,
  and with_time_emb=False without t;
- a graph captured earlier follows the weights: one Trainer optimizer step (Adam + EMA), load_state_dict in place, and the
  re-captures that flatten_params and load_state_dict(assign=True) force;
- one graph per batch size, separate graphs for a deep copy (the EMA model), the switch off returns to eager, and the autograd
  path is never graphed;
- a graphed 3-step sample of the deblurring package against float64 (oracle/deblur_oracle.py around oracle/model2_oracle.py),
  each comparison with a negative control and a bound of at most 3x the value measured on an H100 80GB HBM3 (700 W) beside it;
  the snowification sample with two graphed `Model`s equals its eager run.

Set COLDDIFF_TEST_METRICS=<file> to write every value and control as JSON.  On that card the file runs in about 20 s and
peaks at 2.6 GiB of device memory (the B = 128 forward)."""
import contextlib
import copy
import gc
import io
import json
import math
import os

import pytest
import torch

import deblur_oracle as DO
import model2_oracle as MO

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
NET = dict(ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2, attn_resolutions=(16,), dropout=0.1)
CONFIG2 = dict(image_size=32, channels=3, timesteps=50, kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine')
_METRICS = {}


# --------------------------------------------------------------------------------------------------------------------------
# fixtures and helpers
# --------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module', autouse=True)
def _metrics_file():
    yield
    path = os.environ.get('COLDDIFF_TEST_METRICS')
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        _METRICS['peak_device_memory_gb'] = torch.cuda.max_memory_allocated() / 2 ** 30
        with open(path, 'w') as f:
            json.dump(_METRICS, f, indent=1, sort_keys=True)


@pytest.fixture(autouse=True)
def _free_between_tests():
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _fp64_time_embedding(monkeypatch):
    """oracle/model2_oracle.py builds the sinusoidal table in float32 on the CPU; the references here run in float64 on the GPU"""
    def temb(t, dim):
        half = dim // 2
        f = torch.exp(torch.arange(half, dtype=F64, device=DEV) * -(math.log(10000) / (half - 1)))
        e = t.to(DEV, F64)[:, None] * f[None, :]
        return torch.cat([torch.sin(e), torch.cos(e)], dim=1)
    monkeypatch.setattr(MO, 'timestep_embedding', temb)


class Checks:
    """collects every (value < bound) and (control > bound) of one test, records them, and fails at the end with all of them"""

    def __init__(self, test):
        self.test, self.fails = test, []

    def __call__(self, name, value, bound, control=None):
        _METRICS['%s::%s' % (self.test, name)] = dict(value=float(value), bound=float(bound),
                                                      control=None if control is None else float(control))
        if not float(value) < bound:
            self.fails.append('%s: %.3e >= bound %.3e' % (name, value, bound))
        if control is not None and not float(control) > bound:
            self.fails.append('%s: negative control %.3e does not exceed the bound %.3e' % (name, control, bound))

    def require(self, name, ok):
        if not ok:
            self.fails.append(name)

    def done(self):
        assert not self.fails, '\n'.join(self.fails)


def rel(a, b):
    a, b = a.to(F64), b.to(F64)
    return ((a - b).norm() / (b.norm() + 1e-300)).item()


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _model(S, seed=3, **kw):
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(seed)
    return cdm.Model(resolution=S, in_channels=3, out_ch=3, **dict(NET, **kw)).to(DEV)


def _inputs(B, S, seed, n=3):
    g = gen(seed)
    return [(torch.rand(B, 3, S, S, generator=g, device=DEV) * 2 - 1, torch.randint(0, 50, (B,), generator=g, device=DEV))
            for _ in range(n)]


def _eager(m, x, t=None):
    """the eager inference forward of a network with the same weights: a deep copy with the switch off"""
    ref = copy.deepcopy(m)
    ref.engine.enable_cuda_graph(False)
    with torch.no_grad():
        return ref(x, t) if t is not None else ref(x)


def _deblur(m):
    import cold_diffusion_models_b200 as cdm
    return cdm.GaussianDiffusion(m, device_of_kernel='cuda', loss_type='l1', train_routine='Final', sampling_routine='x0_step_down',
                                 **CONFIG2).to(DEV)


# ==========================================================================================================================
# bit equality with the eager forward
# ==========================================================================================================================
@pytest.mark.parametrize('S,B', [(32, 1), (32, 4), (32, 128), (256, 2)])
def test_replay_equals_eager(S, B):
    m = _model(S).eval()
    ins = _inputs(B, S, seed=S + B)
    with torch.no_grad():
        eager = [m(x, t) for x, t in ins]
        m.engine.enable_cuda_graph(True)
        graphed = [m(x, t) for x, t in ins]
        graphs = len(m.engine._graphs)
        m.engine.enable_cuda_graph(False)
    torch.cuda.synchronize()
    assert graphs == 1
    for i, (a, b) in enumerate(zip(eager, graphed)):
        assert torch.equal(a, b), 'replay %d differs from the eager forward (max %.3e)' % (i, (a - b).abs().max().item())
    assert not torch.equal(graphed[0], graphed[1])


def test_replay_without_time_embedding():
    """the snowification one-shot model: with_time_emb=False and no t (the time path runs at t = 0)"""
    m = _model(32, seed=4, with_time_emb=False).eval()
    ins = _inputs(4, 32, seed=7)
    with torch.no_grad():
        eager = [m(x) for x, _ in ins]
        m.engine.enable_cuda_graph(True)
        graphed = [m(x) for x, _ in ins]
        m.engine.enable_cuda_graph(False)
    for a, b in zip(eager, graphed):
        assert torch.equal(a, b)


# ==========================================================================================================================
# weights followed
# ==========================================================================================================================
def test_graph_follows_trainer_step_and_load_state_dict(tmp_path):
    import cold_diffusion_models_b200 as cdm
    B = 4
    m = _model(32, seed=5)
    gd = _deblur(m)
    (x, t), = _inputs(B, 32, seed=8, n=1)
    eng = m.engine
    eng.enable_cuda_graph(True)
    with torch.no_grad():
        y0 = m(x, t)
    # the Trainer flattens the parameters into one buffer (FusedAdamEMA): the graph captured before holds the old addresses
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=32, train_batch_size=B, train_lr=1e-3, train_num_steps=10 ** 9,
                         gradient_accumulate_every=1, ema_decay=0.995, step_start_ema=0, update_ema_every=1,
                         results_folder=str(tmp_path), dataset='synthetic')
    assert len(eng._graphs) == 0, 'flatten_params kept a graph that addresses the old parameter storage'
    with torch.no_grad():
        y1 = m(x, t)
    g1 = eng._graphs[tuple(x.shape)][0]
    assert torch.equal(y1, y0)
    ema = tr.ema_model.denoise_fn
    assert ema.engine.use_cuda_graph and ema.engine is not eng
    with torch.no_grad():
        e1 = ema(x, t)
    # one optimizer step (Adam + EMA through raw pointers): the same graph replays the new weights
    tr.train_step([torch.rand(B, 3, 32, 32, generator=gen(9), device=DEV) * 2 - 1])
    tr.opt.zero_grad()
    with torch.no_grad():
        y2, e2 = m(x, t), ema(x, t)
    assert eng._graphs[tuple(x.shape)][0] is g1
    assert not torch.equal(y2, y1) and not torch.equal(e2, e1), 'the step did not change the output'
    assert torch.equal(y2, _eager(m, x, t)), 'after the optimizer step'
    assert torch.equal(e2, _eager(ema, x, t)), 'EMA model after the optimizer step'
    # load_state_dict copies in place: the same graph replays the loaded weights
    other = _model(32, seed=6).state_dict()
    m.load_state_dict(other)
    with torch.no_grad():
        y3 = m(x, t)
    assert eng._graphs[tuple(x.shape)][0] is g1
    assert torch.equal(y3, _eager(m, x, t)) and not torch.equal(y3, y2), 'after load_state_dict'
    # ... through the enclosing module as well (Trainer.load, reset_parameters)
    gd.load_state_dict(tr.ema_model.state_dict())
    with torch.no_grad():
        y4 = m(x, t)
    assert torch.equal(y4, e2), 'after GaussianDiffusion.load_state_dict'
    # assign=True rebinds the parameters: the graph is captured again
    m.load_state_dict({k: v.clone() for k, v in other.items()}, assign=True)
    with torch.no_grad():
        y5 = m(x, t)
    assert eng._graphs[tuple(x.shape)][0] is not g1
    assert torch.equal(y5, y3), 'after load_state_dict(assign=True)'


# ==========================================================================================================================
# separation
# ==========================================================================================================================
def test_graphs_per_shape_per_copy_and_switch():
    m = _model(32, seed=10).eval()
    (x4, t4), = _inputs(4, 32, seed=11, n=1)
    (x8, t8), = _inputs(8, 32, seed=12, n=1)
    eng = m.engine
    eng.enable_cuda_graph(True)
    with torch.no_grad():
        y4, y8 = m(x4, t4), m(x8, t8)
    assert sorted(eng._graphs) == [(4, 3, 32, 32), (8, 3, 32, 32)]
    # a deep copy (the Trainer's EMA model) keeps the switch and captures its own graphs
    cp = copy.deepcopy(m)
    assert cp.engine is not eng and cp.engine.use_cuda_graph and len(cp.engine._graphs) == 0
    with torch.no_grad():
        c4 = cp(x4, t4)
    assert list(cp.engine._graphs) == [(4, 3, 32, 32)] and len(eng._graphs) == 2
    assert cp.engine._graphs[(4, 3, 32, 32)][0] is not eng._graphs[(4, 3, 32, 32)][0]
    assert torch.equal(c4, y4)
    # the autograd path is never graphed, and its x.grad is the one of the switch off: within the run-to-run spread of two
    # backwards with the switch off (zero when the backward is deterministic)
    grads = []
    for flag in (True, False, False):
        eng.enable_cuda_graph(flag)
        xr = x4.clone().requires_grad_()
        y = m(xr, t4)
        assert y.grad_fn is not None and len(eng._graphs) == 0
        (y * y).sum().backward()
        grads.append(xr.grad)
        m.zero_grad(set_to_none=True)
    spread = rel(grads[2], grads[1])
    _METRICS['model graph separation::x.grad run-to-run spread'] = spread
    _METRICS['model graph separation::x.grad, switch on vs off'] = rel(grads[0], grads[1])
    assert rel(grads[0], grads[1]) <= 4 * spread
    # switched off: eager again, no graph
    with torch.no_grad():
        e8 = m(x8, t8)
    assert len(eng._graphs) == 0 and torch.equal(e8, y8)


# ==========================================================================================================================
# end to end
# ==========================================================================================================================
def _fp64(sd):
    sd64 = {k: v.detach().to(DEV, F64) for k, v in sd.items()}
    return lambda a, s: MO.model_forward(sd64, a.to(DEV, F64), s, ch=NET['ch'], num_resolutions=4, num_res_blocks=2)


def test_graphed_config2_sample_against_float64():
    """BASELINE config 2 (deblurring, Special_6_routine, T = 50, x0_step_down) with the CIFAR `Model`, 3 reverse steps"""
    ck = Checks('model graph sample')
    B = 8
    m = _model(32, seed=13)
    gd = _deblur(m)
    x = torch.rand(B, 3, 32, 32, generator=gen(14), device=DEV) * 2 - 1
    m.engine.enable_cuda_graph(True)
    with torch.no_grad():
        xt, dr, img = gd.sample(batch_size=B, img=x, t=3)
    m.engine.enable_cuda_graph(False)
    with torch.no_grad():
        eager = gd.sample(batch_size=B, img=x, t=3)
    for name, a, b in zip(('x_t', 'direct', 'sample'), (xt, dr, img), eager):
        ck.require('graphed %s equals eager' % name, torch.equal(a, b))
    o = DO.DeblurOracle(_fp64(m.state_dict()), sampling_routine='x0_step_down', **CONFIG2)
    o.kernels2d = [k.double().cuda() for k in o.kernels2d]
    with torch.no_grad():
        r = o.sample(B, x.double(), t=3)
        x1 = o.degrade(x.double(), 1)
    ck('x_t', rel(xt, r[0]), 3e-7, rel(xt, x1))                           # measured 1.0e-7
    ck('direct', rel(dr, r[1]), 3.1e-3, rel(dr.roll(1, 0), r[1]))         # measured 1.06e-3 (TF32 convolutions)
    ck('sample', rel(img, r[2]), 3.6e-4, rel(xt, r[2]))                  # measured 1.2e-4
    ck.done()


def test_snowification_sample_with_two_graphed_models(tmp_path):
    """the decolorization GaussianDiffusion of the snowification package with a `Model` for denoise_fn and another for
    one_shot_denoise_fn (with_time_emb=False): each network captures its own graph, and the graphed sample equals the eager one"""
    from cold_diffusion_models_b200.snowification_diffusion import GaussianDiffusion as SNGD
    B = 4
    den, one = _model(32, seed=15), _model(32, seed=16, with_time_emb=False)
    with contextlib.redirect_stdout(io.StringIO()):
        gd = SNGD(den, image_size=32, device_of_kernel='cuda', one_shot_denoise_fn=one, channels=3, timesteps=20, loss_type='l1',
                  forward_process_type='Decolorization', decolor_routine='Linear', decolor_total_remove=True, train_routine='Final',
                  sampling_routine='x0_step_down', results_folder=str(tmp_path)).to(DEV)
    x = torch.rand(B, 3, 32, 32, generator=gen(17), device=DEV) * 2 - 1
    out = {}
    for flag in (False, True):
        den.engine.enable_cuda_graph(flag)
        one.engine.enable_cuda_graph(flag)
        with torch.no_grad():
            out[flag] = (gd.sample(batch_size=B, img=x, t=4), one(x))
        if flag:
            assert list(den.engine._graphs) == [(B, 3, 32, 32)] and list(one.engine._graphs) == [(B, 3, 32, 32)]
            assert den.engine._graphs[(B, 3, 32, 32)][0] is not one.engine._graphs[(B, 3, 32, 32)][0]
        den.engine.enable_cuda_graph(False)
        one.engine.enable_cuda_graph(False)
    (se, oe), (sg, og) = out[False], out[True]
    for k in ('xt', 'direct_recons', 'recon'):
        assert torch.equal(sg[k], se[k]), k
    assert torch.equal(og, oe)
