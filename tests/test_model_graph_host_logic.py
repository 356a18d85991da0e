"""CPU check of the HOST LOGIC of the CUDA-graph replay of the inference forward (`engine.enable_cuda_graph`, graphs.py) for the
ConvNeXt `Unet` and the DDPM `Model`: which graphs are captured, kept and dropped, and that a graph keeps reading the right
weights.

The capture (graphs.capture) is replaced by a recording of the forward's C-ABI calls with their arguments, replayed on
tests/abi_emulator.py with the same arguments: like a captured CUDA graph, the replay reads and writes the addresses the
capture saw.  A packed operand rebuilt as a new tensor, or a parameter moved to new storage, would leave the replay reading
stale values, and the replay would differ from the eager forward.  The CUDA kernels and the real capture are exercised by
tests/test_model_graph_gpu.py and tests/test_unet_gpu.py."""
import contextlib
import copy
import io

import pytest
import torch

import abi_emulator


class _RecordedGraph:
    def __init__(self):
        self.calls, self.replays = [], 0

    def replay(self):
        self.replays += 1
        for name, args in self.calls:
            abi_emulator.call(name, *args)


@pytest.fixture()
def emulated(monkeypatch):
    from cold_diffusion_models_b200 import engine, graphs, model2, ops
    captures = []

    def capture(fn, device):
        fn()                                   # the warm-up
        g = _RecordedGraph()
        rec = lambda name, *args: g.calls.append((name, args))      # noqa: E731
        saved = engine.call, model2.call, ops.call
        engine.call = model2.call = ops.call = rec
        try:
            out = fn()
        finally:
            engine.call, model2.call, ops.call = saved
        captures.append(g)
        return g, out

    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)
    monkeypatch.setattr(graphs, 'capture', capture)
    with abi_emulator.patched():
        yield captures


def _net(kind, seed=0, **kw):
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(seed)
    if kind == 'Unet':
        with contextlib.redirect_stdout(io.StringIO()):
            return cdm.Unet(dim=32, dim_mults=(1, 2), channels=3, **kw)
    return cdm.Model(resolution=16, in_channels=3, out_ch=3, ch=32, ch_mult=(1, 2), num_res_blocks=2, attn_resolutions=(8,),
                     dropout=0.1, **kw)


def _packs(m):
    """the packed operands the graphs read, and the suffix of the packed bias sums (conv2 + shortcut)"""
    return (m.engine._packed, '.b2r') if hasattr(m, 'ups') else (m._packed, '.b2s')


def _last_convs(m):
    """(a conv whose bias the forward reads from the parameter, a 3x3 conv whose weight it reads packed)"""
    return (m.final_conv[1], m.final_conv[0].net[3]) if hasattr(m, 'ups') else (m.conv_out, m.conv_out)


def _inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, 16, 16, generator=g) * 2 - 1, torch.randint(0, 6, (B,), generator=g)


def _eager(m, x, t=None):
    ref = copy.deepcopy(m)
    ref.engine.enable_cuda_graph(False)
    with torch.no_grad():
        return ref(x, t) if t is not None else ref(x)


def _perturb(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g))


def test_replay_equals_eager_and_follows_in_place_weight_updates(emulated, kind='Model'):
    m = _net(kind)
    m.eval()
    x, t = _inputs(3, 1)
    m.engine.enable_cuda_graph(True)
    with torch.no_grad():
        y0 = m(x, t)
        x2, t2 = _inputs(3, 2)
        y1 = m(x2, t2)
    assert len(emulated) == 1 and emulated[0].replays == 2
    assert torch.equal(y0, _eager(m, x, t)) and torch.equal(y1, _eager(m, x2, t2))
    P, bias_sum = _packs(m)
    held = {k: P[k].data_ptr() for k in P if k.startswith('cond.') or k.endswith(bias_sum)}
    assert 'cond.w' in held and 'cond.b' in held and any(k.endswith(bias_sum) for k in held)
    _perturb(m, 3)
    with torch.no_grad():
        y2 = m(x, t)
    assert len(emulated) == 1, 'an in-place weight change must not need a new capture'
    assert {k: P[k].data_ptr() for k in held} == held, 'packed operands must be refilled in place'
    assert torch.equal(y2, _eager(m, x, t)) and not torch.equal(y2, y0)


def test_without_time_embedding(emulated, kind='Model'):
    m = _net(kind, with_time_emb=False)
    x, _ = _inputs(2, 4)
    m.engine.enable_cuda_graph(True)
    with torch.no_grad():
        y = m(x)
    assert len(emulated) == 1 and torch.equal(y, _eager(m, x))


def test_one_graph_per_shape_and_switch(emulated, kind='Model'):
    m = _net(kind)
    eng = m.engine
    eng.enable_cuda_graph(True)
    with torch.no_grad():
        for B in (2, 3, 2):
            m(*_inputs(B, B))
    assert sorted(eng._graphs) == [(2, 3, 16, 16), (3, 3, 16, 16)] and len(emulated) == 2
    eng.enable_cuda_graph(False)
    assert not eng.use_cuda_graph and eng._graphs == {}
    with torch.no_grad():
        m(*_inputs(2, 5))
    assert len(emulated) == 2 and eng._graphs == {}


def test_autograd_path_is_never_graphed(emulated, kind='Model'):
    m = _net(kind)
    m.engine.enable_cuda_graph(True)
    x, t = _inputs(2, 6)
    y = m(x.requires_grad_(), t)
    assert y.grad_fn is not None and len(emulated) == 0


def test_deep_copy_keeps_the_switch_and_gets_its_own_graphs(emulated, kind='Model'):
    m = _net(kind)
    m.engine.enable_cuda_graph(True)
    x, t = _inputs(2, 7)
    with torch.no_grad():
        y = m(x, t)
    cp = copy.deepcopy(m)
    assert cp.engine is not m.engine and cp.engine.use_cuda_graph and cp.engine._graphs == {}
    with torch.no_grad():
        yc = cp(x, t)
    assert len(emulated) == 2 and torch.equal(yc, y) and len(m.engine._graphs) == 1


def test_flatten_params_apply_and_load_state_dict(emulated, kind='Model'):
    m = _net(kind)
    eng = m.engine
    eng.enable_cuda_graph(True)
    x, t = _inputs(2, 8)
    key = tuple(x.shape)

    def run():
        with torch.no_grad():
            return m(x, t)
    run()
    # flatten_params (FusedAdamEMA) moves every parameter into one buffer
    eng.flatten_params()
    assert eng._graphs == {}
    y = run()
    assert len(emulated) == 2 and torch.equal(y, _eager(m, x, t))
    # load_state_dict copies in place, directly or through an enclosing module: the graph stays and replays the new weights
    other = _net(kind, seed=1).state_dict()
    m.load_state_dict(other)
    y = run()
    assert len(emulated) == 2 and torch.equal(y, _eager(m, x, t))
    holder = torch.nn.Module()
    holder.net = m
    holder.load_state_dict({'net.' + k: v for k, v in _net(kind, seed=2).state_dict().items()})
    y = run()
    assert len(emulated) == 2 and torch.equal(y, _eager(m, x, t))
    # assign=True rebinds the parameters, and any rebinding is seen: captured again
    m.load_state_dict({k: v.clone() for k, v in other.items()}, assign=True)
    y = run()
    assert len(emulated) == 3 and eng._graphs[key][0] is emulated[-1] and torch.equal(y, _eager(m, x, t))
    with_bias, with_weight = _last_convs(m)
    with torch.no_grad():
        with_bias.bias.data = with_bias.bias.data + 1
        with_weight.weight.data = with_weight.weight.data * 1.5    # new storage, new version counter: packed again
    y = run()
    assert len(emulated) == 4 and torch.equal(y, _eager(m, x, t))
    # _apply (.to(), .float(), ...) drops the workspaces the graphs write, and keeps the switch
    m.float()
    assert m.engine._graphs == {} and m.engine.use_cuda_graph
    y = run()
    assert len(emulated) == 5 and torch.equal(y, _eager(m, x, t))


def test_trainer_step_is_followed_by_the_graphs_of_model_and_ema(emulated, tmp_path, kind='Model'):
    import cold_diffusion_models_b200 as cdm
    m = _net(kind)
    m.engine.enable_cuda_graph(True)
    kw = dict(image_size=16, channels=3, timesteps=6, kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine', loss_type='l2')
    gd = cdm.GaussianDiffusion(m, device_of_kernel='cpu', sampling_routine='x0_step_down', **kw)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=16, train_batch_size=2, train_lr=1e-3, gradient_accumulate_every=1,
                         results_folder=str(tmp_path), dataset='synthetic', step_start_ema=0, update_ema_every=1, ema_decay=0.9)
    ema = tr.ema_model.denoise_fn
    x, t = _inputs(2, 9)
    with torch.no_grad():
        y0, e0 = m(x, t), ema(x, t)
    m.eval()
    tr.train_step([x])
    with torch.no_grad():
        y1, e1 = m(x, t), ema(x, t)
    assert len(emulated) == 2, 'the optimizer step must not need a new capture'
    assert not torch.equal(y1, y0) and not torch.equal(e1, e0)
    assert torch.equal(y1, _eager(m, x, t)) and torch.equal(e1, _eager(ema, x, t))
    # the periodic sample of the EMA model replays its graph
    with torch.no_grad():
        tr.ema_model.sample(batch_size=2, img=x)
    assert len(emulated) == 2 and emulated[1].replays == 2 + 6


# the Unet runs every case above
def test_unet_replay_equals_eager_and_follows_in_place_weight_updates(emulated):
    test_replay_equals_eager_and_follows_in_place_weight_updates(emulated, 'Unet')


def test_unet_without_time_embedding(emulated):
    test_without_time_embedding(emulated, 'Unet')


def test_unet_one_graph_per_shape_and_switch(emulated):
    test_one_graph_per_shape_and_switch(emulated, 'Unet')


def test_unet_autograd_path_is_never_graphed(emulated):
    test_autograd_path_is_never_graphed(emulated, 'Unet')


def test_unet_deep_copy_keeps_the_switch_and_gets_its_own_graphs(emulated):
    test_deep_copy_keeps_the_switch_and_gets_its_own_graphs(emulated, 'Unet')


def test_unet_flatten_params_apply_and_load_state_dict(emulated):
    test_flatten_params_apply_and_load_state_dict(emulated, 'Unet')


def test_unet_trainer_step_is_followed_by_the_graphs_of_model_and_ema(emulated, tmp_path):
    test_trainer_step_is_followed_by_the_graphs_of_model_and_ema(emulated, tmp_path, 'Unet')
