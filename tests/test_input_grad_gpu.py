"""Gradients with respect to the network input, and frozen parameters, for `Unet` and `Model`: x.grad against float64 torch
autograd of oracle/unet_oracle.py and oracle/model2_oracle.py, the backward of a fully or partly frozen network against the
all-trainable backward, three optimizer steps with part of the network frozen, composition with a torch module in front,
and the refusal of create_graph=True.

Every dx comparison also evaluates its metric against a reference that leaves one term of dx out (a negative control) and
asserts that it lands at least 10x past the bound.  Set COLDDIFF_TEST_METRICS=<file> to write every value and control as JSON."""
import contextlib
import ctypes as C
import io
import math

import pytest
import torch
import torch.nn.functional as F

import model2_oracle as MO
import unet_oracle as UO
from test_config3_step_gpu import Checks, _metrics_file, _free_between_tests, _METRICS, rel, gen  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
FP32_BOUND, TF32_BOUND = 2e-4, 1.5e-3          # the parameter-gradient bounds of tests/test_grads_gpu.py
# the Model's TF32 dx: measured 1.60e-3 (32²) and 1.65e-3 (64²) on an H100 80GB HBM3 (700 W), where its fp32 path measures
# 4.3e-6; the bound is the one tests/test_model_large_gpu.py sets for the Model's TF32 forward
MODEL_TF32_BOUND = 2.5e-3
MNET = dict(ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2, attn_resolutions=(16,))


@pytest.fixture(autouse=True)
def _fp64_time_embedding(monkeypatch):
    """oracle/model2_oracle.py builds the sinusoidal table in float32 on the CPU; the references here run in float64 on the GPU"""
    def temb(t, dim):
        half = dim // 2
        f = torch.exp(torch.arange(half, dtype=F64, device=DEV) * -(math.log(10000) / (half - 1)))
        e = t.to(DEV, F64)[:, None] * f[None, :]
        return torch.cat([torch.sin(e), torch.cos(e)], dim=1)
    monkeypatch.setattr(MO, 'timestep_embedding', temb)


def _unet(dim, mults, channels=3, residual=False, with_time_emb=True, seed=3):
    import cold_diffusion_models_b200 as cdm
    sd = UO.make_unet_state_dict(dim, mults, channels, seed=seed, with_time_emb=with_time_emb)
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim, dim_mults=mults, channels=channels, with_time_emb=with_time_emb, residual=residual)
    u.load_state_dict(sd)
    return u.to(DEV)


def _model(S, seed=3):
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(seed)
    return cdm.Model(resolution=S, in_channels=3, out_ch=3, dropout=0.0, **MNET).to(DEV)


def _inputs(B, Cc, S, seed):
    x = torch.rand(B, Cc, S, S, generator=gen(seed), device=DEV) * 2 - 1
    target = torch.rand(B, Cc, S, S, generator=gen(seed + 1), device=DEV) * 2 - 1
    t = torch.randint(0, 50, (B,), generator=gen(seed + 2), device=DEV)
    return x, target, t


def _l2(y, target):
    # L2, not the training L1: the sign() of L1 flips on 1e-4-level forward differences (tests/test_grads_gpu.py)
    return ((target - y) ** 2).sum() / y.numel()


def _engine_dx(net, x, target, t):
    xr = x.clone().requires_grad_(True)
    y = net(xr, t)
    _l2(y, target).backward()
    torch.cuda.synchronize()
    return xr.grad.detach().clone()


def _unet_ref(u, x, target, t, residual):
    """float64 dx and its terms: (dx, depthwise term, res_conv term, dout term) of the first block / the residual output"""
    sd = {k: v.detach().to(DEV, F64) for k, v in u.state_dict().items()}
    x64 = x.to(F64).requires_grad_(True)
    keep = {}
    orig = UO.convnext_block

    def block(sd_, p, xin, temb, ops):
        out = orig(sd_, p, xin, temb, ops)
        if p == 'downs.0.0.':
            out.retain_grad()
            keep['out'] = out
        return out
    UO.convnext_block = block
    try:
        y = UO.unet_forward(sd, x64, t.to(F64), residual=residual)
        yr = y.detach().requires_grad_(True)
        _l2(yr, target.to(F64)).backward()
        y.backward(yr.grad)
    finally:
        UO.convnext_block = orig
    dout = yr.grad if residual else torch.zeros_like(x64)
    res = F.conv_transpose2d(keep['out'].grad, sd['downs.0.0.res_conv.weight'])
    dw = x64.grad - res - dout
    return x64.grad.detach(), dw, res, dout


def _check_dx(ck, name, dx, ref, terms, bound, base=None):
    """dx within `bound` of ref; every reference with one term left out at least 10x past it.  base: a term known exactly
    (dout for residual=True, about 100x the rest of dx) that is taken off both sides for the controls of the other terms"""
    ck(name, rel(dx, ref), bound)
    if base is not None:             # recorded, not bounded: the network's own term, 1/100 of dx (TF32: 1.6e-3)
        _METRICS['%s::%s less dout' % (ck.test, name)] = rel(dx - base, ref - base)
    for tname, term in terms.items():
        ctrl = rel(dx, ref - term) if base is None or term is base else rel(dx - base, ref - base - term)
        ck('%s without %s' % (name, tname), 0.0, bound, ctrl)
        ck.require('%s: leaving out %s gives %.3e, not 10x past the bound %.1e' % (name, tname, ctrl, bound), ctrl > 10 * bound)


# ==========================================================================================================================
# dx against float64
# ==========================================================================================================================
UNET_CASES = [
    # (id, dim, mults, channels, residual, with_time_emb, S, B, fp32 path too)
    ('small-3ch', 32, (1, 2), 3, False, True, 32, 2, True),
    ('small-1ch', 32, (1, 2), 1, False, True, 32, 2, True),
    ('small-residual', 32, (1, 2), 3, True, True, 32, 2, True),
    ('small-no-time', 32, (1, 2), 3, False, False, 32, 2, True),
    ('config3-128', 64, (1, 2, 4, 8), 3, False, True, 128, 4, False),
    ('config3-256', 64, (1, 2, 4, 8), 3, False, True, 256, 2, False),
]


@pytest.mark.parametrize('case', UNET_CASES, ids=[c[0] for c in UNET_CASES])
def test_unet_input_gradient(case):
    from cold_diffusion_models_b200.ops import CONV_TC, CONV_SIMT
    name, dim, mults, Cc, residual, with_t, S, B, fp32 = case
    ck = Checks('unet dx ' + name)
    u = _unet(dim, mults, Cc, residual, with_t)
    x, target, t = _inputs(B, Cc, S, seed=S + Cc)
    ref, dw, res, dout = _unet_ref(u, x, target, t, residual)
    terms = {'the depthwise path': dw, 'the res_conv path': res}
    if residual:
        terms['dout'] = dout
    impls = [('tf32', CONV_TC, TF32_BOUND)] + ([('fp32', CONV_SIMT, FP32_BOUND)] if fp32 else [])
    for tag, impl, bound in impls:
        u.engine.conv_impl = impl
        _check_dx(ck, tag, _engine_dx(u, x, target, t), ref, terms, bound, base=dout if residual else None)
    ck.done()


@pytest.mark.parametrize('S', [32, 64])
def test_model_input_gradient(S):
    from cold_diffusion_models_b200.ops import CONV_TC, CONV_SIMT
    ck = Checks('model dx %d' % S)
    m = _model(S)
    B = 2
    x, target, t = _inputs(B, 3, S, seed=S)
    sd = {k: v.detach().to(DEV, F64) for k, v in m.state_dict().items()}
    x64 = x.to(F64).requires_grad_(True)
    y = MO.model_forward(sd, x64, t, ch=MNET['ch'], num_resolutions=4, num_res_blocks=2)
    _l2(y, target.to(F64)).backward()
    ref = x64.grad.detach()
    impls = [('tf32', CONV_TC, MODEL_TF32_BOUND)] + ([('fp32', CONV_SIMT, FP32_BOUND)] if S == 32 else [])
    for tag, impl, bound in impls:
        m.conv_impl = impl
        _check_dx(ck, tag, _engine_dx(m, x, target, t), ref, {'conv_in': ref}, bound)
    ck.done()


# ==========================================================================================================================
# frozen parameters
# ==========================================================================================================================
_WGRAD_CALLS = ('cd_dwconv7_wgrad', 'cd_small_gemm', 'cd_unpack_wgrad', 'cd_unpack_wgrad_batched')


@contextlib.contextmanager
def _record_calls():
    """every C-ABI call of the package as (name, args)"""
    import cold_diffusion_models_b200 as pkg
    from cold_diffusion_models_b200 import _lib
    import sys
    calls, orig = [], _lib.call

    def rec(name, *args):
        calls.append((name, args))
        return orig(name, *args)
    mods = [m for k, m in list(sys.modules.items()) if k.startswith(pkg.__name__) and getattr(m, 'call', None) is orig]
    for m in mods:
        m.call = rec
    try:
        yield calls
    finally:
        # a package module first imported inside the context (model2_train, on the first training forward of a Model) took
        # `call` from the patched _lib: give it the real one back too, or every later recording misses its calls
        for m in list(sys.modules.values()):
            if getattr(m, 'call', None) is rec:
                m.call = orig


def _parameter_gradient_calls(calls):
    """calls that form a parameter gradient.  cd_conv_wgrad with per-image weights (w_per_batch) is not one: the attention
    backward uses it for activation products (d(weff) of LinearAttention, dk and dv of AttnBlock) that dx needs"""
    out = []
    for name, args in calls:
        if name == 'cd_conv_wgrad' and not args[0]._obj.s[0].w_per_batch:
            out.append(name)
        elif name in _WGRAD_CALLS or name.startswith('cd_colsum'):
            out.append(name)
    return out


def _nets():
    return [('unet', lambda: _unet(32, (1, 2)), 'downs.', 32), ('model', lambda: _model(32), 'down.', 32)]


def _backward(net, x, target, t, need_x):
    for p in net.parameters():
        p.grad = None
    eng = net.engine
    if getattr(eng, 'flat_grad', None) is not None:
        eng.flat_grad.zero_()
    xr = x.clone().requires_grad_(need_x)
    _l2(net(xr, t), target).backward()
    torch.cuda.synchronize()
    grads = {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in net.named_parameters()}
    return (xr.grad.detach().clone() if need_x else None), grads


def _cat(grads, names):
    return torch.cat([grads[n].reshape(-1) for n in names])


@pytest.mark.parametrize('which', ['unet', 'model'])
def test_frozen_network(which):
    _, mk, prefix, S = [n for n in _nets() if n[0] == which][0]
    ck = Checks('frozen ' + which)
    net = mk()
    x, target, t = _inputs(2, 3, S, seed=7)
    dx1, g1 = _backward(net, x, target, t, True)
    dx2, g2 = _backward(net, x, target, t, True)
    names = [n for n, _ in net.named_parameters()]
    spread_dx = rel(dx2, dx1)
    _METRICS['frozen %s::dx run-to-run spread' % which] = spread_dx
    # ---- everything frozen: the input-only backward
    net.requires_grad_(False)
    with _record_calls() as calls:
        dx0, g0 = _backward(net, x, target, t, True)
    ck('input-only dx vs all-trainable (bound 4x the spread)', rel(dx0, dx1), 4 * spread_dx + 1e-30)
    ck.require('frozen parameters got a .grad', all(g is None for g in g0.values()))
    wg = _parameter_gradient_calls(calls)
    ck.require('input-only backward ran parameter-gradient launches: %s' % sorted(set(wg)), not wg)
    ck.require('dx did not reach NCHW through cd_nhwc_to_nchw_add', any(n == 'cd_nhwc_to_nchw_add' for n, _ in calls))
    # ---- part frozen: every downs.* / down.* parameter
    for n, p in net.named_parameters():
        p.requires_grad_(not n.startswith(prefix))
    trainable = [n for n in names if not n.startswith(prefix)]
    spread_g = rel(_cat(g2, trainable), _cat(g1, trainable))
    _METRICS['frozen %s::gradient run-to-run spread' % which] = spread_g
    _, gh = _backward(net, x, target, t, False)
    ck.require('a frozen parameter got a .grad', all(gh[n] is None for n in names if n.startswith(prefix)))
    ck('half-frozen gradients vs all-trainable (bound 4x the spread)', rel(_cat(gh, trainable), _cat(g1, trainable)),
       4 * spread_g + 1e-30)
    ck.done()


def test_trainer_steps_with_frozen_down_path(tmp_path):
    """three optimizer steps with every downs.* parameter frozen: frozen weights and their EMA stay bitwise put, the rest
    follow torch.optim.Adam and the EMA lerp applied to the same gradients"""
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.ops import CONV_SIMT
    sd = UO.make_unet_state_dict(32, (1, 2), 3, seed=3)
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
        u.load_state_dict(sd)
        gd = cdm.GaussianDiffusion(u, image_size=32, device_of_kernel='cuda', channels=3, timesteps=4, kernel_std=0.15,
                                   kernel_size=7, blur_routine='Exponential_reflect', sampling_routine='x0_step_down').cuda()
    for n, p in gd.denoise_fn.named_parameters():
        p.requires_grad_(not n.startswith('downs.'))
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=32, train_batch_size=2, train_lr=1e-3, gradient_accumulate_every=2,
                         results_folder=str(tmp_path), dataset='synthetic', step_start_ema=0, update_ema_every=1, ema_decay=0.5)
    gd.denoise_fn.engine.conv_impl = CONV_SIMT
    net = gd.denoise_fn
    named = dict(net.named_parameters())
    trainable = [n for n in named if not n.startswith('downs.')]
    frozen = [n for n in named if n.startswith('downs.')]
    before = {n: named[n].detach().clone() for n in named}
    ref = {n: named[n].detach().clone() for n in trainable}
    ref_ema = {n: named[n].detach().clone() for n in trainable}
    opt = torch.optim.Adam([ref[n] for n in trainable], lr=1e-3)
    g = torch.Generator().manual_seed(5)
    for step in range(3):
        for _ in range(2):
            x = (torch.rand(2, 3, 32, 32, generator=g) * 2 - 1).cuda()
            t = torch.randint(0, 4, (2,), generator=g).cuda()
            (gd.p_losses(x, t) / 2).backward()
        torch.cuda.synchronize()
        for n in trainable:
            ref[n].grad = named[n].grad.detach().clone()
        assert all(named[n].grad is None for n in frozen)
        # beta = 0.5 keeps the EMA of an unchanged weight bit for bit: w * 0.5 + 0.5 * w is exact
        tr.opt.step(ema_mode=2, ema_beta=0.5)
        tr.opt.zero_grad()
        opt.step()
        with torch.no_grad():
            for n in trainable:
                ref_ema[n].mul_(0.5).add_(0.5 * ref[n])
    torch.cuda.synchronize()
    ema = dict(tr.ema_model.denoise_fn.named_parameters())
    for n in frozen:
        assert torch.equal(named[n].detach(), before[n]), n
        assert torch.equal(ema[n].detach(), before[n]), n
    for n in trainable:
        assert rel(named[n].detach(), ref[n].detach()) < 2e-4, n
        assert rel(ema[n].detach(), ref_ema[n]) < 2e-4, n
    assert max(rel(named[n].detach(), before[n]) for n in trainable) > 1e-3          # the trainable weights really moved
    # the trainable set is fixed at the first step
    named['downs.0.0.ds_conv.weight'].requires_grad_(True)
    with pytest.raises(ValueError, match='downs.0.0.ds_conv.weight'):
        tr.opt.step()


def test_torch_module_in_front_of_the_unet():
    """a trainable nn.Conv2d before the Unet: its weight gradient flows through x.grad of the engine.  The Unet runs its fp32
    path, so the check isolates the composition (the TF32 dx is checked above; through it the pre-conv weight gradient
    measured 1.48e-3)"""
    from cold_diffusion_models_b200.ops import CONV_SIMT
    u = _unet(32, (1, 2))
    u.engine.conv_impl = CONV_SIMT
    pre = torch.nn.Conv2d(3, 3, 3, padding=1).to(DEV)
    x, target, t = _inputs(2, 3, 32, seed=21)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        _l2(u(pre(x), t), target).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    torch.cuda.synchronize()
    sd = {k: v.detach().to(DEV, F64) for k, v in u.state_dict().items()}
    w64 = pre.weight.detach().to(F64).requires_grad_(True)
    b64 = pre.bias.detach().to(F64).requires_grad_(True)
    y = UO.unet_forward(sd, F.conv2d(x.to(F64), w64, b64, padding=1), t.to(F64))
    _l2(y, target.to(F64)).backward()
    ck = Checks('composition')
    ck('pre-conv weight gradient', rel(pre.weight.grad, w64.grad), FP32_BOUND, rel(pre.weight.grad, -w64.grad))
    ck('pre-conv bias gradient', rel(pre.bias.grad, b64.grad), FP32_BOUND, rel(pre.bias.grad, -b64.grad))
    ck.done()


@pytest.mark.parametrize('which', ['unet', 'model'])
def test_create_graph_raises(which):
    _, mk, _, S = [n for n in _nets() if n[0] == which][0]
    net = mk()
    x, target, t = _inputs(1, 3, S, seed=31)
    xr = x.clone().requires_grad_(True)
    loss = _l2(net(xr, t), target)
    with pytest.raises(RuntimeError, match='first order'):
        torch.autograd.grad(loss, [xr], create_graph=True)
