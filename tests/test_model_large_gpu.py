"""The DDPM `Model` (ch = 128, ch_mult = (1, 2, 2, 2), two ResNet blocks per level, attention at 16²) at 64² and 256², and the
split-plane GroupNorm its 256² level runs (planes of more than 128 x 128 pixels), against float64 references computed on the
GPU: plain torch for the GroupNorm entry points, oracle/model2_oracle.py for the network, oracle/deblur_oracle.py around it.

As in tests/test_unet_512_train_gpu.py, every comparison also evaluates its metric on a deliberately wrong reference (a
negative control) and asserts that it exceeds the bound.  Every bound is at most 3x the value measured on an H100 80GB HBM3
(700 W), which is in the comment beside it.  Set COLDDIFF_TEST_METRICS=<file> to write all values and controls as JSON."""
import contextlib
import ctypes as C
import io
import math

import pytest
import torch
import torch.nn.functional as F

import deblur_oracle as DO
import model2_oracle as MO
from test_config3_step_gpu import (Checks, _metrics_file, _free_between_tests, _METRICS, rel, call, ptr, stream, gen,  # noqa: F401
                                   blur_per_image, grad_errors, stats)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
NET = dict(ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2, attn_resolutions=(16,))


@pytest.fixture(autouse=True)
def _fp64_time_embedding(monkeypatch):
    """oracle/model2_oracle.py builds the sinusoidal table in float32 on the CPU; the references here run in float64 on the GPU"""
    def temb(t, dim):
        half = dim // 2
        f = torch.exp(torch.arange(half, dtype=F64, device=DEV) * -(math.log(10000) / (half - 1)))
        e = t.to(DEV, F64)[:, None] * f[None, :]
        return torch.cat([torch.sin(e), torch.cos(e)], dim=1)
    monkeypatch.setattr(MO, 'timestep_embedding', temb)


def _model(S, seed=3, dropout=0.0):
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(seed)
    return cdm.Model(resolution=S, in_channels=3, out_ch=3, dropout=dropout, **NET).to(DEV)


def _fp64(sd):
    sd64 = {k: v.detach().to(DEV, F64) for k, v in sd.items()}
    return lambda a, s: MO.model_forward(sd64, a.to(F64), s, ch=NET['ch'], num_resolutions=4, num_res_blocks=2)


def _ref_grads(sd, x, target, t, norm):
    """fp64 autograd of sum |target - Model(x, t)|^2 / norm, one image at a time -> (gradients by name, outputs)"""
    leaves = {k: v.detach().to(DEV, F64).requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    names = [k for k in leaves if leaves[k].requires_grad]
    acc = {k: torch.zeros_like(leaves[k]) for k in names}
    ys = []
    for i in range(x.shape[0]):
        y = MO.model_forward(leaves, x[i:i + 1].to(F64), t[i:i + 1], ch=NET['ch'], num_resolutions=4, num_res_blocks=2)
        d = target[i:i + 1].to(F64) - y
        for k, g in zip(names, torch.autograd.grad((d * d).sum() / norm, [leaves[k] for k in names])):
            acc[k] += g
        ys.append(y.detach())
        del y, d
    return acc, torch.cat(ys)


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters()}


def _grad_check(ck, name, eg, ref, ctrl, bmed, bworst):
    # the key bias of an AttnBlock adds q . b_k to a whole row of scores, which the softmax ignores: its gradient is zero in
    # exact arithmetic and round-off on both sides
    ref = {k: v for k, v in ref.items() if not k.endswith('.k.bias')}
    errs = grad_errors(eg, ref)
    med, p90, worst = stats(errs)
    cmed, _, cworst = stats(grad_errors(eg, {k: ctrl[k] for k in ref}))
    _METRICS['%s::%s p90' % (ck.test, name)] = p90
    _METRICS['%s::%s worst parameters' % (ck.test, name)] = [(e, n) for e, n in errs[-5:]]
    ck('%s median' % name, med, bmed, cmed)
    ck('%s worst' % name, worst, bworst, cworst)


# ==========================================================================================================================
# the GroupNorm entry points on 256² planes
# ==========================================================================================================================
def _gn64(x, cond, gamma, beta, swish, B, HW, Cc, groups=32):
    h = (x.to(F64).view(B, HW, Cc) + cond.to(F64)[:, None, :]).permute(0, 2, 1)
    z = F.group_norm(h, groups, gamma.to(F64), beta.to(F64), eps=1e-6).permute(0, 2, 1)
    return z * torch.sigmoid(z) if swish else z


def _fp32_one_pass(x, cond, gamma, beta, B, HW, Cc, groups=32):
    """the one-pass fp32 statistics E[v^2] - mean^2 (the negative control of the large-mean case)"""
    v = x.view(B, HW, groups, Cc // groups) + cond.view(B, 1, groups, Cc // groups)
    mean = v.mean(dim=(1, 3), keepdim=True)
    var = ((v * v).mean(dim=(1, 3), keepdim=True) - mean * mean).clamp_min(0)
    z = ((v - mean) * torch.rsqrt(var + 1e-6)).view(B, HW, Cc) * gamma + beta
    return z * torch.sigmoid(z)


@pytest.mark.parametrize('Cc,shift', [(128, 0.0), (256, 0.0), (128, 100.0)])
def test_groupnorm_split_entry_points_at_256(Cc, shift):
    ck = Checks('groupnorm 256 C=%d shift=%g' % (Cc, shift))
    B, HW, ld = 3, 256 * 256, Cc + 8
    g = gen(7)
    x = torch.randn(B * HW, ld, generator=g, device=DEV) * 1.5 + shift
    cond = 0.5 * torch.randn(B, Cc, generator=g, device=DEV)
    gamma = 1 + 0.2 * torch.randn(Cc, generator=g, device=DEV)
    beta = 0.1 * torch.randn(Cc, generator=g, device=DEV)
    dy = torch.randn(B * HW, ld, generator=g, device=DEV)
    xs = x[:, :Cc].contiguous()
    y = torch.full((B * HW, ld), 7.0, device=DEV)
    call('cd_groupnorm_fwd', ptr(x), ld, B, C.c_int64(HW), Cc, 32, ptr(cond), Cc, ptr(gamma), ptr(beta), C.c_float(1e-6), 1,
         ptr(y), ld, stream())
    # backward: dgamma / dbeta accumulate onto 0.5 / -0.25
    dx = torch.full((B * HW, ld), 7.0, device=DEV)
    dg, db, dc = torch.full((Cc,), 0.5, device=DEV), torch.full((Cc,), -0.25, device=DEV), torch.full((B, Cc), 3.0, device=DEV)
    call('cd_groupnorm_bwd', ptr(x), ld, B, C.c_int64(HW), Cc, 32, ptr(cond), Cc, ptr(gamma), ptr(beta), C.c_float(1e-6), 1,
         ptr(dy), ld, ptr(dx), ld, ptr(dg), ptr(db), ptr(dc), Cc, stream())
    torch.cuda.synchronize()
    ck.require('row padding untouched', bool((y[:, Cc:] == 7.0).all()) and bool((dx[:, Cc:] == 7.0).all()))
    x64, c64, g64, b64 = xs.to(F64).requires_grad_(), cond.to(F64).requires_grad_(), gamma.to(F64).requires_grad_(), beta.to(F64).requires_grad_()
    ref = _gn64(x64, c64, g64, b64, True, B, HW, Cc)
    ref.backward(dy[:, :Cc].to(F64).view(B, HW, Cc))
    yv = y[:, :Cc].view(B, HW, Cc)
    ctrl = _fp32_one_pass(xs, cond, gamma, beta, B, HW, Cc) if shift else ref.detach().roll(1, 0)
    # measured 9.4e-8 (C = 128), 9.3e-8 (C = 256), 2.7e-6 (shift 100; the one-pass fp32 statistics give 2.3e-4)
    ck('forward', rel(yv, ref.detach()), {0.0: 2.8e-7, 100.0: 8e-6}[shift], rel(ctrl, ref.detach()))
    dxv = dx[:, :Cc].view(B, HW, Cc)
    # measured 9.3e-8 / 9.2e-8 / 1.7e-6
    ck('dx', rel(dxv, x64.grad.view(B, HW, Cc)), {0.0: 2.7e-7, 100.0: 5e-6}[shift], rel(dxv.roll(1, 0), x64.grad.view(B, HW, Cc)))
    # measured 2.4e-7 / 3.1e-7 / 3.1e-6 and 1.8e-7 / 3.1e-7 / 1.5e-6; the controls forget the accumulation
    ck('dgamma', rel(dg - 0.5, g64.grad), {0.0: 9e-7, 100.0: 9e-6}[shift], rel(dg, g64.grad))
    ck('dbeta', rel(db + 0.25, b64.grad), {0.0: 9e-7, 100.0: 4.5e-6}[shift], rel(db, b64.grad))
    # dcond = the pixel sum of dx: zero in exact arithmetic, so both sides are round-off; bound it against the terms' size
    scale = x64.grad.view(B, HW, Cc).abs().sum(1).max().item()
    # measured 3.2e-9 / 5.0e-9 / 3.5e-8; the control leaves dcond unwritten
    ck('dcond (abs / pixel sum of |dx|)', (dc.to(F64) - c64.grad).abs().max().item() / scale, {0.0: 1.5e-8, 100.0: 1e-7}[shift],
       3.0 / scale)
    ck.done()


# ==========================================================================================================================
# the network: forward and parameter gradients at 64² and 256²
# ==========================================================================================================================
@pytest.mark.parametrize('S', [64, 256])
def test_model_forward_and_gradients(S):
    ck = Checks('model %d' % S)
    B = 2
    m = _model(S)
    sd = m.state_dict()
    x = torch.rand(B, 3, S, S, generator=gen(11), device=DEV) * 2 - 1
    target = torch.rand(B, 3, S, S, generator=gen(12), device=DEV) * 2 - 1
    t = torch.tensor([3, 17], device=DEV)
    m.zero_grad(set_to_none=True)
    y = m(x, t)
    (((target - y) ** 2).sum() / x.numel()).backward()
    torch.cuda.synchronize()
    eg = _grads(m)
    g0, y0 = _ref_grads(sd, x[:1], target[:1], t[:1], x.numel())
    g1, y1 = _ref_grads(sd, x[1:], target[1:], t[1:], x.numel())
    ref = {k: g0[k] + g1[k] for k in g0}
    y64 = torch.cat([y0, y1])
    with torch.no_grad():
        # TF32 convolutions: measured 9.1e-4 (64²) and 8.6e-4 (256²), the same on the inference path
        ck('forward', rel(y.detach(), y64), 2.5e-3, rel(y.detach().roll(1, 0), y64))
        yi = m.eval()(x, t)                                          # the inference path (no autograd)
        ck('inference forward', rel(yi, y64), 2.5e-3, rel(yi.roll(1, 0), y64))
    # measured median 2.4e-3 (64²) and 1.0e-3 (256²), worst 4.1e-3 and 3.9e-3; the control leaves the second image out
    _grad_check(ck, 'grad', eg, ref, g0, {64: 7e-3, 256: 3e-3}[S], 1.1e-2)
    ck.done()


# ==========================================================================================================================
# one Trainer step of the deblurring GaussianDiffusion at 256², the gradient at the new weights and a sample of the EMA model
# ==========================================================================================================================
def _blur(T, denoise_fn=None, **kw):
    kw.update(image_size=256, channels=3, timesteps=T, kernel_std=0.1, kernel_size=11, blur_routine='Exponential_reflect')
    o = DO.DeblurOracle(denoise_fn, **kw)
    o.kernels2d = [k.double().cuda() for k in o.kernels2d]
    return o


def test_model_256_train_step_and_sample(tmp_path):
    import cold_diffusion_models_b200 as cdm
    ck = Checks('model256 train')
    T, B, S = 20, 2, 256
    m = _model(S, seed=5)
    gd = cdm.GaussianDiffusion(m, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, kernel_std=0.1, kernel_size=11,
                               blur_routine='Exponential_reflect', loss_type='l2', sampling_routine='x0_step_down').to(DEV)
    x = torch.rand(B, 3, S, S, generator=gen(13), device=DEV) * 2 - 1
    t = torch.tensor([3, T - 1], device=DEV)
    o = _blur(T)
    xt64 = blur_per_image(o, x.double(), t)
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=1e-3, train_num_steps=10 ** 9,
                         gradient_accumulate_every=1, ema_decay=0.995, fp16=False, results_folder=str(tmp_path), dataset='synthetic')
    torch.manual_seed(0)
    loss = tr.train_step([x]).item()
    ck.require('train_step loss finite (%r)' % loss, math.isfinite(loss) and abs(loss) < 1e3)
    moved = max((m.state_dict()[k].double() - sd0[k].double()).abs().max().item() for k in sd0)
    ck.require('train_step moved the weights (%.3e)' % moved, 1e-5 < moved < 1e-2)
    _METRICS['model256 train::weights moved (max abs)'] = moved
    tr.opt.zero_grad()
    gd.p_losses(x, t).backward()
    torch.cuda.synchronize()
    eg = _grads(m)
    tr.opt.zero_grad()
    sd1 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    ref_new, ref_old = {}, {}
    for sd, out in ((sd1, ref_new), (sd0, ref_old)):
        g0, _ = _ref_grads(sd, xt64[:1], x[:1], t[:1], x.numel())
        g1, _ = _ref_grads(sd, xt64[1:], x[1:], t[1:], x.numel())
        out.update({k: g0[k] + g1[k] for k in g0})
        del g0, g1
    # measured median 5.9e-4, worst 1.1e-3; the control is the gradient at the old weights
    _grad_check(ck, 'grad after the step', eg, ref_new, ref_old, 1.7e-3, 3.3e-3)
    del ref_new, ref_old, eg
    # a 3-step x0_step_down sample of the EMA model
    ema = tr.ema_model
    with torch.no_grad():
        xt, dr, img = ema.sample(batch_size=B, img=x, t=3)
    torch.cuda.synchronize()
    os_ = _blur(T, denoise_fn=_fp64(ema.denoise_fn.state_dict()), sampling_routine='x0_step_down')
    with torch.no_grad():
        r = os_.sample(B, x.double(), t=3)
    # measured 1.2e-7, 1.2e-4 and 6.7e-4
    ck('sample x_t', rel(xt, r[0]), 3.7e-7, rel(xt, blur_per_image(o, x.double(), torch.full((B,), 1))))
    ck('sample direct', rel(dr, r[1]), 3.6e-4, rel(dr.roll(1, 0), r[1]))
    ck('sample', rel(img, r[2]), 2e-3, rel(xt, r[2]))
    ck.done()


# ==========================================================================================================================
# batch independence and dropout at 256²
# ==========================================================================================================================
def test_model_256_batch_independence():
    """B = 1 against one row of a B = 3 batch (other grids for every kernel, the same arithmetic per image): the forward output
    and the gradient.  The controls are another row, and the gradient of a different image."""
    ck = Checks('model256 batch independence')
    S, B = 256, 3
    m = _model(S, seed=8)
    x = torch.rand(B, 3, S, S, generator=gen(14), device=DEV) * 2 - 1
    t = torch.tensor([2, 9, 15], device=DEV)
    m.zero_grad(set_to_none=True)
    y = m(x, t)
    (y[1] ** 2).mean().backward()
    whole = _grads(m)
    m.zero_grad(set_to_none=True)
    y1 = m(x[1:2], t[1:2])
    (y1[0] ** 2).mean().backward()
    one = _grads(m)
    m.zero_grad(set_to_none=True)
    y2 = m(x[2:3], t[2:3])
    (y2[0] ** 2).mean().backward()
    other = _grads(m)
    m.zero_grad(set_to_none=True)
    # TF32 round-off of other grids: measured 6.8e-4 (forward), median 2.9e-4 and worst 2.2e-3 (gradient)
    ck('forward row 1', rel(y[1:2].detach(), y1.detach()), 2e-3, rel(y[2:3].detach(), y1.detach()))
    _grad_check(ck, 'grad', one, whole, other, 8.5e-4, 6.4e-3)
    ck.done()


def test_model_256_dropout_mask_matches_between_forward_and_backward():
    """with dropout = 0.1 in training mode, a step of length eps along the negative gradient changes the loss by -eps |g|^2 to
    first order when the same host seed draws the same masks in the forward and the backward; the control is the zero-order
    prediction (no change)"""
    ck = Checks('model256 dropout')
    S = 256
    m = _model(S, seed=9, dropout=0.1)
    m.train()
    x = torch.rand(1, 3, S, S, generator=gen(15), device=DEV) * 2 - 1
    t = torch.tensor([4], device=DEV)
    torch.manual_seed(5)
    loss = (m(x, t) ** 2).mean()
    loss.backward()
    torch.cuda.synchronize()
    grads = _grads(m)
    gnorm2 = sum((v.double() ** 2).sum().item() for v in grads.values())
    eps = 1e-3 / gnorm2 ** 0.5
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.add_(grads[n], alpha=-eps)
    m.engine.mark_weights_dirty()
    torch.manual_seed(5)
    loss2 = (m(x, t) ** 2).mean()
    predicted = -eps * gnorm2
    ck('first-order loss change', abs((loss2.item() - loss.item()) - predicted) / abs(predicted), 0.064,     # measured 0.021
       abs(loss2.item() - loss.item()) / abs(predicted))
    ck.done()
