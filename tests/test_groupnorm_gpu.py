"""The one-CTA GroupNorm (planes of at most 128 x 128 pixels, one CTA per image) through the real library against float64
references on the GPU: cd_groupnorm_fwd / cd_groupnorm_bwd against torch's F.group_norm and autograd, on every plane of the DDPM
`Model` at 32², 64² and 128² and at the edges of the kernels' thread mapping, and the `Model` itself at the benchmarked 32²
configuration with its GroupNorm inputs shifted to means of tens, against oracle/model2_oracle.py.

The inputs carry means of 0 and 100: statistics formed as E[v²] - mean² in fp32 lose about 1e-3 at a mean of 100, which the
shifted cases and their negative controls (the same one-pass statistics computed by torch in fp32) show.  As in
tests/test_model_large_gpu.py every bound is at most 3x the value measured on an H100 80GB HBM3 (700 W), and every comparison
also evaluates a deliberately wrong reference that must exceed the bound.  COLDDIFF_TEST_METRICS=<file> writes all values as
JSON."""
import ctypes as C

import pytest
import torch

import model2_oracle as MO
from test_config3_step_gpu import Checks, _metrics_file, _free_between_tests, _METRICS, rel, call, ptr, stream, gen  # noqa: F401
from test_model_large_gpu import (_fp64_time_embedding, _gn64, _fp32_one_pass, _model, _ref_grads, _grads,  # noqa: F401
                                  _grad_check, DEV, F64)

pytestmark = pytest.mark.gpu

# (id, B, HW, C, groups): the planes of the `Model` at 32², 64² and 128² (4² ... 128², C = 128 and 256); C = 36 with 4 groups
# (9 channel quads, 56 pixel lanes, 8 idle threads); C = 96 (24 quads that straddle groups of 3, 8 idle threads); C = 2048 (one
# pixel lane per quad); C = groups = 1536 (the backward's shared memory above 48 KB); 9 pixels at C = 128 (16 pixel lanes);
# 128² + 1 pixels, the smallest plane of the split-plane path, next to 128², the largest one-CTA plane
PLANES = [('%dsq-C%d' % (s, c), 4 if s <= 32 else 2, s * s, c, 32) for s in (4, 8, 16, 32, 64, 128) for c in (128, 256)] + [
    ('C36-g4', 3, 64, 36, 4), ('C96', 2, 1000, 96, 32), ('C2048', 2, 64, 2048, 32), ('C1536-g1536', 2, 64, 1536, 1536),
    ('9px-C128', 4, 9, 128, 32), ('128sq+1-C128-split', 2, 128 * 128 + 1, 128, 32)]

# measured on an H100 80GB HBM3 (700 W), by plane id: relative error of (forward, dx, dgamma, dbeta) and |dcond error| / (pixel
# sum of |dx|), at mean 0 and at mean 100.  Each bound is 3x its value.  GroupNorm kernels with the one-pass fp32 statistics
# E[v²] - mean² measured 1.7e-4 to 2.1e-3 on every metric at mean 100 except dcond (2.4e-5 to 8.3e-4).
MEASURED = {
    '4sq-C128': ((9.7e-8, 9.6e-8, 1.2e-7, 8.4e-8, 8.9e-8), (2.6e-6, 1.8e-6, 2.2e-6, 1.4e-6, 1.5e-6)),
    '4sq-C256': ((9.1e-8, 8.9e-8, 1.2e-7, 9.7e-8, 9.6e-8), (2.7e-6, 1.7e-6, 2.8e-6, 1.7e-6, 2.3e-6)),
    '8sq-C128': ((9.1e-8, 9.2e-8, 1.5e-7, 1.1e-7, 5.5e-8), (2.6e-6, 1.7e-6, 2.7e-6, 1.4e-6, 8.8e-7)),
    '8sq-C256': ((9.4e-8, 9.4e-8, 1.3e-7, 1.2e-7, 4.4e-8), (2.4e-6, 1.5e-6, 2.5e-6, 1.7e-6, 6.8e-7)),
    '16sq-C128': ((9.6e-8, 9.4e-8, 1.3e-7, 1.1e-7, 3.2e-8), (2.5e-6, 1.6e-6, 2.6e-6, 1.5e-6, 7.5e-7)),
    '16sq-C256': ((9.2e-8, 9.2e-8, 1.7e-7, 1.3e-7, 3.1e-8), (2.8e-6, 1.7e-6, 2.7e-6, 1.6e-6, 5.0e-7)),
    '32sq-C128': ((9.6e-8, 9.4e-8, 2.1e-7, 1.6e-7, 1.9e-8), (2.7e-6, 1.7e-6, 2.9e-6, 1.5e-6, 1.9e-7)),
    '32sq-C256': ((9.1e-8, 9.0e-8, 2.2e-7, 2.3e-7, 2.9e-8), (2.4e-6, 1.5e-6, 2.3e-6, 1.5e-6, 1.6e-7)),
    '64sq-C128': ((9.6e-8, 9.3e-8, 2.6e-7, 2.6e-7, 1.1e-8), (2.8e-6, 1.7e-6, 2.7e-6, 1.4e-6, 1.1e-7)),
    '64sq-C256': ((9.4e-8, 9.5e-8, 4.1e-7, 3.8e-7, 2.1e-8), (2.5e-6, 1.5e-6, 2.7e-6, 1.6e-6, 1.1e-7)),
    '128sq-C128': ((9.4e-8, 9.4e-8, 6.2e-7, 6.3e-7, 1.3e-8), (2.3e-6, 1.4e-6, 2.6e-6, 1.5e-6, 4.3e-8)),
    '128sq-C256': ((1.0e-7, 1.0e-7, 7.5e-7, 9.4e-7, 2.7e-8), (2.5e-6, 1.6e-6, 2.8e-6, 1.9e-6, 5.5e-8)),
    'C36-g4': ((9.7e-8, 9.2e-8, 2.2e-7, 1.5e-7, 4.4e-8), (2.5e-6, 1.6e-6, 3.2e-6, 1.5e-6, 5.4e-7)),
    'C96': ((9.6e-8, 9.3e-8, 1.9e-7, 1.7e-7, 1.6e-8), (2.5e-6, 1.6e-6, 2.6e-6, 1.2e-6, 3.2e-7)),
    'C2048': ((8.9e-8, 8.9e-8, 1.7e-7, 1.6e-7, 9.4e-8), (2.4e-6, 1.5e-6, 2.5e-6, 1.4e-6, 8.1e-7)),
    'C1536-g1536': ((1.5e-7, 1.5e-7, 2.2e-7, 1.6e-7, 9.8e-8), (1.5e-6, 1.0e-6, 1.6e-6, 9.2e-7, 8.4e-7)),
    '9px-C128': ((9.6e-8, 9.5e-8, 1.4e-7, 1.0e-7, 6.6e-8), (3.3e-6, 2.2e-6, 3.2e-6, 1.9e-6, 2.3e-6)),
    '128sq+1-C128-split': ((9.4e-8, 9.4e-8, 1.7e-7, 1.6e-7, 3.6e-9), (2.4e-6, 1.5e-6, 2.0e-6, 1.6e-6, 5.5e-8)),
}


def _bounds(pid, shift):
    return [3.0 * v for v in MEASURED[pid][shift > 0]]


@pytest.mark.parametrize('shift', [0.0, 100.0], ids=['mean0', 'mean100'])
@pytest.mark.parametrize('pid,B,HW,Cc,groups', PLANES, ids=[p[0] for p in PLANES])
def test_groupnorm_entry_points_against_fp64(pid, B, HW, Cc, groups, shift):
    ck = Checks('groupnorm %s mean %g' % (pid, shift))
    bf, bdx, bdg, bdb, bdc = _bounds(pid, shift)
    ld = Cc + 8
    g = gen(HW + Cc)
    x = torch.randn(B * HW, ld, generator=g, device=DEV) * 1.5 + shift
    cond = 0.5 * torch.randn(B, Cc, generator=g, device=DEV)
    gamma = 1 + 0.2 * torch.randn(Cc, generator=g, device=DEV)
    beta = 0.1 * torch.randn(Cc, generator=g, device=DEV)
    dy = torch.randn(B * HW, ld, generator=g, device=DEV)
    xs = x[:, :Cc].contiguous()
    y = torch.full((B * HW, ld), 7.0, device=DEV)
    call('cd_groupnorm_fwd', ptr(x), ld, B, C.c_int64(HW), Cc, groups, ptr(cond), Cc, ptr(gamma), ptr(beta), C.c_float(1e-6), 1,
         ptr(y), ld, stream())
    # backward: dgamma / dbeta accumulate onto 0.5 / -0.25
    dx = torch.full((B * HW, ld), 7.0, device=DEV)
    dg, db, dc = torch.full((Cc,), 0.5, device=DEV), torch.full((Cc,), -0.25, device=DEV), torch.full((B, Cc), 3.0, device=DEV)
    call('cd_groupnorm_bwd', ptr(x), ld, B, C.c_int64(HW), Cc, groups, ptr(cond), Cc, ptr(gamma), ptr(beta), C.c_float(1e-6), 1,
         ptr(dy), ld, ptr(dx), ld, ptr(dg), ptr(db), ptr(dc), Cc, stream())
    torch.cuda.synchronize()
    ck.require('row padding untouched', bool((y[:, Cc:] == 7.0).all()) and bool((dx[:, Cc:] == 7.0).all()))
    x64, c64, g64, b64 = (t.to(F64).requires_grad_() for t in (xs, cond, gamma, beta))
    ref = _gn64(x64, c64, g64, b64, True, B, HW, Cc, groups)
    ref.backward(dy[:, :Cc].to(F64).view(B, HW, Cc))
    yv, dxv, dx64 = y[:, :Cc].view(B, HW, Cc), dx[:, :Cc].view(B, HW, Cc), x64.grad.view(B, HW, Cc)
    scale = dx64.abs().sum(1).max().item()
    if shift:
        # the controls: GroupNorm with the fp32 one-pass statistics and its fp32 autograd
        x32, c32, g32, b32 = (t.clone().requires_grad_() for t in (xs, cond, gamma, beta))
        ctrl = _fp32_one_pass(x32, c32, g32, b32, B, HW, Cc, groups)
        ctrl.backward(dy[:, :Cc].reshape(B, HW, Cc))
        ctrl = ctrl.detach()
        cdx, cdg, cdb = rel(x32.grad.view(B, HW, Cc), dx64), rel(g32.grad, g64.grad), rel(b32.grad, b64.grad)
    else:
        # the controls: another image's output and dx, dgamma / dbeta without the accumulation
        ctrl = ref.detach().roll(1, 0)
        cdx, cdg, cdb = rel(dxv.roll(1, 0), dx64), rel(dg, g64.grad), rel(db, b64.grad)
    ck('forward', rel(yv, ref.detach()), bf, rel(ctrl, ref.detach()))
    ck('dx', rel(dxv, dx64), bdx, cdx)
    ck('dgamma', rel(dg - 0.5, g64.grad), bdg, cdg)
    ck('dbeta', rel(db + 0.25, b64.grad), bdb, cdb)
    # dcond = the pixel sum of dx: bounded against the terms' size.  Most of the statistics' error cancels in that sum (the
    # one-pass fp32 control measures about 4e-6 on small planes, near the bound), so the control leaves dcond unwritten
    ck('dcond (abs / pixel sum of |dx|)', (dc.to(F64) - c64.grad).abs().max().item() / scale, bdc, 3.0 / scale)
    ck.done()


# ==========================================================================================================================
# the `Model` at 32² (ch = 128, ch_mult = (1, 2, 2, 2), attention at 16²) with GroupNorm inputs of means of tens
# ==========================================================================================================================
def _one_pass_gn(sd, p, x):
    """GroupNorm(32) with the one-pass statistics E[v²] - mean² in the dtype of x"""
    v = x.reshape(x.shape[0], 32, -1)
    mean = v.mean(-1, keepdim=True)
    var = ((v * v).mean(-1, keepdim=True) - mean * mean).clamp_min(0)
    xh = ((v - mean) * torch.rsqrt(var + 1e-6)).view_as(x)
    return xh * sd[p + '.weight'][:, None, None] + sd[p + '.bias'][:, None, None]


def _fp32_one_pass_model(monkeypatch, sd, x, target, t, norm):
    """the network in fp32 (no TF32) with one-pass GroupNorm statistics -> (output, gradients by name): the negative control"""
    temb64 = MO.timestep_embedding
    with monkeypatch.context() as mp:
        mp.setattr(MO, 'gn', _one_pass_gn)
        mp.setattr(MO, 'timestep_embedding', lambda tt, dim: temb64(tt, dim).float())
        mp.setattr(torch.backends.cudnn, 'allow_tf32', False)
        mp.setattr(torch.backends.cuda.matmul, 'allow_tf32', False)
        leaves = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
        names = [k for k in leaves if leaves[k].requires_grad]
        y = MO.model_forward(leaves, x, t, ch=128, num_resolutions=4, num_res_blocks=2)
        d = target - y
        grads = torch.autograd.grad((d * d).sum() / norm, [leaves[k] for k in names])
    return y.detach(), dict(zip(names, grads))


def test_model_32_with_shifted_groupnorm_inputs(monkeypatch):
    """fp32 CUDA-core convolutions (CONV_SIMT), so that no TF32 rounding hides a GroupNorm error; conv_in and every temb_proj
    get a large bias, so every GroupNorm of the network sees a mean of tens"""
    from cold_diffusion_models_b200.ops import CONV_SIMT
    ck = Checks('model 32 shifted')
    S, B = 32, 2
    m = _model(S, seed=4)
    with torch.no_grad():
        m.conv_in.bias += 40.0
        for n, p in m.named_parameters():
            if n.endswith('temb_proj.bias'):
                p += 20.0
    m.engine.mark_weights_dirty()
    m.conv_impl = CONV_SIMT
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.rand(B, 3, S, S, generator=gen(21), device=DEV) * 2 - 1
    target = torch.rand(B, 3, S, S, generator=gen(22), device=DEV) * 2 - 1
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
    yc, gc = _fp32_one_pass_model(monkeypatch, sd, x, target, t, x.numel())
    with torch.no_grad():
        # measured 8.3e-7 on both paths; the fp32 network with one-pass statistics gives 2.3e-5, and GroupNorm kernels with the
        # one-pass statistics measured 6.5e-5
        ck('forward', rel(y.detach(), y64), 2.4e-6, rel(yc, y64))
        yi = m.eval()(x, t)                                          # the inference path (no autograd)
        ck('inference forward', rel(yi, y64), 2.4e-6, rel(yc, y64))
    # measured median 2.7e-6, worst 1.15e-5 (the control: 2.5e-4 and 7.7e-4; GroupNorm kernels with the one-pass statistics:
    # 7.1e-4 and 2.2e-3)
    _grad_check(ck, 'grad', eg, ref, gc, 7.8e-6, 3.4e-5)
    ck.done()
