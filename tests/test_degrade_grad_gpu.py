"""`GaussianDiffusion.degrade` of every package: its gradients against float64 torch autograd of the oracles, its values against
`q_sample` (bit for bit), `q_sample` left detached, the cases that refuse a gradient, and one reconstruction-guidance step
through a frozen config-3 Unet.

Each gradient comparison uses L = <degrade(x), w> with a random w, so dx is the adjoint applied to w.  It also evaluates its
metric against a wrong reference (a negative control: A w A^T instead of A^T w A, swapped lerp coefficients, swapped mask
windows, the mix of the next step) and asserts that the control lands at least 10x past the bound.  The bounds are at most
3x the values measured on an H100 80GB HBM3 (700 W), given beside them.  Set COLDDIFF_TEST_METRICS=<file> to write every value and
control as JSON."""
import contextlib
import io

import pytest
import torch

import deblur_oracle as DO
import defading_gen_oracle as DGO
import defading_oracle as DFO
import denoise_oracle as DNO
import resolution_oracle as RO
import snow_oracle as SO
import unet_oracle as UO
from test_config3_step_gpu import Checks, _metrics_file, _free_between_tests, rel, gen  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
TF32_BOUND = 1.5e-3                  # the TF32 input-gradient bound of tests/test_input_grad_gpu.py
BLUR = dict(timesteps=20, kernel_size=15, kernel_std=0.1, blur_routine='Exponential_reflect')


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _images(B, Cc, S, seed):
    return torch.rand(B, Cc, S, S, generator=gen(seed), device=DEV) * 2 - 1


def _grads(fn, xs, w):
    """(out, [d<fn(*xs), w>/dx for x in xs]) with the engine"""
    xr = [x.clone().requires_grad_(True) for x in xs]
    out = fn(*xr)
    (out * w).sum().backward()
    torch.cuda.synchronize()
    return out.detach(), [x.grad.detach() for x in xr]


def _ref_grads(fn, xs, w):
    """float64 autograd of the oracle"""
    xr = [x.to(F64).requires_grad_(True) for x in xs]
    out = fn(*xr)
    return torch.autograd.grad((out * w.to(F64)).sum(), xr)


# ==========================================================================================================================
# the blur family: deblurring and resolution
# ==========================================================================================================================
def _deblur(S, discrete=False):
    import cold_diffusion_models_b200 as cdm
    gd = _quiet(cdm.GaussianDiffusion, torch.nn.Identity(), image_size=S, device_of_kernel=DEV, channels=3, discrete=discrete, **BLUR)
    return gd.to(DEV)


def _deblur_oracle(S):
    o = DO.DeblurOracle(None, image_size=S, channels=3, **BLUR)
    o.kernels2d = [k.to(DEV, F64) for k in o.kernels2d]
    return o


def _resolution(S, T=8):
    from cold_diffusion_models_b200.resolution import GaussianDiffusion
    return _quiet(GaussianDiffusion, torch.nn.Identity(), image_size=S, device_of_kernel=DEV, channels=3, timesteps=T).to(DEV)


# (package, S, B, t, bound): t values per sample; resolution's -1 rows take the level max(t), as its q_sample does.  The bound
# holds the forward values and dx against float64, measured (forward / dx): deblurring 128 9.7e-8 / 9.7e-8, 256 1.68e-7 /
# 1.71e-7, 512 2.69e-7 / 2.70e-7; resolution 128 1.02e-7 / 1.02e-7, 256 6.0e-8 / 6.0e-8
BLUR_CASES = [
    ('deblurring', 128, 3, [0, 19, 9], 2.5e-7),
    ('deblurring', 256, 3, [19, 4, 11], 4.5e-7),
    ('deblurring', 512, 1, [17], 7e-7),
    ('resolution', 128, 3, [7, -1, 2], 2.5e-7),
    ('resolution', 256, 2, [5, 0], 1.5e-7),
]


@pytest.mark.parametrize('case', BLUR_CASES, ids=['%s-%d' % (c[0], c[1]) for c in BLUR_CASES])
def test_blur_family_gradient(case):
    name, S, B, tl, bound = case
    ck = Checks('degrade grad %s %d' % (name, S))
    t = torch.tensor(tl, device=DEV)
    x, w = _images(B, 3, S, seed=S + 1), _images(B, 3, S, seed=S + 2)
    if name == 'deblurring':
        gd, o = _deblur(S), _deblur_oracle(S)
        oracle = lambda v: o.q_sample(v, t)
    else:
        gd = _resolution(S)
        o = RO.ResolutionOracle(None, image_size=S, channels=3, timesteps=gd.num_timesteps)
        oracle = lambda v: o.q_sample(v, torch.where(t < 0, t.max(), t))
    out, (dx,) = _grads(lambda v: gd.degrade(v, t), [x], w)
    (ref,) = _ref_grads(oracle, [x], w)
    with torch.no_grad():
        ctrl = oracle(w.to(F64))                    # A w A^T: the forward operator instead of its transpose
    ck('forward vs float64', rel(out, oracle(x.to(F64)).detach()), bound)
    ck('dx', rel(dx, ref), bound, rel(dx, ctrl))
    ck.require('control not 10x past the bound', rel(dx, ctrl) > 10 * bound)
    ck.done()


@pytest.mark.parametrize('S', [128, 256])
def test_blur_adjoint_collapse(S):
    """the `discrete` mean-collapse at T-1 without its truncation (BlurDegrade with quantize = 0): the gradient of
    mean(A X A^T) 11^T, A^T (mean(w) 11^T) A, on both the one-CTA and the row-strip kernels"""
    from cold_diffusion_models_b200.autograd import BlurDegrade
    ck = Checks('degrade collapse %d' % S)
    gd, o = _deblur(S), _deblur_oracle(S)
    T = gd.num_timesteps
    t = torch.tensor([T - 1, 3], device=DEV)
    x, w = _images(2, 3, S, seed=S + 3), _images(2, 3, S, seed=S + 4)

    def oracle(v):
        y = o.q_sample(v, t)
        return torch.cat([y[:1].mean((2, 3), keepdim=True).expand_as(y[:1]), y[1:]])
    _, (dx,) = _grads(lambda v: BlurDegrade.apply(v, gd._ops_cum, t, -1, T, 1, 0), [x], w)
    (ref,) = _ref_grads(oracle, [x], w)
    with torch.no_grad():
        ctrl = o.q_sample(w.to(F64), t)            # the adjoint without the collapse (and transposed)
    bound = 3.5e-7                                 # measured: 128 1.32e-7, 256 1.35e-7
    ck('dx', rel(dx, ref), bound, rel(dx, ctrl))
    ck.require('control not 10x past the bound', rel(dx, ctrl) > 10 * bound)
    ck.done()


# ==========================================================================================================================
# elementwise families
# ==========================================================================================================================
def test_defading_mask_gradient():
    """'Random_Incremental': every sample reads its own window of the 2S x 2S masks; control = the windows swapped"""
    from cold_diffusion_models_b200.defading import GaussianDiffusion
    S, T = 64, 10
    kw = dict(image_size=S, channels=3, timesteps=T, kernel_std=0.1, initial_mask=11, fade_routine='Random_Incremental')
    gd = _quiet(GaussianDiffusion, torch.nn.Identity(), device_of_kernel=DEV, **kw).to(DEV)
    o = DFO.DefadeOracle(None, **kw)
    o.fade_kernels = o.fade_kernels.to(DEV, F64)
    t = torch.tensor([9, 0, 4], device=DEV)
    rx, ry = torch.tensor([0, 40, 17], device=DEV), torch.tensor([33, 2, 60], device=DEV)
    x, w = _images(3, 3, S, seed=31), _images(3, 3, S, seed=32)
    out, (dx,) = _grads(lambda v: gd.degrade(v, t, _offsets=(rx, ry)), [x], w)
    (ref,) = _ref_grads(lambda v: o.q_sample(v, t, rx, ry), [x], w)
    (ctrl,) = _ref_grads(lambda v: o.q_sample(v, t, ry, rx), [x], w)
    ck = Checks('degrade grad defading')
    bound = 1.4e-8                                 # measured: 4.95e-9
    ck('dx', rel(dx, ref), bound, rel(dx, ctrl))
    ck.require('control not 10x past the bound', rel(dx, ctrl) > 10 * bound)
    ck.done()


# (d x_start, d x_end) bounds; measured: defading_generation 1.41e-8, 2.23e-8; denoising and demixing 2.38e-8, 2.39e-8
LERP_BOUNDS = {'defading_generation': (4e-8, 6e-8), 'denoising': (6e-8, 6e-8), 'demixing': (6e-8, 6e-8)}


@pytest.mark.parametrize('package', ['defading_generation', 'denoising', 'demixing'])
def test_lerp_gradients(package):
    """both images' gradients of the two lerps; control = the two coefficients swapped"""
    import importlib
    mod = importlib.import_module('cold_diffusion_models_b200.' + package)
    S, T, B = 64, 30, 3
    if package == 'defading_generation':
        gd = _quiet(mod.GaussianDiffusion, torch.nn.Identity(), image_size=S, channels=3, timesteps=T, kernel_std=0.15,
                    initial_mask=11).to(DEV)
        o = DGO.DefadingGenOracle(None, image_size=S, channels=3, timesteps=T, kernel_std=0.15, initial_mask=11)
        o.alphas, o.one_minus_alphas = o.alphas.to(DEV, F64), o.one_minus_alphas.to(DEV, F64)
    else:
        gd = _quiet(mod.GaussianDiffusion, torch.nn.Identity(), image_size=S, channels=3, timesteps=T).to(DEV)
        o = DNO.DenoiseOracle(None, image_size=S, channels=3, timesteps=T)
        o.sa, o.sb = o.sa.to(DEV, F64), o.sb.to(DEV, F64)
    t = torch.tensor([0, 29, 12], device=DEV)
    x1, x2, w = _images(B, 3, S, seed=41), _images(B, 3, S, seed=42), _images(B, 3, S, seed=43)
    _, (d1, d2) = _grads(lambda a, b: gd.degrade(a, b, t), [x1, x2], w)
    r1, r2 = _ref_grads(lambda a, b: o.q_sample(a, b, t), [x1, x2], w)
    ck = Checks('degrade grad ' + package)
    b1, b2 = LERP_BOUNDS[package]
    ck('d x_start', rel(d1, r1), b1, rel(d1, r2))
    ck('d x_end', rel(d2, r2), b2, rel(d2, r1))
    ck.require('controls not 10x past the bound', rel(d1, r2) > 10 * b1 and rel(d2, r1) > 10 * b2)
    # one input only: the other gets no gradient
    xr = x1.clone().requires_grad_(True)
    (gd.degrade(xr, x2, t) * w).sum().backward()
    ck('d x_start alone', rel(xr.grad, r1), b1)
    ck.done()


def _decolor(S, T, to_lab=False):
    from cold_diffusion_models_b200.snowification import GaussianDiffusion
    return _quiet(GaussianDiffusion, torch.nn.Identity(), image_size=S, device_of_kernel=DEV, channels=3, timesteps=T,
                  forward_process_type='Decolorization', decolor_routine='Linear', decolor_total_remove=False,
                  to_lab=to_lab).to(DEV)


def test_decolor_gradient():
    """the per-pixel C x C mix, with q_sample's t = -1 quirk; control = the mix of the next step"""
    S, T = 64, 12
    gd = _decolor(S, T)
    fp = SO.DecolorFP(gd.forward_process.factors, 3)
    fp.w = [m.to(DEV, F64) for m in fp.w]
    o = SO.SnowOracle(None, fp, timesteps=T)
    t = torch.tensor([-1, 5, 2, 10], device=DEV)
    x, w = _images(4, 3, S, seed=51), _images(4, 3, S, seed=52)
    _, (dx,) = _grads(lambda v: gd.degrade(v, t), [x], w)
    (ref,) = _ref_grads(lambda v: o.q_sample(v, t), [x], w)
    (ctrl,) = _ref_grads(lambda v: o.q_sample(v, torch.where(t >= 0, t + 1, t)), [x], w)
    ck = Checks('degrade grad decolor')
    bound = 8e-8                                   # measured: 3.07e-8
    ck('dx', rel(dx, ref), bound, rel(dx, ctrl))
    ck.require('control not 10x past the bound', rel(dx, ctrl) > 10 * bound)
    ck.done()


def test_chanmix_transposes_the_table():
    """the decolor mixes are symmetric, so the transposed table is checked with a random one: dx = M_t^T w per pixel"""
    from cold_diffusion_models_b200.autograd import ChanmixDegrade
    T, Cc, S = 5, 4, 32
    mats = torch.randn(T, Cc, Cc, generator=gen(61), device=DEV)
    t = torch.tensor([4, -1, 0], device=DEV)
    x, w = _images(3, Cc, S, seed=62), _images(3, Cc, S, seed=63)
    _, (dx,) = _grads(lambda v: ChanmixDegrade.apply(v, mats, mats.transpose(1, 2).contiguous(), t), [x], w)
    eye = torch.eye(Cc, device=DEV, dtype=F64)
    M = torch.stack([mats[int(i)].to(F64) if i >= 0 else eye for i in t])
    ref = torch.einsum('bji,bjhw->bihw', M, w.to(F64))
    ctrl = torch.einsum('bij,bjhw->bihw', M, w.to(F64))
    ck = Checks('degrade chanmix transpose')
    bound = 1e-7                                   # measured: 3.92e-8
    ck('dx', rel(dx, ref), bound, rel(dx, ctrl))
    ck.require('control not 10x past the bound', rel(dx, ctrl) > 10 * bound)
    ck.done()


# ==========================================================================================================================
# values, detachment, refusals
# ==========================================================================================================================
def _all_packages():
    """(name, module, degrade args, q_sample args) for every package and variant"""
    from cold_diffusion_models_b200 import defading, defading_generation, demixing, denoising, resolution, snowification
    S, B = 32, 3
    x, x2 = _images(B, 3, S, seed=71), _images(B, 3, S, seed=72)
    t = torch.tensor([3, 0, 7], device=DEV)
    out = []
    for disc in (False, True):
        out.append(('deblurring discrete=%s' % disc, _deblur(S, disc), (x, t), {}))
    out.append(('deblurring 256', _deblur(256), (_images(2, 3, 256, seed=73), torch.tensor([2, 19], device=DEV)), {}))
    r = _resolution(S)
    out.append(('resolution t=-1', r, (x, torch.tensor([-1, 2, 5], device=DEV)), {}))
    for disc in (False, True):
        gd = _quiet(defading.GaussianDiffusion, torch.nn.Identity(), image_size=S, device_of_kernel=DEV, channels=3, timesteps=10,
                    fade_routine='Random_Incremental', discrete=disc).to(DEV)
        offs = (torch.tensor([1, 30, 7], device=DEV), torch.tensor([20, 0, 32], device=DEV))
        out.append(('defading discrete=%s' % disc, gd, (x, t), dict(_offsets=offs)))
    gd = _quiet(defading_generation.GaussianDiffusion, torch.nn.Identity(), image_size=S, channels=3, timesteps=10).to(DEV)
    out.append(('defading_generation', gd, (x, x2, t), {}))
    out.append(('defading_generation int t', gd, (x, x2, 6), {}))
    for mod in (denoising, demixing):
        gd = _quiet(mod.GaussianDiffusion, torch.nn.Identity(), image_size=S, channels=3, timesteps=10).to(DEV)
        out.append((mod.__name__.split('.')[-1], gd, (x, x2, t), {}))
    tq = torch.tensor([-1, 2, 9], device=DEV)
    out.append(('decolor', _decolor(S, 10), (x, tq), {}))
    out.append(('decolor lab', _decolor(S, 10, to_lab=True), (x, tq), {}))
    snow = _quiet(snowification.GaussianDiffusion, torch.nn.Identity(), image_size=S, device_of_kernel=DEV, channels=3, timesteps=10,
                  forward_process_type='Snow').to(DEV)
    out.append(('snow', snow, (x, tq), {}))
    return out


def test_degrade_equals_q_sample_and_q_sample_stays_detached():
    bad = []
    for name, gd, args, kw in _all_packages():
        want = gd.q_sample(*args, **kw)
        with torch.no_grad():
            got = gd.degrade(*args, **kw)
        if not torch.equal(got, want):
            bad.append('%s: degrade != q_sample' % name)
        if not (name.startswith('snow') or 'lab' in name or 'discrete=True' in name):
            xr = [a.clone().requires_grad_(True) if torch.is_tensor(a) and a.is_floating_point() else a for a in args]
            got = gd.degrade(*xr, **kw)
            if not torch.equal(got.detach(), want) or got.grad_fn is None:
                bad.append('%s: differentiable degrade differs or has no grad_fn' % name)
            q = gd.q_sample(*xr, **kw)
            if q.grad_fn is not None or q.requires_grad:
                bad.append('%s: q_sample is attached to the graph' % name)
    assert not bad, bad


def test_refusals():
    """no derivative: `discrete`, snow and the Lab decolor path raise when a gradient is requested, and run without one"""
    cases = [c for c in _all_packages() if c[0] in ('deblurring discrete=True', 'defading discrete=True', 'snow', 'decolor lab')]
    assert len(cases) == 4
    for name, gd, args, kw in cases:
        xr = args[0].clone().requires_grad_(True)
        with pytest.raises(RuntimeError, match='not differentiable'):
            gd.degrade(xr, *args[1:], **kw)
        with torch.no_grad():
            assert torch.equal(gd.degrade(xr, *args[1:], **kw), gd.q_sample(args[0], *args[1:], **kw)), name


def test_create_graph_raises():
    for name, gd, args, kw in _all_packages():
        if name.startswith('snow') or 'lab' in name or 'discrete=True' in name or 'int t' in name:
            continue
        xr = args[0].clone().requires_grad_(True)
        y = gd.degrade(xr, *args[1:], **kw)
        loss = ((y - 0.5) ** 2).sum()
        with pytest.raises(RuntimeError, match='first order'):
            torch.autograd.grad(loss, [xr], create_graph=True)


# ==========================================================================================================================
# reconstruction guidance through a frozen Unet
# ==========================================================================================================================
def test_guidance_step_through_frozen_unet():
    """x_t.grad of ||degrade(R(x_t, t), s) - y||^2 with a frozen config-3 Unet at 128², B = 4, against float64 autograd of
    oracle/unet_oracle.py composed with the blur oracle.  Control: the degradation's backward with A instead of A^T."""
    import cold_diffusion_models_b200 as cdm
    S, B = 128, 4
    sd = UO.make_unet_state_dict(64, (1, 2, 4, 8), 3, seed=3)
    u = _quiet(cdm.Unet, 64, dim_mults=(1, 2, 4, 8), channels=3)
    u.load_state_dict(sd)
    u = u.to(DEV).requires_grad_(False)
    gd = _deblur(S)
    o = _deblur_oracle(S)
    x_t, y = _images(B, 3, S, seed=81), _images(B, 3, S, seed=82) * 0.5
    t = torch.tensor([19, 5, 12, 0], device=DEV)
    s = torch.tensor([4, 2, 9, 0], device=DEV)
    xr = x_t.clone().requires_grad_(True)
    ((gd.degrade(u(xr, t), s) - y) ** 2).sum().backward()
    torch.cuda.synchronize()
    sd64 = {k: v.detach().to(DEV, F64) for k, v in u.state_dict().items()}
    x64 = x_t.to(F64).requires_grad_(True)
    R = UO.unet_forward(sd64, x64, t.to(F64))
    d = o.q_sample(R, s) - y.to(F64)
    (ref,) = torch.autograd.grad((d ** 2).sum(), x64, retain_graph=True)
    with torch.no_grad():
        wrong = o.q_sample(2 * d, s)                    # A (2d) A^T reaching R instead of A^T (2d) A
    (ctrl,) = torch.autograd.grad(R, x64, wrong)
    ck = Checks('guidance step')
    # measured: 1.20e-3 (the control 2.8e-2)
    ck('x_t.grad (TF32)', rel(xr.grad, ref), TF32_BOUND, rel(xr.grad, ctrl))
    ck.require('control not 10x past the bound', rel(xr.grad, ctrl) > 10 * TF32_BOUND)
    ck.require('a frozen parameter got a .grad', all(p.grad is None for p in u.parameters()))
    ck.done()
