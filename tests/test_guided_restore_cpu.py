"""Guided restoration (`GaussianDiffusion.restore`) without a GPU.

* The new entry points run from their CUDA source on the CPU (tests/simt_cpu) against float64 numpy: the guidance gradients
  D_s^T (D_s x0 - y) of the blur / resize family (one pass up to 128², two passes above; dense random and reflect-blur
  operators, neither symmetric), of the masks (per-sample `Random_*` windows) and of the channel mixes, and the guided updates
  with their "- weight g" epilogue.  With g = NULL each update is the unguided kernel bit for bit.
* The adjoint identity <D_s x, r> = <x, D_s^T r> that the guidance gradient rests on, with the emulated forward.
* The packages' `restore` on the emulated ABI (numpy statements of tests/guided_oracle.py, and the CUDA sources): weight = 0 is
  `sample`'s final image bit for bit, weight > 0 matches the float64 restatement, parameters come back as they were, and the
  refusals raise ValueError."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'simt_cpu'))

import abi_emulator  # noqa: E402
import guided_oracle as GO  # noqa: E402
import strided_oracle as SO  # noqa: E402
from test_blur_large_cpu import P, images, operators, ref_apply, apply, step_down, rel  # noqa: E402

F64 = torch.float64
NULL = C.c_void_p(0)


@pytest.fixture(scope='module', params=['ascending', 'descending'])
def lib(request):
    """threads of a block resumed in ascending / descending order: a missing barrier shows under at least one of them"""
    import build
    lib = C.CDLL(build.build_all())
    lib.simt_set_reverse_order(int(request.param == 'descending'))
    yield lib
    lib.simt_set_reverse_order(0)


def ref_guide(x, y, ops, idx):
    """float64 A^T (A X A^T - Y) A per plane (idx < 0: X - Y)"""
    R = ref_apply(x, ops, idx) - y.double().numpy()
    if idx < 0:
        return R
    A = ops[idx].double().numpy()
    return np.einsum('ji,...jk,kl->...il', A, R, A)


def blur_guide(lib, x, y, ops, idx, work=True):
    B, Cc, S, _ = x.shape
    out = torch.full_like(x, float('nan'))
    ws = torch.full_like(x, float('nan')) if work else None
    assert lib.cd_blur_guide_grad(P(x), P(y), P(out), P(ws), P(ops), idx, B, Cc, S, ops.shape[0], NULL) == 0
    return out


def blur_step(lib, xt, xhat, g, w, ops, hi, lo):
    B, Cc, S, _ = xhat.shape
    out = torch.full_like(xhat, float('nan'))
    assert lib.cd_blur_guided_step(P(xt), P(xhat), P(g), C.c_float(w), P(out), P(ops), hi, lo, B, Cc, S, ops.shape[0], NULL) == 0
    return out


def dot(a, b):
    return float((torch.as_tensor(a).double() * torch.as_tensor(b).double()).sum())


# ---- blur / resize family ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('S,kind', [(32, 'blur'), (32, 'dense'), (128, 'dense'), (132, 'blur'), (132, 'dense')])
def test_blur_guide_grad_matches_float64(lib, S, kind):
    """one pass up to 128² (the residual on chip), the apply with a '- y' epilogue and the adjoint above"""
    T = 4
    ops = operators(S, T, kind, seed=31)
    Cc = 2 if S <= 128 else 1
    x, y = images(2, Cc, S, seed=32), images(2, Cc, S, seed=33)
    for idx in (2, -1):
        got = blur_guide(lib, x, y, ops, idx, work=S > 128)
        want = ref_guide(x, y, ops, idx)
        assert rel(got, want) < 1e-5, (idx, rel(got, want))
        if idx >= 0:
            # controls: y subtracted (not D^T D x), and the adjoint applied (not the forward operator twice)
            assert rel(got, ref_guide(x, torch.zeros_like(y), ops, idx)) > 1e-2
            assert rel(got, ref_apply(torch.from_numpy(ref_apply(x, ops, idx) - y.double().numpy()), ops, idx)) > 1e-2


@pytest.mark.parametrize('S', [32, 132])
def test_blur_guide_grad_rests_on_the_adjoint_identity(lib, S):
    """<D x, r> = <x, D^T r>: with x0 = 0 the guidance gradient is -D^T y, and D is the emulated cd_blur_apply"""
    ops = operators(S, 3, 'dense', seed=34)
    x, r = images(1, 2, S, seed=35), images(1, 2, S, seed=36)
    dt_r = -blur_guide(lib, torch.zeros_like(x), r, ops, 1)
    lhs, rhs = dot(apply(lib, x, ops, t_scalar=1), r), dot(x, dt_r)
    assert abs(lhs - rhs) < 1e-5 * (abs(lhs) + abs(rhs) + 1), (lhs, rhs)


@pytest.mark.parametrize('S', [32, 132])
def test_blur_guided_step(lib, S):
    T = 5
    ops = operators(S, T, 'dense', seed=37)
    xt, xhat, g = images(2, 1, S, seed=38), images(2, 1, S, seed=39), images(2, 1, S, seed=40)
    w = 0.37
    for hi, lo in ((4, 1), (2, -1)):
        got = blur_step(lib, xt, xhat, g, w, ops, hi, lo)
        want = xt.double().numpy() - ref_apply(xhat, ops, hi) + ref_apply(xhat, ops, lo) - w * g.double().numpy()
        assert rel(got, want) < 1e-5, (hi, lo)
        assert torch.equal(blur_step(lib, xt, xhat, None, w, ops, hi, lo), step_down(lib, xt, xhat, ops, hi, lo))
        got = blur_step(lib, None, xhat, g, w, ops, hi, lo)
        assert rel(got, ref_apply(xhat, ops, lo) - w * g.double().numpy()) < 1e-5, (hi, lo)
        assert torch.equal(blur_step(lib, None, xhat, None, w, ops, hi, lo), apply(lib, xhat, ops, t_scalar=lo))


def test_blur_guide_grad_refusals(lib):
    def err():
        buf = C.create_string_buffer(512)
        lib.cd_last_error(buf, 512)
        return buf.value
    ops = torch.zeros(1, 132, 132)
    x = torch.zeros(1, 1, 132, 132)
    assert lib.cd_blur_guide_grad(P(x), P(x), P(x.clone()), NULL, P(ops), 0, 1, 1, 132, 1, NULL) != 0
    assert b'needs a workspace' in err()
    for S in (516, 130):
        x = torch.zeros(1, 1, S, S)
        ops = torch.zeros(1, S, S)
        assert lib.cd_blur_guide_grad(P(x), P(x), P(x.clone()), P(x.clone()), P(ops), 0, 1, 1, S, 1, NULL) != 0
        assert b'image size %d unsupported' % S in err()
        assert lib.cd_blur_guided_step(NULL, P(x), P(x), C.c_float(1.0), P(x.clone()), P(ops), 0, 0, 1, 1, S, 1, NULL) != 0


# ---- masks and channel mixes ---------------------------------------------------------------------------------------------
def _masks(S, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(T, 2 * S, 2 * S, generator=g).contiguous()


def _window(masks, idx, rx, ry, S):
    if idx < 0:
        return torch.ones(len(rx), 1, S, S, dtype=F64)
    return torch.stack([masks[idx, int(a):int(a) + S, int(b):int(b) + S].double() for a, b in zip(rx, ry)])[:, None]


@pytest.mark.parametrize('backend', ['numpy', 'cuda_source'])
def test_mask_guide_grad_and_step(backend):
    GO.install_emulator()
    call = abi_emulator.call if backend == 'numpy' else abi_emulator.call_cuda_source
    S, T, B, Cc = 12, 6, 3, 2
    masks = _masks(S, T, 41)
    rx, ry = torch.tensor([0, 7, 12]), torch.tensor([5, 12, 1])
    x, y, g, xt = (images(B, Cc, S, seed=s) for s in (42, 43, 44, 45))
    for idx in (4, -1):
        out = torch.full_like(x, float('nan'))
        call('cd_mask_guide_grad', P(x), P(y), P(out), P(masks), idx, P(rx), P(ry), B, Cc, S, 2 * S, NULL)
        m = _window(masks, idx, rx, ry, S)
        assert rel(out, m * (m * x.double() - y.double())) < 1e-6
        if idx >= 0:     # the windows are per sample and not swapped
            assert rel(out, _window(masks, idx, ry, rx, S) * (_window(masks, idx, ry, rx, S) * x.double() - y.double())) > 1e-2
    w = 0.6
    for hi, lo in ((5, 2), (1, -1)):
        mh, ml = _window(masks, hi, rx, ry, S), _window(masks, lo, rx, ry, S)
        for xt_ in (xt, None):
            out, plain, unguided = (torch.full_like(x, float('nan')) for _ in range(3))
            call('cd_mask_guided_step', P(xt_), P(x), P(g), C.c_float(w), P(out), P(masks), hi, lo, P(rx), P(ry), B, Cc, S, 2 * S, NULL)
            base = (xt.double() - x.double() * mh if xt_ is not None else 0) + x.double() * ml
            assert rel(out, base - w * g.double()) < 1e-6, (hi, lo, xt_ is None)
            call('cd_mask_guided_step', P(xt_), P(x), NULL, C.c_float(w), P(unguided), P(masks), hi, lo, P(rx), P(ry), B, Cc, S, 2 * S,
                 NULL)
            if xt_ is None:
                call('cd_mask_apply', P(x), P(plain), P(masks), NULL, lo, P(rx), P(ry), B, Cc, S, 2 * S, 0, NULL)
            else:
                call('cd_mask_step_down', P(xt), P(x), P(plain), P(masks), hi, lo, P(rx), P(ry), B, Cc, S, 2 * S, NULL)
            assert torch.equal(unguided, plain)


@pytest.mark.parametrize('backend', ['numpy', 'cuda_source'])
def test_chanmix_guide_grad_and_step(backend):
    GO.install_emulator()
    call = abi_emulator.call if backend == 'numpy' else abi_emulator.call_cuda_source
    T, B, Cc, S = 5, 3, 3, 6
    gen = torch.Generator().manual_seed(46)
    mats = torch.randn(T, Cc, Cc, generator=gen).contiguous()          # not symmetric: a missing transpose shows
    x, y, g, xt = (images(B, Cc, S, seed=s) for s in (47, 48, 49, 50))
    t = torch.tensor([3, 0, 5])
    HW = C.c_int64(S * S)
    out = torch.full_like(x, float('nan'))
    call('cd_chanmix_guide_grad', P(x), P(y), P(out), P(mats), P(t), -1, B, Cc, HW, NULL)
    X, Y = x.double().flatten(2), y.double().flatten(2)
    for b in range(B):
        i = int(t[b]) - 1
        want = X[b] - Y[b] if i < 0 else mats[i].double().T @ (mats[i].double() @ X[b] - Y[b])
        assert rel(out[b].flatten(1), want) < 1e-6, b
        if i >= 0:
            assert rel(out[b].flatten(1), mats[i].double() @ (mats[i].double() @ X[b] - Y[b])) > 1e-2
    w = 1.3
    th, tl = torch.tensor([4, 2, 5]), torch.tensor([1, 0, 3])
    for mode in (0, 1):
        got, plain, unguided = (torch.full_like(x, float('nan')) for _ in range(3))
        xt_ = xt if mode else None
        tl_ = tl if mode else None
        call('cd_chanmix_guided', P(xt_), P(x), P(g), C.c_float(w), P(got), P(mats), P(th), P(tl_), -1, -1, B, Cc, HW, mode, NULL)
        call('cd_chanmix_guided', P(xt_), P(x), NULL, C.c_float(w), P(unguided), P(mats), P(th), P(tl_), -1, -1, B, Cc, HW, mode, NULL)
        call('cd_chanmix', P(xt_), P(x), P(plain), P(mats), P(th), P(tl_), -1, -1, B, Cc, HW, mode, NULL)
        assert torch.equal(unguided, plain)
        assert rel(got, plain.double() - w * g.double()) < 1e-6


# ---- the packages' restore on the emulated ABI ---------------------------------------------------------------------------
def net(x, t):
    """a small deterministic stand-in for the restoration network: smooth in x, depends on t"""
    return torch.tanh(0.8 * x + 0.01 * t.to(x.dtype)[:, None, None, None]) * 0.9


class _Net(torch.nn.Module):
    """net above, scaled by a parameter (1.0), so that the freezing of the parameters during restore is visible"""

    def __init__(self):
        super().__init__()
        self.scale = torch.nn.Parameter(torch.ones(()))

    def forward(self, x, t):
        return net(x, t) * self.scale


@pytest.fixture(params=['numpy', 'cuda_source'])
def emulated(request, monkeypatch):
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)
    SO.install_emulator()
    GO.install_emulator()
    with abi_emulator.patched(request.param):
        yield


def _image(S=16, B=2, seed=0):
    return torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def _packages(routine):
    """(name, diffusion, sample(x, steps) -> final image, D_s(x, s) of the package, float64 update, float64 D_s, restore kwargs)"""
    import deblur_oracle as DO, resolution_oracle as RO, defading_oracle as FO, snow_oracle as NO
    from cold_diffusion_models_b200 import deblurring, resolution, defading, snowification
    out = []
    kw = dict(image_size=16, channels=3, timesteps=8, kernel_std=0.3, kernel_size=5, blur_routine='Exponential_reflect')
    gd = deblurring.GaussianDiffusion(_Net(), device_of_kernel='cpu', sampling_routine=routine, **kw)
    D = SO.deblur_D(DO.DeblurOracle(net, **kw))
    out.append(('deblurring', gd, lambda x, s, K: gd.sample(batch_size=2, img=x, t=s, steps=K)[2], lambda x, s: gd._degrade_to(x, s),
                SO.cold_update(D, routine), D, {}))
    gr = resolution.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', channels=3, timesteps=6,
                                      resolution_routine='Incremental', sampling_routine=routine)
    D = SO.resolution_D(RO.ResolutionOracle(net, image_size=16, channels=3, timesteps=6, resolution_routine='Incremental'))
    out.append(('resolution', gr, lambda x, s, K: gr.sample(batch_size=2, img=x, t=s, steps=K)[2], lambda x, s: gr._apply_op(x, s - 1),
                SO.cold_update(D, routine), D, {}))
    kw = dict(image_size=16, channels=3, timesteps=8, kernel_std=0.1, initial_mask=11, fade_routine='Random_Incremental')
    gf = defading.GaussianDiffusion(_Net(), device_of_kernel='cpu', sampling_routine=routine, **kw)
    offs = (torch.tensor([3, 16]), torch.tensor([9, 0]))
    D = SO.defading_D(FO.DefadeOracle(net, **kw), *offs)
    out.append(('defading', gf, lambda x, s, K: gf.sample(batch_size=2, faded_recon_sample=x, t=s, _offsets=offs, steps=K)[2],
                lambda x, s: gf._fade(x, s - 1, *offs), SO.cold_update(D, routine), D, {'_offsets': offs}))
    gs = snowification.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', channels=3, timesteps=6,
                                         forward_process_type='Decolorization', sampling_routine=routine)
    fp = NO.DecolorFP(gs.forward_process.factors)
    fp.w = [w.double() for w in fp.w]
    D = SO.snow_D(fp)
    out.append(('snowification', gs, lambda x, s, K: gs.sample(batch_size=2, img=x, t=s, steps=K)['recon'],
                lambda x, s: gs._degrade(x, torch.full((x.shape[0],), s, dtype=torch.long), -1), SO.snow_update(D, routine), D, {}))
    return out


@pytest.mark.parametrize('routine', ['default', 'x0_step_down'])
def test_restore_at_weight_zero_is_sample_bit_for_bit(emulated, routine):
    x = _image()
    for name, gd, sample, Ds, _, _, kw in _packages(routine):
        T = gd.num_timesteps
        for s, K in ((T, None), (T, 3), (T - 2, 1), (3, 3)):
            y = Ds(x, s)
            assert torch.equal(gd.restore(y, s, weight=0.0, steps=K, **kw), sample(x, s, K)), (name, s, K)


@pytest.mark.parametrize('routine', ['default', 'x0_step_down'])
def test_restore_matches_the_float64_restatement(emulated, routine):
    x = _image(seed=1)
    for name, gd, sample, Ds, update, D64, kw in _packages(routine):
        T = gd.num_timesteps
        params = list(gd.parameters()) + list(getattr(gd, 'denoise_fn', getattr(gd, 'defade_fn', None)).parameters())
        for s, K, w in ((T, 1, 0.5), (T, 3, 0.2), (T - 1, T - 1, 0.05)):
            y = Ds(x, s)
            got = gd.restore(y, s, weight=w, steps=K, **kw)
            y64 = y.double()
            ref = GO.guided_reverse(net, y64, s, K, update, lambda a: D64(a, s), w, 2)
            err = ((got.double() - ref).norm() / ref.norm()).item()
            assert err < 1e-5, (name, s, K, err)
            bad = GO.guided_reverse(net, y64, s, K, update, lambda a: D64(a, s), w, 2, guide_on='x0')
            assert ((got.double() - bad).norm() / ref.norm()).item() > 100 * max(err, 1e-7), name
            unguided = GO.guided_reverse(net, y64, s, K, update, lambda a: D64(a, s), 0.0, 2)
            assert ((got.double() - unguided).norm() / ref.norm()).item() > 100 * max(err, 1e-7), name
        assert all(p.grad is None for p in params), name


def test_restore_freezes_and_restores_parameters(emulated):
    from cold_diffusion_models_b200 import deblurring
    n = _Net()
    gd = deblurring.GaussianDiffusion(n, image_size=16, device_of_kernel='cpu', channels=3, timesteps=4, kernel_std=0.3,
                                      kernel_size=5, sampling_routine='x0_step_down')
    y = gd._degrade_to(_image(), 4).requires_grad_()
    seen = []
    orig = n.forward

    def spy(x, t):
        seen.append(n.scale.requires_grad)
        return orig(x, t)
    n.forward = spy
    gd.restore(y, 4, weight=0.3, steps=2)
    assert seen == [False, False] and n.scale.requires_grad and n.scale.grad is None and y.grad is None
    n.scale.requires_grad_(False)
    gd.restore(y, 4, weight=0.3, steps=2)
    assert not n.scale.requires_grad
    n.scale.requires_grad_(True)
    seen.clear()

    def boom(x, t):                     # the second step raises
        if len(seen) == 1:
            raise RuntimeError('network failed')
        seen.append(n.scale.requires_grad)
        return orig(x, t)
    n.forward = boom
    with pytest.raises(RuntimeError, match='network failed'):
        gd.restore(y, 4, weight=0.3, steps=4)
    assert n.scale.requires_grad and n.scale.grad is None and y.grad is None


def test_restore_refusals(emulated):
    from cold_diffusion_models_b200 import deblurring, resolution, defading, snowification
    y = _image()
    mk = lambda **k: deblurring.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', channels=3, timesteps=6,
                                                 kernel_std=0.3, kernel_size=5, **k)
    cases = [
        (mk(discrete=True), 'discrete'),
        (mk(blur_routine='Individual_Incremental'), 'Individual_Incremental'),
        (mk(sampling_routine='ddim'), 'ddim'),
        (mk(train_routine='Step'), 'Step'),
        (resolution.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', timesteps=4, sampling_routine='other'), 'other'),
        (resolution.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', timesteps=4, train_routine='Step'), 'Step'),
        (defading.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', timesteps=4, discrete=True), 'discrete'),
        (defading.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', timesteps=4, sampling_routine='other'), 'other'),
        (snowification.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', timesteps=4, forward_process_type='Snow'),
         'snow'),
        (snowification.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', timesteps=4, to_lab=True), 'Lab'),
        (snowification.GaussianDiffusion(_Net(), image_size=16, device_of_kernel='cpu', timesteps=4, train_routine='Step_Gradient'),
         'Step_Gradient'),
    ]
    for gd, what in cases:
        with pytest.raises(ValueError, match=what):
            gd.restore(y, 2, weight=0.1)
    gd = mk()
    for s in (0, 7, -1, 2.0, None, True):
        with pytest.raises(ValueError, match='level'):
            gd.restore(y, s, weight=0.1)
    for w in (-0.1, float('nan'), float('inf'), None, '1'):
        with pytest.raises(ValueError, match='weight'):
            gd.restore(y, 3, weight=w)
    for K in (0, 4, 2.5):
        with pytest.raises(ValueError, match='steps'):
            gd.restore(y, 3, weight=0.1, steps=K)
    with pytest.raises(ValueError, match='shape'):
        gd.restore(y[:, :2], 3, weight=0.1)
    # the deblurring 'x0_step_down' with Individual_Incremental blur strides, so it restores
    gd = mk(blur_routine='Individual_Incremental', sampling_routine='x0_step_down')
    assert gd.restore(gd._degrade_to(y, 3), 3, weight=0.1, steps=2).shape == y.shape
