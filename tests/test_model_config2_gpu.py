"""The DDPM `Model` (ch = 128, ch_mult = (1, 2, 2, 2), two ResNet blocks per level, attention at 16²) at the benchmarked
config-2 training step -- CIFAR-10 32², micro-batches of 128, dropout 0.1, the L1 loss, the Special_6_routine blur (k = 3,
T = 50) -- and at the 128² shape of the CelebA snowification / decolor drivers, against float64 references computed on the GPU
(oracle/model2_oracle.py, oracle/deblur_oracle.py, plain torch).

At B = 128 the engine dispatches differently from the B = 2 runs of the other Model tests: the conditioning-matrix gradient
dcond . Wc takes the plain `small_gemm_kernel` (split-K only for B * 512 <= 132 * 128), the column sums over B rows take the
vectorised kernel, and the weight-gradient splits and the per-image attention products run other grids.

1. End to end with dropout on (`model.train()`): every `cd_dropout` call of the step is recorded and its (seed, element index)
   mask is rebuilt in the float64 reference, which applies it after swish(norm2(h)) as the Model does.  Parameter gradients of
   one micro-batch, one `Trainer.train_step` (two micro-batches, Adam + EMA) and the gradient at the new weights, the inference
   forward, a 3-step x0_step_down sample, and batch independence.  128² runs at B = 16 (the drivers' train_batch_size).
2. The Model's memory-bound entry points called directly at the arguments a recorded B = 128 step passes (and B = 32 for the
   split-K `cd_small_gemm`), and every convolution descriptor of that step replayed on TF32-rounded operands, together with
   forwards whose Cout is not a multiple of 4 (the 3-channel conv_out) into rows that continue with live columns.
3. Profiler passes at B = 128 and B = 2 show that the kernels checked here are the ones that run.

Every comparison also evaluates its metric on a deliberately wrong reference (a negative control) and asserts that it lands at
least 10x past the bound.  Every bound is at most 3x the value measured on an H100 80GB HBM3 (700 W), which is in the comment
beside it.  Set COLDDIFF_TEST_METRICS=<file> to write all values and controls as JSON.  The file runs in about 50 s on that card;
its peak device memory is 19.2 GiB.  The 128² float64 references run 2 images per chunk and stay well under a minute, so the
128² checks run the drivers' full B = 16 end to end."""
import contextlib
import ctypes as C
import io
import math
import types

import pytest
import torch
import torch.nn.functional as F

import deblur_oracle as DO
import model2_oracle as MO
from test_config3_step_gpu import (Checks, _metrics_file, _free_between_tests, _METRICS, rel, call, ptr, stream, gen,  # noqa: F401
                                   blur_per_image, grad_errors, stats, randn, sentinel, F32)
from test_input_grad_gpu import _record_calls
from test_model_large_gpu import _fp64_time_embedding, _grad_check, _grads, _fp64, NET  # noqa: F401
from test_unet_32_gpu import _spec, _replay, _engine_tensors, _label, tf32_rn  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
T = 50
P_DROP = 0.1
LR = 2e-5
P32 = F32(P_DROP)
KEEP_SCALE = float(torch.tensor(1.0) / (1 - torch.tensor(P_DROP)))      # 1 / (1 - p) as the kernel forms it, in fp32
NBLOCKS = 22                                                            # ResNet blocks per forward


class Checks10(Checks):
    """Checks whose negative controls must land at least 10x past their bounds"""

    def __call__(self, name, value, bound, control=None):
        super().__call__(name, value, bound, control)
        if control is not None and not float(control) > 10 * bound:
            self.fails.append('%s: negative control %.3e is not 10x past the bound %.3e' % (name, control, bound))


# ==========================================================================================================================
# the dropout mask, restated
# ==========================================================================================================================
def _s64(v):
    return v - (1 << 64) if v >= 1 << 63 else v


_GOLD, _MIX1, _MIX2 = (_s64(c) for c in (0x9E3779B97F4A7C15, 0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53))


def _srl(h, n):
    """logical right shift of the uint64 bits held in int64 (torch's >> on int64 is arithmetic)"""
    return (h >> n) & ((1 << (64 - n)) - 1)


def uniform01(seed, idx):
    """tests/abi_emulator.py::_uniform01 in torch int64 arithmetic (products wrap modulo 2^64 as uint64 products do)"""
    h = (idx * _GOLD) ^ _s64(seed)
    h = h ^ _srl(h, 33)
    h = h * _MIX1
    h = h ^ _srl(h, 33)
    h = h * _MIX2
    h = h ^ _srl(h, 33)
    return _srl(h, 40).to(torch.float32) * (1.0 / 16777216.0)


def _keep(seed, B, H, W, Cc, offset=0):
    """the kept elements (NCHW bool) of one cd_dropout call over an NHWC [B][H][W][C] tensor: uniform01(seed, i) >= p at the
    element index i = ((b H + y) W + x) C + c (+ offset: the control of an index off by one)"""
    idx = torch.arange(B * H * W * Cc, device=DEV, dtype=torch.int64) + offset
    return (uniform01(seed, idx) >= P32).view(B, H, W, Cc).permute(0, 3, 1, 2)


_MASKS = {}                 # block name -> kept elements of the images the reference is running


def _resblock_with_dropout(sd, p, x, temb):
    """oracle/model2_oracle.py's resblock with the training-mode dropout between swish(norm2(h)) and conv2 (M2:117-131)"""
    h = F.conv2d(MO.swish(MO.gn(sd, p + '.norm1', x)), sd[p + '.conv1.weight'], sd[p + '.conv1.bias'], padding=1)
    h = h + F.linear(MO.swish(temb), sd[p + '.temb_proj.weight'], sd[p + '.temb_proj.bias'])[:, :, None, None]
    h = MO.swish(MO.gn(sd, p + '.norm2', h))
    if p in _MASKS:
        h = h * _MASKS[p].to(h.dtype) * KEEP_SCALE
    h = F.conv2d(h, sd[p + '.conv2.weight'], sd[p + '.conv2.bias'], padding=1)
    if (p + '.nin_shortcut.weight') in sd:
        x = F.conv2d(x, sd[p + '.nin_shortcut.weight'], sd[p + '.nin_shortcut.bias'])
    return x + h


@pytest.fixture(autouse=True)
def _oracle_dropout(monkeypatch):
    monkeypatch.setattr(MO, 'resblock', _resblock_with_dropout)
    _MASKS.clear()
    yield
    _MASKS.clear()


def _block_order():
    """the ResNet blocks in forward order (model2_oracle.model_forward, model2_train.forward_train)"""
    names = ['down.%d.block.%d' % (lv, ib) for lv in range(4) for ib in range(2)] + ['mid.block_1', 'mid.block_2']
    return names + ['up.%d.block.%d' % (lv, ib) for lv in reversed(range(4)) for ib in range(3)]


def _block_shape(m, name, S):
    lv = 3 if name.startswith('mid') else int(name.split('.')[1])
    return S >> lv, m.get_submodule(name).out_channels


def _v(a):
    return getattr(a, 'value', a)


def _dropout_calls(calls):
    """(npix, C, p, seed) of every cd_dropout call, in launch order"""
    return [(_v(a[2]), _v(a[3]), _v(a[4]), _v(a[5])) for n, a in calls if n == 'cd_dropout']


def _check_dropout_calls(ck, m, S, B, drops, tag):
    """forward calls map onto the ResNet blocks in forward order with the blocks' (npix, C); the backward replays each
    block's mask in reverse order.  -> the forward seeds"""
    ck.require('%s: %d cd_dropout calls (%d)' % (tag, 2 * NBLOCKS, len(drops)), len(drops) == 2 * NBLOCKS)
    fwd, bwd = drops[:NBLOCKS], drops[NBLOCKS:]
    for (npix, Cc, p, _), name in zip(fwd, _block_order()):
        res, co = _block_shape(m, name, S)
        ck.require('%s: dropout of %s is (npix %d, C %d, p %g), not (%d, %d, %g)' % (tag, name, npix, Cc, p, B * res * res, co, P32),
                   (npix, Cc, p) == (B * res * res, co, P32))
    ck.require('%s: the backward replays the forward masks in reverse order' % tag, bwd == fwd[::-1])
    return [d[3] for d in fwd]


def _keeps(m, S, B, seeds, shift=0):
    """block name -> kept elements; shift = 1: every block gets the mask of the next block's call (the control)"""
    out = {}
    for i, name in enumerate(_block_order()):
        res, co = _block_shape(m, name, S)
        out[name] = _keep(seeds[(i + shift) % NBLOCKS], B, res, res, co)
    return out


# ==========================================================================================================================
# model, diffusion, references
# ==========================================================================================================================
CASES = [('cifar32-b128', 32, 128, 8), ('celeba128-b16', 128, 16, 2)]          # (name, S, B, images per fp64 chunk)


def _model(S, seed):
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(seed)
    return cdm.Model(resolution=S, in_channels=3, out_ch=3, dropout=P_DROP, **NET).to(DEV)


def _gd(m, S):
    import cold_diffusion_models_b200 as cdm
    return cdm.GaussianDiffusion(m, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1', kernel_std=0.1,
                                 kernel_size=3, blur_routine='Special_6_routine', train_routine='Final',
                                 sampling_routine='x0_step_down').to(DEV)


def _blur(S, denoise_fn=None, **kw):
    kw.update(image_size=S, channels=3, timesteps=T, kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine')
    o = DO.DeblurOracle(denoise_fn, **kw)
    o.kernels2d = [k.double().cuda() for k in o.kernels2d]
    return o


def _batch(B, S, seed):
    x = torch.rand(B, 3, S, S, generator=gen(seed), device=DEV) * 2 - 1
    t = torch.randint(0, T, (B,), generator=gen(seed + 1), device=DEV)
    t[0], t[1] = 0, T - 1
    return x, t


def _ref(sd, xt64, t, gy, keeps, chunk):
    """float64 Model output with the given dropout masks (None: no dropout) and, when gy is given, the VJP gy . dY/dparams,
    `chunk` images at a time -> (gradients by name or None, output)"""
    leaves = {k: v.detach().to(DEV, F64).requires_grad_(gy is not None) for k, v in sd.items()}
    names = list(leaves)
    acc = {k: torch.zeros_like(v) for k, v in leaves.items()} if gy is not None else None
    ys = []
    for c in range(0, xt64.shape[0], chunk):
        _MASKS.clear()
        if keeps is not None:
            _MASKS.update({k: v[c:c + chunk] for k, v in keeps.items()})
        with torch.set_grad_enabled(gy is not None):
            y = MO.model_forward(leaves, xt64[c:c + chunk], t[c:c + chunk], ch=NET['ch'], num_resolutions=4, num_res_blocks=2)
        if gy is not None:
            for k, g in zip(names, torch.autograd.grad(y, [leaves[k] for k in names], gy[c:c + chunk])):
                acc[k] += g
        ys.append(y.detach())
        del y
    _MASKS.clear()
    return acc, torch.cat(ys)


def _engine_micro_batch(m, gd, x, t, seed):
    """forward + backward of one micro-batch under the host seed `seed`, then the same forward again (same seeds, same
    masks) for its output -> (gradients, output, loss, dropout calls of the step, of the repeated forward)"""
    m.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    with _record_calls() as calls:
        loss = gd.p_losses(x, t)
        loss.backward()
        torch.cuda.synchronize()
    eg = _grads(m)
    m.zero_grad(set_to_none=True)
    xt = gd.q_sample(x, t)
    torch.manual_seed(seed)
    with _record_calls() as again:
        y = m(xt, t).detach()
    return eg, y, loss.item(), _dropout_calls(calls), _dropout_calls(again)


def _gy(y, x):
    """upstream gradient of the L1 loss mean |x0 - y| at the engine's own output"""
    return torch.sign(y.double() - x.double()) / y.numel()


# ==========================================================================================================================
# 1 + 3. end to end
# ==========================================================================================================================
def test_dropout_mask_statement_matches_cd_dropout():
    """cd_dropout on ones (rows padded to ld = C + 4) over 2^25 + 2048 elements keeps exactly the elements uniform01 keeps,
    scaled by fp32 1 / (1 - p); level 0 of a B = 128 32² step has 2^24 elements and of a B = 16 128² step 2^25.  Control: the
    mask of the index off by one."""
    ck = Checks10('dropout statement')
    Cc, ld = 128, 132
    npix = (1 << 25) // Cc + 16
    seed = 0x5DEECE66D1234567 & ((1 << 62) - 1)
    x = torch.ones(npix, ld, device=DEV)
    y = sentinel(npix, ld)
    call('cd_dropout', ptr(x), ld, C.c_int64(npix), Cc, C.c_float(P_DROP), C.c_uint64(seed), ptr(y), ld, stream())
    torch.cuda.synchronize()
    keep = _keep(seed, 1, npix, 1, Cc).permute(0, 2, 3, 1).reshape(npix, Cc)
    got = y[:, :Cc]
    ck.require('kept elements equal 1 / (1 - p) exactly', bool((got[keep] == KEEP_SCALE).all()))
    ck.require('dropped elements are 0', bool((got[~keep] == 0).all()))
    ck.require('row padding untouched', bool((y[:, Cc:] == 7.0).all()))
    for lo in (0, (1 << 24) - 4096, (1 << 25) - 4096, npix * Cc - 4096):     # the statement at, below and above 2^24, 2^25
        k = keep.reshape(-1)[lo:lo + 8192]
        ck.require('mask at indices %d..%d' % (lo, lo + 8191), bool(torch.equal(got.reshape(-1)[lo:lo + 8192] != 0, k)))
    # control: the statement at the index off by one disagrees with the kernel on about 2 p (1 - p) = 18 % of the elements
    shifted = _keep(seed, 1, npix, 1, Cc, offset=1).permute(0, 2, 3, 1).reshape(npix, Cc)
    ctrl = (shifted != (got != 0)).double().mean().item()
    _METRICS['dropout statement::kept fraction'] = keep.double().mean().item()
    _METRICS['dropout statement::control mismatched fraction'] = ctrl
    ck.require('control: the index off by one mismatches %.3f of the elements' % ctrl, ctrl > 0.1)
    ck.done()


# bounds per case, each at most 3x the value measured on the H100 (in the comment below it)
BOUNDS = {
    'cifar32-b128': dict(xt=3.5e-7, sxt=3e-7, out=3.8e-3, loss=2.9e-5, tloss=2.7e-5, flip=4.1e-4, gmed=4.3e-3, gworst=2e-2, adam=8.9e-3, amed=5.8e-3,
                         aworst=1.5e-2, inf=4e-3, direct=3e-3, sample=3.2e-4),
    # measured: x_t 1.18e-7 (the sample's 1.0e-7), output 1.27e-3, L1 loss 9.8e-6 (train_step 9.0e-6), signs 1.37e-4, gradient median 1.44e-3 / worst
    # 6.75e-3, Adam 2.98e-3 (the fp32 rounding of p against lr = 2e-5), after the step 1.94e-3 / 5.05e-3, inference forward
    # 1.34e-3, sample direct 1.01e-3, sample 1.09e-4
    'celeba128-b16': dict(xt=2.3e-7, sxt=3e-7, out=3.8e-3, loss=5e-5, tloss=4.5e-5, flip=5e-4, gmed=8.1e-3, gworst=1.58e-2, adam=8.9e-3, amed=8.8e-3,
                          aworst=1.8e-2, inf=4.2e-3, direct=3.1e-3, sample=3.5e-4),
    # measured: x_t 7.8e-8 (the sample's 1.02e-7), output 1.29e-3, L1 loss 1.68e-5 (train_step 1.52e-5), signs 1.67e-4, gradient median 2.73e-3 / worst
    # 5.28e-3, Adam 2.98e-3, after the step 2.95e-3 / 6.10e-3, inference forward 1.40e-3, sample direct 1.06e-3, sample 1.17e-4
}


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_model_step_with_dropout_against_fp64(case, tmp_path):
    """the parameter gradients of one micro-batch with dropout 0.1 (masks rebuilt from the recorded seeds), the inference
    forward, one Trainer step at the benchmark's hyper-parameters (loss, Adam, EMA copy) and the gradient at the new weights,
    and a 3-step x0_step_down sample of the EMA model, against float64"""
    import cold_diffusion_models_b200 as cdm
    name, S, B, chunk = case
    bd = BOUNDS[name]
    ck = Checks10('model step %s' % name)
    m = _model(S, seed=3)
    m.train()
    gd = _gd(m, S)
    o = _blur(S)
    x, t = _batch(B, S, 40 + S)
    x2, t2 = _batch(B, S, 60 + S)
    xt64 = blur_per_image(o, x.double(), t)
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    # ---- one micro-batch: dropout calls, x_t, output, loss, sign agreement, gradients
    eg, y, loss, drops, again = _engine_micro_batch(m, gd, x, t, seed=21)
    seeds = _check_dropout_calls(ck, m, S, B, drops, 'step')
    ck.require('the repeated forward draws the same masks', again == drops[:NBLOCKS])
    ck('x_t', rel(gd.q_sample(x, t), xt64), bd['xt'],
       rel(gd.q_sample(x, t), blur_per_image(o, x.double(), torch.where(t < T - 1, t + 1, t - 1))))
    gy = _gy(y, x)
    keeps = _keeps(m, S, B, seeds)
    ref, y64 = _ref(sd0, xt64, t, gy, keeps, chunk)
    del keeps
    shifted, y_sh = _ref(sd0, xt64, t, gy, _keeps(m, S, B, seeds, shift=1), chunk)
    nodrop, y_nd = _ref(sd0, xt64, t, gy, None, chunk)
    ck('output', rel(y, y64), bd['out'], rel(y_nd, y64))
    ck('output (control: masks shifted by one block)', rel(y, y64), bd['out'], rel(y_sh, y64))
    lref = (x.double() - y64).abs().mean().item()
    ck('L1 loss', abs(loss - lref) / lref, bd['loss'], abs((x.double() - y_nd).abs().mean().item() - lref) / lref)
    s_eng, s_ref = torch.sign(y.double() - x.double()), torch.sign(y64 - x.double())
    ck('sign(y - x0) differs from fp64 (fraction)', (s_eng != s_ref).double().mean().item(), bd['flip'],
       (torch.sign(y_nd - x.double()) != s_ref).double().mean().item())
    _grad_check(ck, 'grad', eg, ref, nodrop, bd['gmed'], bd['gworst'])
    _grad_check(ck, 'grad (control: masks shifted by one block)', eg, ref, shifted, bd['gmed'], bd['gworst'])
    del eg, ref, shifted, nodrop, y_sh
    # ---- the inference forward (eval mode: no dropout, cd_time_mlp2_fwd's two-launch branch)
    m.eval()
    with torch.no_grad():
        yi = m(gd.q_sample(x, t), t)
    m.train()
    ck('inference forward', rel(yi, y_nd), bd['inf'], rel(yi, y64))
    del y64, y_nd, yi
    # ---- one Trainer step over (x, t) and (x2, t2); what the optimizer read is snapshotted
    with contextlib.redirect_stdout(io.StringIO()):
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=LR, train_num_steps=10 ** 9,
                         gradient_accumulate_every=2, ema_decay=0.995, fp16=False, results_folder=str(tmp_path),
                         dataset='synthetic')
    eng = m.engine
    ts = iter([t, t2])
    gd.forward = lambda d: gd.p_losses(d, next(ts))
    snap, step = {}, tr.opt.step

    def snapshot_step(**kw):
        snap.update(p0=eng.flat_param.clone(), g0=eng.flat_grad.clone(), kw=kw)
        step(**kw)
    tr.opt.step = snapshot_step
    torch.manual_seed(31)
    try:
        with _record_calls() as calls:
            tloss = tr.train_step([x, x2]).item()
            torch.cuda.synchronize()
    finally:
        tr.opt.step = step
        del gd.forward
    drops = _dropout_calls(calls)
    ck.require('train_step: two micro-batches of dropout calls (%d)' % len(drops), len(drops) == 4 * NBLOCKS)
    s1 = _check_dropout_calls(ck, m, S, B, drops[:2 * NBLOCKS], 'train_step mb1')
    s2 = _check_dropout_calls(ck, m, S, B, drops[2 * NBLOCKS:], 'train_step mb2')
    xt64_2 = blur_per_image(o, x2.double(), t2)
    with torch.no_grad():
        l1 = (x.double() - _ref(sd0, xt64, t, None, _keeps(m, S, B, s1), chunk)[1]).abs().mean().item()
        l2 = (x2.double() - _ref(sd0, xt64_2, t2, None, _keeps(m, S, B, s2), chunk)[1]).abs().mean().item()
    tref = (l1 + l2) / 2
    # control: the micro-batch losses summed instead of averaged over gradient_accumulate_every
    ck('train_step loss', abs(tloss - tref) / tref, bd['tloss'], abs(l1 + l2 - tref) / tref)
    # Adam at step 1 in float64 (the kernel's fp32 betas) on the gradient it read: an update of lr sign(g) where g != 0;
    # control: no bias correction
    gs = snap['kw'].get('grad_scale', 1.0)
    p = snap['p0'].double().clone().requires_grad_(True)
    p.grad = snap['g0'].double() * gs
    ta = torch.optim.Adam([p], lr=LR, betas=(F32(0.9), F32(0.999)), eps=1e-8)
    ta.step()
    d_r = p.detach() - snap['p0'].double()
    d_k = eng.flat_param.double() - snap['p0'].double()
    wrong = -LR * 0.1 * p.grad / (0.001 ** 0.5 * p.grad.abs() + 1e-8)
    ck('Adam update (max |err| / lr)', (d_k - d_r).abs().max().item() / LR, bd['adam'], (wrong - d_r).abs().max().item() / LR)
    ck.require('EMA copied the new weights at step 0', bool(torch.equal(tr._ema_unet.engine.flat_param, eng.flat_param)))
    del p, d_r, d_k, wrong, snap, ta
    # ---- gradient at the new weights; control: the reference at the old weights
    sd1 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    eg, y, _, drops, again = _engine_micro_batch(m, gd, x, t, seed=51)
    tr.opt.zero_grad()
    seeds = _check_dropout_calls(ck, m, S, B, drops, 'after the step')
    keeps = _keeps(m, S, B, seeds)
    gy = _gy(y, x)
    ref_new, _ = _ref(sd1, xt64, t, gy, keeps, chunk)
    ref_old, _ = _ref(sd0, xt64, t, gy, keeps, chunk)
    del keeps
    _grad_check(ck, 'grad after the step', eg, ref_new, ref_old, bd['amed'], bd['aworst'])
    del eg, ref_new, ref_old
    # ---- a 3-step x0_step_down sample of the EMA model (eager, as the benchmark samples)
    ema = tr.ema_model
    with torch.no_grad():
        xt, dr, img = ema.sample(batch_size=B, img=x, t=3)
    torch.cuda.synchronize()
    os_ = _blur(S, denoise_fn=_fp64(ema.denoise_fn.state_dict()), sampling_routine='x0_step_down')
    with torch.no_grad():
        parts = [os_.sample(min(chunk, B - c), x[c:c + chunk].double(), t=3) for c in range(0, B, chunk)]
    r = [torch.cat([q[j] for q in parts]) for j in range(3)]
    ck('sample x_t', rel(xt, r[0]), bd['sxt'], rel(xt, blur_per_image(o, x.double(), torch.full((B,), 1))))
    ck('sample direct reconstruction', rel(dr, r[1]), bd['direct'], rel(dr.roll(1, 0), r[1]))
    ck('sample', rel(img, r[2]), bd['sample'], rel(xt, r[2]))
    ck.done()


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_model_batch_independence(case):
    """row k of a full batch against the same image run alone (other grids, splits and tiles; the same arithmetic per image):
    the forward output and the gradient of |y_k|^2, without dropout.  Controls: another row, another image's gradient."""
    name, S, B, _ = case
    ck = Checks10('batch independence %s' % name)
    m = _model(S, seed=8)
    m.eval()                                  # autograd still takes the training path; eval mode turns the dropout off
    x, t = _batch(B, S, 90 + S)
    k = B - 5
    m.zero_grad(set_to_none=True)
    y = m(x, t)
    (y[k] ** 2).mean().backward()
    whole = _grads(m)
    m.zero_grad(set_to_none=True)
    y1 = m(x[k:k + 1], t[k:k + 1])
    (y1[0] ** 2).mean().backward()
    one = _grads(m)
    m.zero_grad(set_to_none=True)
    y2 = m(x[k + 1:k + 2], t[k + 1:k + 2])
    (y2[0] ** 2).mean().backward()
    other = _grads(m)
    m.zero_grad(set_to_none=True)
    # measured forward 7.7e-4 / 7.5e-4 (cifar32-b128 / celeba128-b16), gradient median 1.65e-3 / 1.39e-3, worst 5.2e-3 / 3.5e-3
    bf, bmed, bworst = {'cifar32-b128': (2.3e-3, 4.9e-3, 1.5e-2), 'celeba128-b16': (2.2e-3, 4.1e-3, 1e-2)}[name]
    ck('forward row %d' % k, rel(y[k:k + 1].detach(), y1.detach()), bf, rel(y[k + 1:k + 2].detach(), y1.detach()))
    _grad_check(ck, 'grad', one, whole, other, bmed, bworst)
    ck.done()


# ==========================================================================================================================
# 2. the entry points at the arguments of a recorded step
# ==========================================================================================================================
# positions of the scalar arguments, and of the pointers whose presence matters, in each entry point's argument list
_SCALARS = {
    'cd_softmax_rows': ((1, 2, 3, 4), ()), 'cd_softmax_bwd_rows': ((2, 3, 4, 5), ()),
    'cd_transpose_batched': ((1, 2, 3, 4), ()), 'cd_upsample_nearest2x': ((1, 2, 3, 4, 5, 7), ()),
    'cd_upsample_nearest2x_bwd': ((1, 2, 3, 4, 5, 7), ()), 'cd_timestep_embedding': ((1, 2), ()),
    'cd_linear_fwd': ((1, 4, 5), ()), 'cd_swish': ((2,), (0, 4)), 'cd_small_gemm': ((1, 2, 4, 5, 7, 8, 9, 10, 11), ()),
    'cd_colsum': ((1, 2, 3), ()), 'cd_groupnorm_fwd': ((1, 2, 3, 4, 5, 7, 10, 11, 13), (6,)),
    'cd_groupnorm_bwd': ((1, 2, 3, 4, 5, 7, 10, 11, 13, 15, 19), (6, 16, 18)),
}


def _model_spans(m):
    return _engine_tensors(types.SimpleNamespace(_bufs=m._bufs, _packed=m._packed, flat_grad=m.engine.flat_grad,
                                                 flat_param=m.engine.flat_param))


@pytest.fixture(scope='module')
def rec():
    """the scalar arguments of the Model's own entry points in a 32² training step (dropout on) at B = 128 and B = 32, and
    the deduplicated cd_conv_fwd / cd_conv_wgrad descriptors of the B = 128 step"""
    from cold_diffusion_models_b200 import ops
    m = _model(32, seed=11)
    m.train()
    gd = _gd(m, 32)
    out = {}
    for B in (128, 32):
        x, t = _batch(B, 32, 500 + B)
        m.zero_grad(set_to_none=True)
        torch.manual_seed(B)
        with _record_calls() as calls:
            gd.p_losses(x, t).backward()
            torch.cuda.synchronize()
        args = {}
        for name, a in calls:
            if name in _SCALARS:
                sc, nz = _SCALARS[name]
                key = tuple(_v(a[i]) for i in sc) + tuple(bool(_v(a[i])) for i in nz)
                args.setdefault(name, [])
                if key not in args[name]:
                    args[name].append(key)
        convs = {}
        if B == 128:
            spans = _model_spans(m)
            for name, a in calls:
                if name == 'cd_conv_fwd':
                    sp = _spec('fwd', a[0]._obj, a[1], spans)
                elif name == 'cd_conv_wgrad':
                    sp = _spec('wgrad', a[0]._obj, a[5], spans, dout=(a[1].value, a[2]), db=bool(a[4].value))
                else:
                    continue
                convs.setdefault(repr(sorted(sp.items())), sp)
        out[B] = dict(args=args, convs=list(convs.values()), sumC=m._sumC)
    out['impl'] = ops.CONV_TC
    yield out
    del m, gd


def test_softmax_rows_against_fp64(rec):
    """cd_softmax_rows and cd_softmax_bwd_rows at every (ld, rows, n, scale) of the B = 128 step, on scores of the size the
    network makes and on scores shifted by +2000 (scaled logits far above fp32 expf's overflow at ~88).  Controls: the scale 1
    instead of c^-1/2, and every row's reference taken from the next row."""
    ck = Checks10('softmax')
    fwd, bwd = rec[128]['args']['cd_softmax_rows'], rec[128]['args']['cd_softmax_bwd_rows']
    ck.require('the 16² attention (rows 128 * 256, n 256, c^-1/2 = 1/16) is among the calls', (256, 128 * 256, 256, 1 / 16) in fwd)
    ck.require('forward and backward take the same arguments', sorted(fwd) == sorted(bwd))
    g = gen(800)
    for ld, rows, n, scale in fwd:
        for shift in (0.0, 2000.0):
            key = 'rows %d n %d shift %g' % (rows, n, shift)
            z = randn(rows, ld, g=g, scale=2.0 / scale) + shift
            s = z.clone()
            call('cd_softmax_rows', ptr(s), ld, C.c_int64(rows), n, C.c_float(scale), stream())
            ref = torch.softmax(z[:, :n].double() * scale, dim=1)
            ck(key + ' forward', rel(s[:, :n], ref), 1.9e-7,           # measured <= 6.4e-8
               rel(torch.softmax(z[:, :n].double(), dim=1), ref))
            ck(key + ' forward (control: next row)', rel(s[:, :n], ref), 1.9e-7, rel(s[:, :n].roll(1, 0), ref))
            ck.require(key + ': padding untouched', bool(torch.equal(s[:, n:], z[:, n:])))
            ds0 = randn(rows, ld, g=g)
            ds = ds0.clone()
            call('cd_softmax_bwd_rows', ptr(s), ptr(ds), ld, C.c_int64(rows), n, C.c_float(scale), stream())
            s64, d64 = s[:, :n].double(), ds0[:, :n].double()
            dref = s64 * (d64 - (d64 * s64).sum(1, keepdim=True)) * scale
            ck(key + ' backward', rel(ds[:, :n], dref), 2.1e-7,        # measured <= 7.2e-8
               rel(dref / scale, dref) if scale != 1 else rel(dref * 2, dref))
            ck(key + ' backward (control: next row)', rel(ds[:, :n], dref), 2.1e-7, rel(ds[:, :n].roll(1, 0), dref))
            del z, s, ds0, ds
    ck.done()


def test_transpose_and_upsample(rec):
    """cd_transpose_batched (bit-exact) and cd_upsample_nearest2x (bit-exact) at the B = 128 step's arguments and from a
    concat-buffer slice (ld = 2C, channel offset C); cd_upsample_nearest2x_bwd against the float64 sum of the four children"""
    ck = Checks10('transpose and upsample')
    a = rec[128]['args']
    g = gen(810)
    ck.require('transpose of the 16² attention (B 128, 256 x 256) among the calls', (256, 128, 256, 256) in a['cd_transpose_batched'])
    for ld, B, R, Cc in a['cd_transpose_batched']:
        src = randn(B, R, ld, g=g)
        dst = sentinel(B, Cc, R)
        call('cd_transpose_batched', ptr(src), ld, B, R, Cc, ptr(dst), stream())
        ck.require('transpose B%d %dx%d exact' % (B, R, Cc), bool(torch.equal(dst, src[..., :Cc].transpose(1, 2))))
    ups = a['cd_upsample_nearest2x']
    ck.require('upsamples 4 -> 8, 8 -> 16, 16 -> 32 recorded', sorted({u[2] for u in ups}) == [4, 8, 16])
    for x_ld, B, H, W, Cc, y_ld in ups + [(2 * u[4], u[1], u[2], u[3], u[4], u[5]) for u in ups]:
        c0 = x_ld - Cc                              # 0 at the recorded ld; the second channel slice of a concat buffer above
        x = randn(B, H, W, x_ld, g=g)
        y = sentinel(B, 2 * H, 2 * W, y_ld)
        call('cd_upsample_nearest2x', C.c_void_p(x.data_ptr() + 4 * c0), x_ld, B, H, W, Cc, ptr(y), y_ld, stream())
        ref = x[..., c0:c0 + Cc].repeat_interleave(2, 1).repeat_interleave(2, 2)
        key = 'upsample %dx%d C%d x_ld %d' % (H, W, Cc, x_ld)
        ck.require(key + ' exact', bool(torch.equal(y[..., :Cc], ref)) and bool((y[..., Cc:] == 7.0).all()))
    for dy_ld, B, H, W, Cc, dx_ld in a['cd_upsample_nearest2x_bwd']:
        for wide in (0, 1):
            dld = dx_ld * (1 + wide)
            dy = randn(B, 2 * H, 2 * W, dy_ld, g=g)
            dx = sentinel(B, H, W, dld)
            call('cd_upsample_nearest2x_bwd', ptr(dy), dy_ld, B, H, W, Cc, ptr(dx), dld, stream())
            d64 = dy[..., :Cc].double()
            ref = d64[:, 0::2, 0::2] + d64[:, 0::2, 1::2] + d64[:, 1::2, 0::2] + d64[:, 1::2, 1::2]
            key = 'upsample_bwd %dx%d C%d dx_ld %d' % (H, W, Cc, dld)
            ck(key, rel(dx[..., :Cc], ref), 1.2e-7,                    # measured <= 4.1e-8
               rel(ref - d64[:, 1::2, 1::2], ref))
            ck.require(key + ': padding untouched', bool((dx[..., Cc:] == 7.0).all()))
    ck.done()


def test_time_path_entry_points_against_fp64(rec):
    """cd_timestep_embedding (t in [0, 50) and [0, 1000)), cd_linear_fwd at every recorded (K, M, N), cd_swish forward and
    backward, cd_colsum over B rows (recorded) and over B * H * W rows (the bias gradient of a frozen convolution weight)"""
    ck = Checks10('time path')
    a = rec[128]['args']
    g = gen(820)
    (B, dim), = a['cd_timestep_embedding']
    ck.require('timestep embedding at (B, dim) = (128, 128)', (B, dim) == (128, 128))
    for hi in (T, 1000):
        t = torch.randint(0, hi, (B,), generator=g, device=DEV)
        t[0], t[1] = 0, hi - 1
        emb = sentinel(B, dim)
        call('cd_timestep_embedding', ptr(t), B, dim, ptr(emb), stream())
        half = dim // 2
        f = torch.exp(torch.arange(half, dtype=F64, device=DEV) * -(math.log(10000) / (half - 1)))
        ref = torch.cat([torch.sin(t.double()[:, None] * f), torch.cos(t.double()[:, None] * f)], 1)
        wrong = torch.cat([torch.sin((t + 1).double()[:, None] * f), torch.cos((t + 1).double()[:, None] * f)], 1)
        # max abs error, measured 4.3e-6 (t < 50) and 8.7e-5 (t < 1000: the fp32 argument t * f carries t's magnitude)
        ck('timestep embedding t < %d' % hi, (emb.double() - ref).abs().max().item(), {T: 1.2e-5, 1000: 2.6e-4}[hi],
           (wrong - ref).abs().max().item())
    lin = a['cd_linear_fwd']
    sumC = rec[128]['sumC']
    ck.require('linear layers (128, 512), (512, 512), (512, sumC)', sorted(lin) == sorted([(128, B, 512), (512, B, 512), (512, B, sumC)]))
    for K, M, N in lin:
        x, w, b = randn(M, K, g=g), randn(N, K, g=g, scale=K ** -0.5), randn(N, g=g)
        y = sentinel(M, N)
        call('cd_linear_fwd', ptr(x), K, ptr(w), ptr(b), M, N, ptr(y), stream())
        ref = x.double() @ w.double().t() + b.double()
        ks = K - K // 8
        ck('linear K%d N%d' % (K, N), rel(y, ref), 2.2e-7,             # measured <= 7.4e-8
           rel(x.double()[:, :ks] @ w.double()[:, :ks].t() + b.double(), ref))
    for n, with_dy, with_act in a['cd_swish']:
        pre = randn(n, g=g, scale=3.0)
        dy = randn(n, g=g)
        y, act = sentinel(n), sentinel(n)
        call('cd_swish', ptr(dy) if with_dy else C.c_void_p(0), ptr(pre), C.c_int64(n), ptr(y) if with_dy else C.c_void_p(0),
             ptr(act) if with_act else C.c_void_p(0), stream())
        p64 = pre.double().requires_grad_(True)
        a64 = p64 * torch.sigmoid(p64)
        gr, = torch.autograd.grad(a64, p64, dy.double())
        if with_act:
            ck('swish n%d' % n, rel(act, a64.detach()), 1.35e-7,        # measured 4.6e-8
               rel(p64.detach() * torch.sigmoid(1.702 * p64.detach()), a64.detach()))
        if with_dy:
            ck('swish backward n%d' % n, rel(y, gr), 2.8e-7,            # measured 9.5e-8
               rel(dy.double() * torch.sigmoid(p64.detach()), gr))
        ck.require('swish n%d: unrequested outputs untouched' % n,
                   bool((act == 7.0).all()) != with_act and bool((y == 7.0).all()) != with_dy)
    cols = a['cd_colsum']
    ck.require('column sums over B rows recorded', any(r == B for _, r, _ in cols))
    # bound by rows: measured <= 8.1e-8 over B rows, 2.9e-7 over 128 * 256 rows, 4.6e-7 over 128 * 1024 rows
    cbound = {B: 2.4e-7, B * 256: 8.6e-7, B * 1024: 1.37e-6}
    for ld, rows, Cc in cols + [(128, B * 1024, 128), (256, B * 256, 256), (384, B * 1024, 128)]:
        x = randn(rows, ld, g=g)
        out0 = randn(Cc + 8, g=g)
        out = out0.clone()
        call('cd_colsum', ptr(x), ld, C.c_int64(rows), Cc, ptr(out), stream())
        ref = out0[:Cc].double() + x[:, :Cc].double().sum(0)
        ck('colsum rows %d C%d ld %d' % (rows, Cc, ld), rel(out[:Cc], ref), cbound[rows],
           rel(out0[:Cc].double() + x[:-1, :Cc].double().sum(0), ref))
        ck.require('colsum rows %d C%d: beyond C untouched' % (rows, Cc), bool(torch.equal(out[Cc:], out0[Cc:])))
    ck.done()


def test_small_gemm_of_the_time_backward(rec):
    """cd_small_gemm at every (lda, transA, ldb, transB, ldc, M, N, K, accumulate) that the time backward issues at B = 128
    (small_gemm_kernel for every product) and at B = 32 (split-K for dcond . Wc and dtemb . W1).  Controls: the last K/8
    of the contraction missing, and (accumulating calls) the accumulation dropped."""
    ck = Checks10('small_gemm')
    g = gen(830)
    cases = [(B, k) for B in (128, 32) for k in rec[B]['args']['cd_small_gemm']]
    sumC = rec[128]['sumC']
    ck.require('dcond . Wc recorded at B = 128 and B = 32',
               (sumC, 0, 512, 0, 512, 128, 512, sumC, 0) in rec[128]['args']['cd_small_gemm'] and
               (sumC, 0, 512, 0, 512, 32, 512, sumC, 0) in rec[32]['args']['cd_small_gemm'])
    # bound by (B, K): measured 1.27e-6 (128, 4992: small_gemm_kernel's 4992-long loop), 5.6e-7 (32, 4992: split-K), 4.0e-7 /
    # 1.9e-7 (128 / 32, 512), 2.06e-7 (128, 128) and 1.04e-7 (32, 32)
    gbound = {(128, 4992): 3.8e-6, (32, 4992): 1.7e-6, (128, 512): 1.2e-6, (32, 512): 5.6e-7, (128, 128): 6.2e-7, (32, 32): 3.1e-7}
    ck.require('sumC = 4992', sumC == 4992)
    for B, (lda, ta, ldb, tb, ldc, M, N, K, acc) in cases:
        Ab = randn(K if ta else M, lda, g=g)
        Bb = randn(N if tb else K, ldb, g=g)
        A = (Ab[:, :M].t() if ta else Ab[:, :K]).double()
        Bm = (Bb[:, :K].t() if tb else Bb[:, :N]).double()
        c0 = randn(M, ldc, g=g)
        cm = c0.clone()
        call('cd_small_gemm', ptr(Ab), lda, ta, ptr(Bb), ldb, tb, ptr(cm), ldc, M, N, K, acc, stream())
        base = c0[:, :N].double() if acc else 0
        ref = A @ Bm + base
        ks = K - max(1, K // 8)
        key = 'B%d ta%d tb%d M%d N%d K%d acc%d' % (B, ta, tb, M, N, K, acc)
        ck(key, rel(cm[:, :N], ref), gbound[B, K],
           rel(A[:, :ks] @ Bm[:ks] + base, ref))
        if acc:
            ck(key + ' (control: accumulation dropped)', rel(cm[:, :N], ref), gbound[B, K], rel(A @ Bm, ref))
        ck.require(key + ': columns beyond N untouched', bool(torch.equal(cm[:, N:], c0[:, N:])))
    ck.done()


def _gn64(x, gamma, beta, swish, B, HW, Cc, groups, eps):
    z = F.group_norm(x.view(B, HW, Cc).permute(0, 2, 1), groups, gamma, beta, eps=eps).permute(0, 2, 1)
    return z * torch.sigmoid(z) if swish else z


def test_groupnorm_at_the_concat_widths(rec):
    """cd_groupnorm_fwd / cd_groupnorm_bwd at every recorded call of the B = 128 step with C = 384 or 512 (the up path's
    concat buffers: norm1 of the up blocks, which takes no conditioning), dgamma / dbeta accumulating.  Controls: every image's
    reference taken from the next image."""
    ck = Checks10('groupnorm concat widths')
    g = gen(840)
    fw = [k for k in rec[128]['args']['cd_groupnorm_fwd'] if k[3] in (384, 512)]
    bw = [k for k in rec[128]['args']['cd_groupnorm_bwd'] if k[3] in (384, 512)]
    ck.require('C = 384 and 512 recorded (forward and backward)', {k[3] for k in fw} == {384, 512} == {k[3] for k in bw})
    ck.require('no conditioning at the concat widths', not any(k[-1] for k in fw) and not any(k[-3] or k[-1] for k in bw))
    for x_ld, B, HW, Cc, groups, cond_ld, eps, swish, y_ld, _ in fw:
        x = randn(B * HW, x_ld, g=g, scale=1.5) + 0.5
        gamma, beta = 1 + randn(Cc, g=g, scale=0.2), randn(Cc, g=g, scale=0.1)
        y = sentinel(B * HW, y_ld)
        call('cd_groupnorm_fwd', ptr(x), x_ld, B, C.c_int64(HW), Cc, groups, C.c_void_p(0), cond_ld, ptr(gamma), ptr(beta),
             C.c_float(eps), swish, ptr(y), y_ld, stream())
        ref = _gn64(x[:, :Cc].double(), gamma.double(), beta.double(), swish, B, HW, Cc, groups, eps)
        yv = y[:, :Cc].view(B, HW, Cc)
        ck('fwd %dpx C%d' % (HW, Cc), rel(yv, ref), 2.7e-7, rel(yv, ref.roll(1, 0)))  # measured <= 9.1e-8
        ck.require('fwd %dpx C%d: padding untouched' % (HW, Cc), bool((y[:, Cc:] == 7.0).all()))
    for x_ld, B, HW, Cc, groups, cond_ld, eps, swish, dy_ld, dx_ld, dcond_ld, _, has_params, _ in bw:
        x = randn(B * HW, x_ld, g=g, scale=1.5) + 0.5
        gamma, beta = 1 + randn(Cc, g=g, scale=0.2), randn(Cc, g=g, scale=0.1)
        dy = randn(B * HW, dy_ld, g=g)
        dx = sentinel(B * HW, dx_ld)
        dg0, db0 = randn(Cc, g=g), randn(Cc, g=g)
        dg, db = dg0.clone(), db0.clone()
        call('cd_groupnorm_bwd', ptr(x), x_ld, B, C.c_int64(HW), Cc, groups, C.c_void_p(0), cond_ld, ptr(gamma), ptr(beta),
             C.c_float(eps), swish, ptr(dy), dy_ld, ptr(dx), dx_ld, ptr(dg) if has_params else C.c_void_p(0),
             ptr(db) if has_params else C.c_void_p(0), C.c_void_p(0), dcond_ld, stream())
        x64 = x[:, :Cc].double().requires_grad_(True)
        g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        out = _gn64(x64, g64, b64, swish, B, HW, Cc, groups, eps)
        gx, gg, gb = torch.autograd.grad(out, (x64, g64, b64), dy[:, :Cc].double().view(B, HW, Cc))
        key = 'bwd %dpx C%d' % (HW, Cc)
        dxv, gxv = dx[:, :Cc].view(B, HW, Cc), gx.view(B, HW, Cc)
        ck(key + ' dx', rel(dxv, gxv), 2.8e-7, rel(dxv, gxv.roll(1, 0)))                 # measured <= 9.4e-8
        if has_params:
            ck(key + ' dgamma', rel(dg, dg0.double() + gg), 1.09e-6, rel(dg, gg))       # measured <= 3.65e-7
            ck(key + ' dbeta', rel(db, db0.double() + gb), 1.06e-6, rel(db, gb))         # measured <= 3.54e-7
        ck.require(key + ': padding untouched', bool((dx[:, Cc:] == 7.0).all()))
    ck.done()


# relative error against fp64 over max(1, sqrt(K / 2304)) (fp32 accumulation error grows with the contraction length K); over
# the 141 replayed descriptors this measured at most 5.3e-6 (out), 5.7e-6 (dw) and 9.5e-8 (db).  No descriptor has an out2.
CONV_BOUND = {'out': 1.5e-5, 'out2': 1.5e-5, 'dw': 1.7e-5, 'db': 2.8e-7}


def test_convolutions_of_the_b128_step_replayed_against_fp64(rec):
    """every cd_conv_fwd / cd_conv_wgrad descriptor of a B = 128 training step, replayed on TF32-rounded operands: the dense
    3x3 and 1x1 convolutions with their data gradients, the two-source skip concats (384 / 512 -> C with the shortcut), the
    stride-2 downsamples and their parity data gradients, the 4 x 4 levels, and the AttnBlock's per-image products (s . v on
    wgmma, q . k^T, ds and dq on the CUDA cores, dv by per-image wgrad on wgmma and dk on the CUDA cores).  Controls: the last
    image's reference replaced by the first image's (forward), the last image left out (weight gradient)."""
    from cold_diffusion_models_b200 import ops
    ck = Checks10('B128 convolutions')
    g = gen(2025)
    seen = set()
    specs = rec[128]['convs']
    for sp in specs:
        ck.require('%s: engine asked for TF32-rounded outputs' % _label(sp), not sp['rnd'])
        res, ok = _replay(sp, g)
        ck.require('%s: outside the written region untouched' % _label(sp), ok)
        for what, v, c, K in res:
            b = CONV_BOUND[what] * max(1.0, (K / 2304) ** 0.5)
            ck('%s %s' % (_label(sp), what), v, b, c)
        wpb = any(s[6] for s in sp['srcs'])
        seen.add((sp['kind'], sp['impl'] == ops.CONV_TC, sp['Hg'], len(sp['srcs']), sp['sy'], wpb))
    _METRICS['B128 convolutions::replayed'] = len(specs)
    TC, SIMT = True, False
    for kind, impl, H, nsrc, sy, wpb, what in [
            ('fwd', TC, 16, 1, 1, True, 's . v (per-image weights on wgmma)'),
            ('fwd', SIMT, 16, 1, 1, True, 'q . k^T, ds, dq (per-image weights on the CUDA cores)'),
            ('wgrad', TC, 16, 1, 1, True, 'dv (per-image weight gradient on wgmma)'),
            ('wgrad', SIMT, 16, 1, 1, True, 'dk (per-image weight gradient on the CUDA cores)'),
            ('fwd', TC, 32, 2, 1, False, 'two-source skip concat at 32²'),
            ('fwd', TC, 4, 2, 1, False, 'two-source skip concat at 4²'),
            ('fwd', TC, 16, 1, 2, False, 'stride-2 downsample 32 -> 16'),
            ('wgrad', TC, 16, 1, 2, False, 'stride-2 downsample weight gradient'),
            ('fwd', TC, 4, 1, 1, False, '4 x 4 level on the tensor cores'),
            ('wgrad', TC, 4, 1, 1, False, '4 x 4 level weight gradient on wgmma')]:
        ck.require('%s ran' % what, (kind, impl, H, nsrc, sy, wpb) in seen)
    ck.done()


# (B, side, Cout, out_ld, c0): 3x3 forwards whose Cout is not a multiple of 4, into a view whose row continues with live
# columns.  By shape these grids would take the 16 x 16 shared-row kernel, whose TMA stores write whole 16-byte groups.
NARROW_COUT = [(128, 32, 3, 4, 0), (128, 32, 3, 8, 0), (128, 32, 3, 8, 4), (128, 32, 6, 8, 0), (16, 128, 3, 8, 4)]


@pytest.mark.parametrize('case', NARROW_COUT, ids=['B%d-%d-Cout%d-ld%d-c0%d' % c for c in NARROW_COUT])
def test_conv_forward_with_cout_not_a_multiple_of_4(case):
    """the Model's conv_out (128 -> 3 channels, rows of 4 floats) and 3- / 6-channel slices of wider rows: the forward leaves
    every element outside its view untouched and matches float64.  Control: the last image's reference replaced by the
    first image's."""
    from cold_diffusion_models_b200 import ops
    B, S, Cout, ld, c0 = case
    ck = Checks10('narrow Cout %s' % (case,))
    taps = tuple((dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1))
    sp = dict(kind='fwd', impl=ops.CONV_TC, B=B, Hg=S, Wg=S, sy=1, sx=1, Cout=Cout, srcs=((128, 128, S, S, 0, taps, 0),),
              omap=(1, 1, 0, 0), rnd=0, out=(ld, c0, S, S), bias=True, act=ops.ACT_NONE, resid=None, out2=None, aux=None)
    res, ok = _replay(sp, gen(2100 + Cout + ld + c0))
    ck.require('outside the %d-channel view untouched' % Cout, ok)
    (what, v, c, K), = res
    ck('out', v, CONV_BOUND[what] * max(1.0, (K / 2304) ** 0.5), c)
    ck.done()


# ==========================================================================================================================
# 4. the kernels that run
# ==========================================================================================================================
def _kernel_names(m, gd, B, train=True):
    from torch.profiler import profile, ProfilerActivity
    x, t = _batch(B, 32, 700 + B)
    torch.manual_seed(1)

    def run():
        if train:
            gd.p_losses(x, t).backward()
        else:
            with torch.no_grad():
                m(x, t)
        torch.cuda.synchronize()
        m.zero_grad(set_to_none=True)
    run()                                                     # first pass outside the trace: buffers, packs
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
    return {e.name for e in prof.events()}


def test_dispatch_at_b128_and_b2():
    """one 32² training step under torch.profiler at B = 128 and at B = 2, and one inference forward at B = 128: the kernels
    this file checks are the ones that run, and the cd_small_gemm branch changes with B as the tests above assume"""
    m = _model(32, seed=12)
    m.train()
    gd = _gd(m, 32)
    n128, n2 = _kernel_names(m, gd, 128), _kernel_names(m, gd, 2)
    m.eval()
    ninf = _kernel_names(m, gd, 128, train=False)
    has = lambda names, k: any(k in n for n in names)
    fails = []
    for k in ('small_gemm_kernel', 'dropout_kernel', 'softmax_rows_kernel', 'softmax_bwd_rows_kernel', 'upsample_nearest2x_kernel',
              'upsample_nearest2x_bwd_kernel', 'transpose_batched_kernel', 'timestep_embedding_kernel', 'linear_kernel',
              'swish_kernel', 'colsum_vec_kernel'):
        if not has(n128, k):
            fails.append('%s missing at B = 128' % k)
    if has(n128, 'small_gemm_splitk_kernel'):
        fails.append('small_gemm_splitk_kernel ran at B = 128')
    if not has(n2, 'small_gemm_splitk_kernel'):
        fails.append('small_gemm_splitk_kernel missing at B = 2')
    for k in ('time_mlp2_dense_kernel', 'cond_proj_kernel'):
        if not has(ninf, k):
            fails.append('%s missing in the B = 128 inference forward' % k)
    assert not fails, (fails, sorted(n for n in n128 | n2 if 'kernel' in n)[:80])
