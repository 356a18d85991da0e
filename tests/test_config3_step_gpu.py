"""The benchmarked training step -- `Unet(64, (1, 2, 4, 8))` on 3 x 128^2 images, Exponential_reflect blur (k = 15, T = 200), two
micro-batches of 32 and the fused Adam + EMA step -- and the memory-bound kernels it runs, at the shapes and launch configurations
of that step, against float64 references computed on the GPU (oracle/unet_oracle.py, oracle/deblur_oracle.py, plain torch).

Every comparison also evaluates its metric on a deliberately wrong reference (a "negative control": an image left out, an
overwrite instead of an accumulation, a step index off by one, ...) and asserts that it exceeds the bound, so each bound is shown
to catch the class of bug it is there for.  The bounds were set from a run on an H100 80GB HBM3; the measured values are in the
comments beside them.  Set COLDDIFF_TEST_METRICS=<file> to write every measured value and control to a JSON file.

References run in float64 in chunks of at most 8 images (a full-batch q_sample would stack 200 blurred copies) and are freed
between tests."""
import contextlib
import ctypes as C
import gc
import io
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

import deblur_oracle as DO
import unet_oracle as UO

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F64 = torch.float64
C3 = dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3, image_size=128, timesteps=200, kernel_size=15, kernel_std=0.01,
          blur_routine='Exponential_reflect', sampling_routine='x0_step_down')
LEVELS = [(128, 64), (64, 128), (32, 256), (16, 512)]          # (image side, channels) of the four Unet levels
# The training-step tests run Adam at lr 1e-3 instead of the benchmark's 2e-5: one step then moves every weight by about 1e-3,
# so the gradient at the new weights differs from the one at the old weights by far more than the TF32 rounding (B5's control).
LR = 1e-3
_METRICS = {}


# --------------------------------------------------------------------------------------------------------------------------
# helpers
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


class Checks:
    """collects every (value < bound) and (control > bound) of one test, records them, and fails at the end with all of them"""

    def __init__(self, test):
        self.test, self.fails = test, []

    def __call__(self, name, value, bound, control=None):
        key = '%s::%s' % (self.test, name)
        _METRICS[key] = dict(value=float(value), bound=float(bound), control=None if control is None else float(control))
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


def maxabs(a, b):
    return (a.to(F64) - b.to(F64)).abs().max().item()


def call(name, *args):
    from cold_diffusion_models_b200._lib import call as _call
    _call(name, *args)


def ptr(t):
    from cold_diffusion_models_b200._lib import ptr as _ptr
    return _ptr(t)


def stream():
    from cold_diffusion_models_b200._lib import stream as _stream
    return _stream()


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(*shape, g, scale=1.0):
    return torch.randn(*shape, generator=g, device=DEV) * scale


def sentinel(*shape):
    return torch.full(shape, 7.0, device=DEV)


def blur_oracle(S, routine='Exponential_reflect', kernel_size=15, kernel_std=0.01, discrete=False):
    o = DO.DeblurOracle(None, image_size=S, channels=3, timesteps=200, kernel_std=kernel_std, kernel_size=kernel_size,
                        blur_routine=routine, discrete=discrete)
    o.kernels2d = [k.double().cuda() for k in o.kernels2d]
    return o


def blur_per_image(o, x64, t, chunk=8):
    """x_{t_b} = blur steps 0..t_b applied to image b (t_b < 0: the image itself): the sequential fp64 stencils of DeblurOracle,
    at most `chunk` images at a time, keeping only each image's own step"""
    out = x64.clone()
    tl = [int(v) for v in t]
    for c in range(0, x64.shape[0], chunk):
        h, tc = x64[c:c + chunk], tl[c:c + chunk]
        for i in range(max(tc) + 1):
            h = o.blur_step(i, h)
            for j, tj in enumerate(tc):
                if tj == i:
                    out[c + j] = h[j]
    return out


def F32(v):
    """the float nearest to v in fp32: cd_adam_ema_step takes its betas as fp32, so (1 - beta2) is 1 - fp32(0.999), 1.3e-5 below
    torch.optim.Adam's 1 - 0.999 (the same relative shift of exp_avg_sq); the references use the betas the kernel receives"""
    return float(torch.tensor(v, dtype=torch.float32))


def quantize(x):
    """DB:954-958 (8-bit truncation toward zero)"""
    q = (x + 1) * 0.5 * 255
    return torch.trunc(q) / 255 * 2 - 1


# --------------------------------------------------------------------------------------------------------------------------
# the benchmarked model
# --------------------------------------------------------------------------------------------------------------------------
class Config3:
    pass


@pytest.fixture(scope='module')
def c3(tmp_path_factory):
    """Unet, GaussianDiffusion and Trainer built the way bench.py builds them, from a deterministic reference-format state_dict,
    with three micro-batches of 32 images and fixed per-image t"""
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        unet = cdm.Unet(dim=C3['dim'], dim_mults=C3['dim_mults'], channels=C3['channels']).to(DEV)
        unet.load_state_dict(UO.make_unet_state_dict(64, (1, 2, 4, 8), 3, seed=3))
        gd = cdm.GaussianDiffusion(unet, image_size=128, device_of_kernel='cuda', channels=3, timesteps=C3['timesteps'],
                                   loss_type='l2', kernel_std=C3['kernel_std'], kernel_size=C3['kernel_size'],
                                   blur_routine=C3['blur_routine'], train_routine='Final', sampling_routine=C3['sampling_routine'],
                                   discrete=False).to(DEV)
        tr = cdm.Trainer(gd, None, image_size=128, train_batch_size=32, train_lr=LR, train_num_steps=10 ** 9,
                         gradient_accumulate_every=2, ema_decay=0.995, fp16=False,
                         results_folder=str(tmp_path_factory.mktemp('results')), dataset='synthetic')
    g = torch.Generator().manual_seed(1234)
    xs = [(torch.rand(32, 3, 128, 128, generator=g) * 2 - 1).to(DEV) for _ in range(3)]
    ts = [torch.randint(0, 200, (32,), generator=g).to(DEV) for _ in range(3)]
    for t in ts:
        t[0], t[1], t[2] = 0, 199, 1
    s = Config3()
    s.unet, s.gd, s.tr, s.eng, s.xs, s.ts = unet, gd, tr, unet.engine, xs, ts
    s.oracle = blur_oracle(128)
    yield s
    s.eng.conv_impl = 1
    del s


def engine_grads(unet):
    return {n: p.grad.detach().clone() for n, p in unet.named_parameters()}


def ref_step(sd, x0, xt64, t, norm, chunk=2, want=True):
    """fp64 autograd of sum_b |x0_b - R(x_t_b, t_b)|^2 / norm through oracle/unet_oracle.py, `chunk` images at a time.
    -> (gradients by parameter name, loss, network output)"""
    leaves = {k: v.detach().to(DEV, F64).requires_grad_(want) for k, v in sd.items()}
    names = list(leaves)
    acc = {k: torch.zeros_like(v) for k, v in leaves.items()} if want else None
    loss, ys = 0.0, []
    for i in range(0, x0.shape[0], chunk):
        with torch.set_grad_enabled(want):
            y = UO.unet_forward(leaves, xt64[i:i + chunk], t[i:i + chunk].to(F64))
            d = x0[i:i + chunk].to(F64) - y
            lo = (d * d).sum() / norm
        if want:
            for k, gr in zip(names, torch.autograd.grad(lo, [leaves[k] for k in names])):
                acc[k] += gr
        loss += lo.item()
        ys.append(y.detach())
        del y, d, lo
    return acc, loss, torch.cat(ys)


def grad_errors(eng_g, ref_g):
    return sorted((rel(eng_g[n], ref_g[n]), n) for n in ref_g)


def stats(errs):
    return errs[len(errs) // 2][0], errs[int(len(errs) * 0.9)][0], errs[-1][0]


# ==========================================================================================================================
# A. memory-bound kernels at the config-3 shapes
# ==========================================================================================================================
@pytest.mark.parametrize('S,routine', [(128, 'Exponential_reflect'), (64, 'Exponential_reflect'), (128, 'Incremental')])
def test_blur_apply_and_step_down_against_fp64_stencils(S, routine):
    """cd_blur_apply (q_sample with per-sample t, `discrete` collapse and 8-bit truncation) and cd_blur_step_down (Algorithm 2)
    at B = 32 against the sequential fp64 blur steps; S = 128 is the largest shared-memory layout (three 128 x 128 planes)"""
    from cold_diffusion_models_b200.degradation import build_blur_operators
    ck = Checks('blur[%d,%s]' % (S, routine))
    kstd = 0.01 if routine == 'Exponential_reflect' else 0.5
    B, T = 32, 200
    o = blur_oracle(S, routine, 15, kstd)
    ops_cum = build_blur_operators(routine, T, 15, kstd, S)[0].to(DEV)
    g = gen(S + len(routine))
    x = torch.rand(B, 3, S, S, generator=g, device=DEV) * 2 - 1
    x64 = x.double()
    t = torch.tensor([-1, 0, 1, 100, 199] * 6 + [199, 0], device=DEV)
    ref = blur_per_image(o, x64, t)
    ref_shift = blur_per_image(o, x64, torch.where(t < 199, t + 1, t - 1))       # control: every step index off by one
    last = (t == T - 1)
    ref_col = ref.clone()
    ref_col[last] = ref[last].mean(dim=(2, 3), keepdim=True).expand_as(ref[last])
    for collapse in (0, 1):
        r = ref_col if collapse else ref
        for quant in (0, 1):
            out = sentinel(B, 3, S, S)
            call('cd_blur_apply', ptr(x), ptr(out), ptr(ops_cum), ptr(t), 0, B, 3, S, T, collapse, quant, stream())
            if quant:
                d = (out.double() - quantize(r)).abs()
                # truncation at a 1/255 boundary flips on fp32-level differences: at most two levels, on few pixels
                ck('q_sample c%d q1 max' % collapse, d.max().item(), 2 / 255 + 1e-6)
                ck('q_sample c%d q1 flipped fraction' % collapse, (d > 1e-6).double().mean().item(), 7e-6,      # measured <= 2.5e-6
                   ((quantize(ref_shift) - quantize(r)).abs() > 1e-6).double().mean().item())
            else:
                ck('q_sample c%d' % collapse, maxabs(out, r), 4e-7, maxabs(ref_shift, r))        # measured <= 1.4e-7
    # Algorithm-2 update x_{t-1} = x_t - D(xhat, t) + D(xhat, t - 1) for the highest, a middle and the first step
    xt = torch.rand(B, 3, S, S, generator=g, device=DEV) * 2 - 1
    for hi in (199, 100, 0):
        d_hi = blur_per_image(o, x64, torch.full((B,), hi))
        d_lo = blur_per_image(o, x64, torch.full((B,), hi - 1))
        for collapse in ((0, 1) if hi == T - 1 else (0,)):
            dh = d_hi.mean(dim=(2, 3), keepdim=True).expand_as(d_hi) if collapse else d_hi
            r = xt.double() - dh + d_lo
            out = sentinel(B, 3, S, S)
            call('cd_blur_step_down', ptr(xt), ptr(x), ptr(out), ptr(ops_cum), hi, hi - 1, B, 3, S, T, collapse, stream())
            wrong = xt.double() - blur_per_image(o, x64, torch.full((B,), max(hi - 2, -1))) + d_lo if hi > 0 else xt.double()
            ck('step_down hi=%d c%d' % (hi, collapse), maxabs(out, r), 6e-7, maxabs(wrong, r))      # measured <= 2.3e-7
    ck.done()


@pytest.mark.parametrize('mode', [0, 1])
def test_loss_kernel_against_fp64(mode):
    """cd_loss_fwd_bwd at n = 32 * 3 * 128^2: grad_scale != 1, the loss added to a non-zero scalar, exactly equal elements
    (L1: the gradient of sign(0) is 0)"""
    ck = Checks('loss[%s]' % ('l1' if mode == 0 else 'l2'))
    n = 32 * 3 * 128 * 128
    g = gen(21 + mode)
    x0 = torch.rand(n, generator=g, device=DEV) * 2 - 1
    xh = x0 + randn(n, g=g, scale=0.3)
    eq = torch.arange(n, device=DEV) % 7 == 3
    xh[eq] = x0[eq]
    loss = torch.full((), 0.25, device=DEV)
    dx = sentinel(n)
    gs = 0.37
    call('cd_loss_fwd_bwd', ptr(x0), ptr(xh), C.c_int64(n), mode, C.c_float(gs), ptr(loss), ptr(dx), stream())
    d = xh.double() - x0.double()
    lref = 0.25 + (d.abs().mean() if mode == 0 else (d * d).mean()).item()
    gref = (torch.sign(d) if mode == 0 else 2 * d) / n * gs
    ck('loss', abs(loss.item() - lref) / lref, 1.5e-6, abs(lref - 0.25 - lref) / lref)      # measured 4.8e-8 (l1), 5.2e-7 (l2)
    ck('grad', rel(dx, gref), 1.5e-7, rel(gref / gs, gref))                                 # measured 1.3e-8 (l1), 5.5e-8 (l2)
    ck.require('gradient at equal elements is exactly 0', bool((dx[eq] == 0).all()) if mode == 0 else True)
    ck.done()


def _engine_lds(c3):
    """(x_ld of the attention LayerNorm, ld of the block LayerNorm) per level, read from a training forward of the live engine"""
    save = {}
    x = c3.xs[0][:2]
    c3.eng.forward(x, c3.ts[0][:2], save=save)
    out = []
    for i in range(4):
        att = save['downs.%d.2' % i]
        blk = save['downs.%d.1' % i]
        out.append((att['x'].ld, blk['ld_h'], blk['x'].ld))
    return out


@pytest.mark.parametrize('B', [32, 2])
def test_layernorm_forward_and_backward_against_fp64_autograd(c3, B):
    """cd_layernorm_fwd (default kernel) and cd_layernorm_bwd at every level's (pixels, channels), with the row strides the
    engine uses and with a channel slice of a concat buffer, with and without `addend`, dg / dbeta accumulating"""
    ck = Checks('layernorm[B=%d]' % B)
    lds = _engine_lds(c3)
    for lvl, ((side, Cc), (att_ld, blk_ld, _)) in enumerate(zip(LEVELS, lds)):
        npix = B * side * side
        g = gen(100 + lvl)
        for tag, ld, c0 in (('engine-ld', att_ld, 0), ('concat-slice', 2 * Cc, Cc)):
            xbuf = randn(npix, ld, g=g, scale=2.0) + 0.3
            xv = xbuf[:, c0:c0 + Cc]
            gam, bet = 1 + randn(Cc, g=g, scale=0.2), randn(Cc, g=g, scale=0.1)
            y, st = sentinel(npix, blk_ld), sentinel(npix, 2)
            call('cd_layernorm_fwd', C.c_void_p(xv.data_ptr()), ld, C.c_int64(npix), Cc, ptr(gam), ptr(bet), C.c_float(1e-5),
                 ptr(y), blk_ld, ptr(st), 0, stream())
            x64 = xv.double().t().reshape(1, Cc, npix, 1).requires_grad_(True)
            g64, b64 = gam.double().reshape(1, Cc, 1, 1), bet.double().reshape(1, Cc, 1, 1)
            y64 = UO.layer_norm(x64, g64, b64)
            yref = y64.detach().reshape(Cc, npix).t()
            var_nm1 = torch.var(x64.detach(), dim=1, unbiased=True, keepdim=True)       # control: unbiased variance
            ywrong = ((x64.detach() - x64.detach().mean(1, keepdim=True)) / (var_nm1 + 1e-5).sqrt() * g64 + b64).reshape(Cc, npix).t()
            ck('fwd L%d %s' % (lvl, tag), rel(y[:, :Cc], yref), 1.8e-7, rel(ywrong, yref))          # measured <= 6.2e-8
            ck.require('fwd L%d %s: padding untouched' % (lvl, tag), bool((y[:, Cc:] == 7.0).all()))
            dy = randn(npix, Cc, g=g)
            gx, = torch.autograd.grad(y64, x64, dy.double().t().reshape(1, Cc, npix, 1))
            gx = gx.reshape(Cc, npix).t()
            dgr = (dy.double() * ((x64.detach().reshape(Cc, npix).t() - x64.detach().mean(1).reshape(npix, 1)) /
                                  (x64.detach().var(1, unbiased=False).reshape(npix, 1) + 1e-5).sqrt())).sum(0)
            dbr = dy.double().sum(0)
            for with_add in (0, 1):
                addbuf = randn(npix, 2 * Cc, g=g)
                add = addbuf[:, :Cc] if with_add else None
                dg0, db0 = randn(Cc, g=g), randn(Cc, g=g)
                dg, db = dg0.clone(), db0.clone()
                dh = sentinel(npix, blk_ld)
                call('cd_layernorm_bwd', ptr(dy), Cc, C.c_void_p(xv.data_ptr()), ld, ptr(st), ptr(gam), C.c_int64(npix), Cc,
                     ptr(add), 2 * Cc if with_add else 0, ptr(dh), blk_ld, ptr(dg), ptr(db), stream())
                dref = gx + (add.double() if with_add else 0)
                k = 'bwd L%d %s add%d' % (lvl, tag, with_add)
                ck(k + ' dh', rel(dh[:, :Cc], dref), 2e-7,                 # measured <= 6.9e-8
                   rel(gx if with_add else gx + addbuf[:, :Cc].double(), dref))
                ck(k + ' dg', rel(dg, dg0.double() + dgr), 2e-6,          # measured <= 7.1e-7
                   rel(dgr, dg0.double() + dgr))
                ck(k + ' dbeta', rel(db, db0.double() + dbr), 2e-6,      # measured <= 7.1e-7
                   rel(dbr, db0.double() + dbr))
            del xbuf, y, st, x64, y64, yref, ywrong, gx, dy, dh
    ck.done()


def _attn_core64(k, v, w_out, scale):
    """the attention core of unet_oracle.linear_attention_block as the per-image effective weight of the `to_out` projection:
    to_out(einsum(softmax_n(k) v^T, q * scale)) == conv1x1(q, weff[b]) with
    weff[b, co, h*32+d] = scale * sum_e w_out[co, h*32+e] * ctx[b, h, d, e], ctx = softmax_n(k) v^T  (k, v: [B][n][128])"""
    B, n, _ = k.shape
    kk = k.transpose(1, 2).reshape(B, 4, 32, n).softmax(dim=-1)
    vv = v.transpose(1, 2).reshape(B, 4, 32, n)
    ctx = torch.einsum('bhdn,bhen->bhde', kk, vv)
    weff = scale * torch.einsum('che,bhde->bchd', w_out.reshape(-1, 4, 32), ctx)
    return weff.reshape(B, -1, 128), ctx


@pytest.mark.parametrize('B', [32, 2])
def test_linear_attention_kernels_against_fp64(B):
    """cd_linattn_context_det with the engine's plan and with a hand plan whose last block is ragged, cd_linattn_weff,
    cd_linattn_bwd_small and the default (tensor-core) cd_linattn_bwd_kv against fp64 (autograd of the attention core)"""
    from cold_diffusion_models_b200 import ops
    ck = Checks('linattn[B=%d]' % B)
    scale = 32 ** -0.5
    cases = [(s * s, Cc) for s, Cc in LEVELS] + [(1000, 64)]
    for n, dim in cases:
        g = gen(300 + n)
        qkv = randn(B, n, 384, g=g)
        qkv[..., 128:256] *= 2.0
        kmax_ref = qkv[..., 128:256].max(dim=1).values
        ksum_ref, ctx_ref, ctx_tail, tsum = [], [], [], []
        for c in range(0, B, 8):                        # fp64 references 8 images at a time
            k64, v64 = qkv[c:c + 8, :, 128:256].double(), qkv[c:c + 8, :, 256:].double()
            e = torch.exp(k64 - kmax_ref[c:c + 8].double()[:, None, :])
            ksum_ref.append(e.sum(1))
            ctx_ref.append(torch.einsum('bnc,bne->bce', e, v64).reshape(-1, 4, 32, 4, 32).diagonal(dim1=1, dim2=3).permute(0, 3, 1, 2))
            et = torch.exp(k64[:, :-32] - k64[:, :-32].max(1, keepdim=True).values)   # control: the last 32 pixels dropped
            tsum.append(et.sum(1))
            ctx_tail.append(torch.einsum('bnc,bne->bce', et, v64[:, :-32]).reshape(-1, 4, 32, 4, 32).diagonal(dim1=1, dim2=3).permute(0, 3, 1, 2))
            del k64, v64, e, et
        ksum_ref, ctx_ref, ctx_tail, tsum = (torch.cat(a) for a in (ksum_ref, ctx_ref, ctx_tail, tsum))
        ctxn_ref = ctx_ref / ksum_ref.reshape(B, 4, 32, 1)
        ctxn_tail = ctx_tail / tsum.reshape(B, 4, 32, 1)
        plans = [('engine', ops.linattn_ctx_plan(B, n, DEV))]
        ppb = 224
        plans.append(('ragged', (-(-n // ppb), ppb)))
        assert n % ppb != 0
        for tag, (nblk, ppb_) in plans:
            ws = torch.empty(B, nblk, 4352, device=DEV)
            kmax, ksum, ctx = sentinel(B, 128), sentinel(B, 128), sentinel(B, 4, 32, 32)
            call('cd_linattn_context_det', ptr(qkv), 384, B, n, nblk, ppb_, ptr(ws), ptr(kmax), ptr(ksum), ptr(ctx), stream())
            key = 'ctx n=%d %s' % (n, tag)
            ck.require(key + ': kmax exact', bool(torch.equal(kmax, kmax_ref)))
            ck(key + ' ksum', rel(ksum, ksum_ref), 5e-7,                 # measured <= 1.8e-7
               rel(ksum.roll(1, 0), ksum_ref))
            ckn = ctx.double() / ksum.double().reshape(B, 4, 32, 1)
            # measured 9.4e-6 with the engine's plan at B = 32, n = 16384 (1376 pixels per block), <= 2.4e-6 elsewhere: the error grows
            # linearly with the pixels a block sums, as the truncating fp32 accumulation inside mma.sync does
            ck(key + ' ctx', rel(ckn, ctxn_ref), 2.8e-5, rel(ctxn_tail, ctxn_ref))
            del ws
        # effective weight, from the kernel's own context
        w_out = randn(dim, 128, g=g, scale=128 ** -0.5)
        weff = sentinel(B, dim, 128)
        call('cd_linattn_weff', ptr(ctx), ptr(ksum), ptr(w_out), B, dim, C.c_float(scale), 0, ptr(weff), stream())
        cn = (ctx.double() / ksum.double().reshape(B, 4, 32, 1))
        wref = (scale * torch.einsum('che,bhde->bchd', w_out.double().reshape(dim, 4, 32), cn)).reshape(B, dim, 128)
        ck('weff n=%d' % n, rel(weff, wref), 3.3e-7,                   # measured <= 1.1e-7
           rel(weff.roll(1, 0), wref) if B > 1 else rel(weff * 1.01, wref))
        # backward of the core: dweff -> dw_out (accumulated), dk, dv
        dweff = randn(B, dim, 128, g=g)
        dk_ref, dv_ref, dw_ref = [], [], 0
        for c in range(0, B, 8):
            kl, vl = qkv[c:c + 8, :, 128:256].double().requires_grad_(True), qkv[c:c + 8, :, 256:].double().requires_grad_(True)
            wl = w_out.double().requires_grad_(True)
            wr, _ = _attn_core64(kl, vl, wl, scale)
            a, b_, w_ = torch.autograd.grad(wr, (kl, vl, wl), dweff[c:c + 8].double())
            dk_ref.append(a)
            dv_ref.append(b_)
            dw_ref = dw_ref + w_
            del kl, vl, wl, wr, a, b_
        dk_ref, dv_ref = torch.cat(dk_ref), torch.cat(dv_ref)
        dw0 = randn(dim, 128, g=g)
        dw = dw0.clone()
        dctxn, rowdot = sentinel(B, 4, 32, 32), sentinel(B, 128)
        call('cd_linattn_bwd_small', ptr(dweff), ptr(ctx), ptr(ksum), ptr(w_out), B, dim, C.c_float(scale), ptr(dw), ptr(dctxn),
             ptr(rowdot), stream())
        ck('bwd_small n=%d dw_out' % n, rel(dw, dw0.double() + dw_ref), 3.8e-6,      # measured <= 1.3e-6
           rel(dw_ref, dw0.double() + dw_ref))
        for dld in ((384, 392) if n == 1000 else (384,)):
            dq = sentinel(B, n, dld)
            call('cd_linattn_bwd_kv', ptr(qkv), 384, B, n, ptr(kmax), ptr(ksum), ptr(dctxn), ptr(rowdot), ptr(dq), dld, stream())
            key = 'bwd_kv n=%d dld=%d' % (n, dld)
            ck(key + ' dk', rel(dq[..., 128:256], dk_ref), 2.3e-6,      # measured <= 7.8e-7
               rel(dq[..., 128:256].roll(1, 0), dk_ref) if B > 1 else rel(dq[..., 128:256], dk_ref - dk_ref.mean(1, keepdim=True)))
            ck(key + ' dv', rel(dq[..., 256:384], dv_ref), 2.3e-6,      # measured <= 4.9e-7
               rel(dq[..., 256:384].roll(1, 0), dv_ref) if B > 1 else rel(dq[..., 256:384] * 1.01, dv_ref))
            ck.require(key + ': q columns and padding untouched', bool((dq[..., :128] == 7.0).all() and (dq[..., 384:] == 7.0).all()))
            del dq
        del qkv, dk_ref, dv_ref
    ck.done()


@pytest.mark.parametrize('B', [32, 2])
def test_column_sums_against_fp64(c3, B):
    """cd_colsum and cd_colsum_batched (default kernels) over B * 16384 rows, into a wider output row (out_ld > C) that starts
    non-zero; the engine's sumC is the row stride of the batched sums"""
    ck = Checks('colsum[B=%d]' % B)
    sumC = c3.eng.sumC
    for side, Cc in LEVELS:
        rows = side * side
        g = gen(400 + Cc)
        x = randn(B, rows, Cc, g=g)
        out0 = randn(Cc + 16, g=g)
        out = out0.clone()
        call('cd_colsum', ptr(x), Cc, C.c_int64(B * rows), Cc, ptr(out), stream())
        ref = out0[:Cc].double() + x.double().sum((0, 1))
        short = out0[:Cc].double() + x.reshape(-1, Cc)[:-2048].double().sum(0)      # control: the last 2048 rows dropped
        ck('colsum C=%d' % Cc, rel(out[:Cc], ref), 1.3e-6, rel(short, ref))          # measured <= 4.5e-7
        ck.require('colsum C=%d: beyond C untouched' % Cc, bool(torch.equal(out[Cc:], out0[Cc:])))
        off = 64
        ob0 = randn(B, sumC, g=g)
        ob = ob0.clone()
        call('cd_colsum_batched', ptr(x), Cc, B, C.c_int64(rows), Cc, C.c_void_p(ob.data_ptr() + 4 * off), sumC, stream())
        refb = ob0[:, off:off + Cc].double() + x.double().sum(1)
        ck('colsum_batched C=%d' % Cc, rel(ob[:, off:off + Cc], refb), 1e-6,       # measured <= 3.3e-7
          
           rel(ob0[:, off:off + Cc].double() + x[:, :-2048].double().sum(1), refb))
        ck.require('colsum_batched C=%d: other columns untouched' % Cc,
                   bool(torch.equal(ob[:, :off], ob0[:, :off]) and torch.equal(ob[:, off + Cc:], ob0[:, off + Cc:])))
    ck.done()


def test_final_projection_forward_and_backward_against_fp64():
    """cd_conv1x1_to_nchw (with the residual image) and cd_conv1x1_to_nchw_bwd at B = 32, 128^2, 64 -> 3 channels"""
    ck = Checks('final_proj')
    B, H, Cc, Co = 32, 128, 64, 3
    g = gen(500)
    x = randn(B, H, H, Cc, g=g)
    w, b = randn(Co, Cc, g=g, scale=0.125), randn(Co, g=g)
    r = randn(B, Co, H, H, g=g)
    out = sentinel(B, Co, H, H)
    call('cd_conv1x1_to_nchw', ptr(x), Cc, B, H, H, Cc, ptr(w), ptr(b), Co, ptr(r), ptr(out), stream())
    ref = torch.einsum('bhwc,oc->bohw', x.double(), w.double()) + b.double()[None, :, None, None] + r.double()
    ck('fwd', rel(out, ref), 3.6e-7,           # measured 1.2e-7
        rel(ref - r.double(), ref))
    dout = randn(B, Co, H, H, g=g)
    dx = sentinel(B, H, H, Cc)
    dw0, db0 = randn(Co, Cc, g=g), randn(Co, g=g)
    dw, db = dw0.clone(), db0.clone()
    call('cd_conv1x1_to_nchw_bwd', ptr(dout), ptr(x), Cc, B, H, H, Cc, ptr(w), Co, ptr(dx), Cc, ptr(dw), ptr(db), stream())
    dxr = torch.einsum('bohw,oc->bhwc', dout.double(), w.double())
    dwr = torch.einsum('bohw,bhwc->oc', dout.double(), x.double())
    dbr = dout.double().sum((0, 2, 3))
    ck('bwd dx', rel(dx, dxr), 1.1e-7,        # measured 3.6e-8
        rel(dx.roll(1, 0), dxr))
    ck('bwd dw', rel(dw, dw0.double() + dwr), 1.5e-6,       # measured 5.2e-7
        rel(dwr, dw0.double() + dwr))
    ck('bwd db', rel(db, db0.double() + dbr), 1.2e-6,       # measured 3.9e-7
        rel(dbr, db0.double() + dbr))
    ck.done()


def test_time_mlp_helpers_against_fp64(c3):
    """cd_time_mlp_fwd, cd_gelu_bwd and cd_small_gemm (both transposes, with and without accumulation, and the split-K branch
    that the dgt = dcond . Wc product takes) at B = 32, dim = 64 and the engine's sumC"""
    ck = Checks('time_mlp')
    B, dim, sumC = 32, 64, c3.eng.sumC
    g = gen(600)
    t = torch.randint(0, 200, (B,), device=DEV, generator=g)
    w1, b1 = randn(4 * dim, dim, g=g, scale=0.125), randn(4 * dim, g=g, scale=0.1)
    w2, b2 = randn(dim, 4 * dim, g=g, scale=0.06), randn(dim, g=g, scale=0.1)
    wc, bc = randn(sumC, dim, g=g, scale=0.125), randn(sumC, g=g, scale=0.1)
    sinemb, hid, temb, cond = sentinel(B, dim), sentinel(B, 4 * dim), sentinel(B, dim), sentinel(B, sumC)
    call('cd_time_mlp_fwd', ptr(t), B, dim, ptr(w1), ptr(b1), ptr(w2), ptr(b2), ptr(wc), ptr(bc), sumC, ptr(sinemb), ptr(hid),
         ptr(temb), ptr(cond), stream())
    se = UO.sinusoidal_pos_emb(t.to(F64), dim)
    hr = se @ w1.double().t() + b1.double()
    tr = F.gelu(hr) @ w2.double().t() + b2.double()
    cr = F.gelu(tr) @ wc.double().t() + bc.double()
    se_wrong = UO.sinusoidal_pos_emb((t + 1).to(F64), dim)                       # control: t off by one
    ck('sinemb', rel(sinemb, se), 1.7e-6,        # measured 5.8e-7
       rel(se_wrong, se))
    ck('hid_pre', rel(hid, hr), 1.7e-6,          # measured 5.7e-7
       rel(hr.roll(1, 0), hr))
    ck('temb', rel(temb, tr), 1.9e-6,             # measured 6.6e-7
       rel(tr.roll(1, 0), tr))
    ck('cond_all', rel(cond, cr), 1.8e-6,         # measured 6.3e-7
       rel(cr - bc.double(), cr))
    # gelu backward: y = dy * gelu'(pre), act = gelu(pre)
    pre = randn(B * 4 * dim, g=g, scale=2.0)
    dy = randn(B * 4 * dim, g=g)
    y, act = sentinel(B * 4 * dim), sentinel(B * 4 * dim)
    call('cd_gelu_bwd', ptr(dy), ptr(pre), C.c_int64(pre.numel()), ptr(y), ptr(act), stream())
    p64 = pre.double().requires_grad_(True)
    a64 = F.gelu(p64)
    gr, = torch.autograd.grad(a64, p64, dy.double())
    ck('gelu_bwd y', rel(y, gr), 1.5e-7,         # measured 4.9e-8
       rel(dy.double() * torch.sigmoid(1.702 * p64.detach()), gr))
    ck('gelu_bwd act', rel(act, a64.detach()), 1.1e-7,       # measured 3.6e-8
       rel(F.gelu(p64.detach(), approximate='tanh') * 1.001, a64.detach()))
    # small GEMMs: C (+)= op(A) op(B); op(X) = X^T when trans
    dcond = randn(B, sumC, g=g)
    cases = [('dW_mlp = dcond^T gt', 1, 0, 64, dim, B, 1), ('dgt = dcond Wc (split-K)', 0, 0, B, dim, sumC, 0),
             ('dgt accumulate (split-K)', 0, 0, B, dim, sumC, 1), ('A B^T', 0, 1, B, 4 * dim, dim, 1),
             ('A^T B^T split-K', 1, 1, 8, 16, 1024, 1)]
    for name, ta, tb, M, N, K, accum in cases:
        A = randn(*((K, M) if ta else (M, K)), g=g)
        Bm = randn(*((N, K) if tb else (K, N)), g=g)
        c0 = randn(M, N, g=g)
        cm = c0.clone()
        call('cd_small_gemm', ptr(A), A.shape[1], ta, ptr(Bm), Bm.shape[1], tb, ptr(cm), N, M, N, K, accum, stream())
        prod = (A.double().t() if ta else A.double()) @ (Bm.double().t() if tb else Bm.double())
        ref = prod + (c0.double() if accum else 0)
        ks = K - max(1, K // 8)                                                       # control: the last K slice dropped
        short = (A.double().t() if ta else A.double())[:, :ks] @ (Bm.double().t() if tb else Bm.double())[:ks] + (c0.double() if accum else 0)
        ck('small_gemm %s' % name, rel(cm, ref), 1.1e-6, rel(short, ref))      # measured <= 3.7e-7
    ck.done()


@pytest.mark.parametrize('step', [1, 1000])
def test_fused_adam_ema_against_fp64(c3, step):
    """cd_adam_ema_step over a buffer of the engine's flat size, ema_mode 0 / 1 / 2 and grad_scale 0.5, against the Adam formula
    of torch.optim.Adam (and the EMA of DB:73-81) in fp64, element by element"""
    ck = Checks('adam[step=%d]' % step)
    c3.eng.flatten_params()
    n = c3.eng.flat_param.numel()
    lr, eps, gs = 1e-3, 1e-8, 0.5
    b1, b2, beta = F32(0.9), F32(0.999), F32(0.995)          # the kernel receives the betas as fp32 (see F32)
    for mode in (0, 1, 2):
        g = gen(700 + mode + step)
        p0 = randn(n, g=g, scale=0.05)
        gr = randn(n, g=g, scale=0.01)
        gr[::97] = 0
        m0 = randn(n, g=g, scale=0.005) if step > 1 else torch.zeros(n, device=DEV)
        v0 = randn(n, g=g, scale=1e-4).square() if step > 1 else torch.zeros(n, device=DEV)
        e0 = p0 + randn(n, g=g, scale=1e-3)
        p, m, v, e = p0.clone(), m0.clone(), v0.clone(), e0.clone()
        call('cd_adam_ema_step', ptr(p), ptr(gr), ptr(m), ptr(v), ptr(e), C.c_int64(n), C.c_float(lr), C.c_float(b1),
             C.c_float(b2), C.c_float(eps), step, mode, C.c_float(beta), C.c_float(gs), stream())
        g64 = gr.double() * gs
        m64 = b1 * m0.double() + (1 - b1) * g64
        v64 = b2 * v0.double() + (1 - b2) * g64 * g64
        bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
        upd = lr / bc1 * m64 / (v64.sqrt() / math.sqrt(bc2) + eps)
        p64 = p0.double() - upd
        wrong = p0.double() - lr * m64 / (v64.sqrt() + eps)                             # control: no bias correction
        scale_p = p0.double().abs() + upd.abs() + lr
        key = 'mode %d' % mode
        ck(key + ' param', ((p.double() - p64).abs() / scale_p).max().item(), 9e-7,     # measured <= 3.0e-7
           ((wrong - p64).abs() / scale_p).max().item())
        ck(key + ' exp_avg', rel(m, m64), 7.5e-8,       # measured 2.6e-8
           rel(m64 - (1 - b1) * g64 * 0.5, m64))
        ck(key + ' exp_avg_sq', rel(v, v64), 1.2e-7,    # measured 3.9e-8
           rel(b2 * v0.double() + (1 - b2) * gr.double().square(), v64))
        if mode == 0:
            ck.require(key + ': EMA untouched', bool(torch.equal(e, e0)))
        else:
            eref = p.double() if mode == 1 else e0.double() * beta + (1 - beta) * p.double()
            ewrong = p0.double() if mode == 1 else p.double() * beta + (1 - beta) * e0.double()
            sc = e0.double().abs() + p.double().abs() + lr
            ck(key + ' ema', ((e.double() - eref).abs() / sc).max().item(), 3.5e-7,     # measured <= 1.1e-7
               ((ewrong - eref).abs() / sc).max().item())
        del p0, gr, m0, v0, e0, p, m, v, e, g64, m64, v64, upd, p64, wrong, scale_p
        gc.collect()
        torch.cuda.empty_cache()
    ck.done()


# ==========================================================================================================================
# B. the config-3 training step end to end
# ==========================================================================================================================
def _microbatch(c3, x, t, scale):
    loss = c3.gd.p_losses(x, t)
    (loss * scale).backward()
    return loss.detach()


def test_fp32_path_step_at_128_matches_fp64_autograd(c3):
    """B1: the fp32 CUDA-core convolutions (CONV_SIMT), B = 2 at 128^2: q_sample, the L2 loss and all 238 parameter gradients
    against fp64 autograd of the oracle"""
    from cold_diffusion_models_b200.ops import CONV_SIMT, CONV_TC
    ck = Checks('B1 fp32 path')
    x, t = c3.xs[0][:2], c3.ts[0][:2]
    c3.tr.opt.zero_grad()
    c3.eng.conv_impl = CONV_SIMT
    try:
        xt = c3.gd.q_sample(x, t)
        xt64 = blur_per_image(c3.oracle, x.double(), t)
        ck('q_sample max abs', maxabs(xt, xt64), 3.5e-7,      # measured 1.2e-7
        maxabs(xt64, blur_per_image(c3.oracle, x.double(), torch.where(t < 199, t + 1, t - 1))))
        loss = _microbatch(c3, x, t, 1.0)
        torch.cuda.synchronize()
    finally:
        c3.eng.conv_impl = CONV_TC
    eg = engine_grads(c3.unet)
    c3.tr.opt.zero_grad()
    sd = c3.unet.state_dict()
    ref, lref, _ = ref_step(sd, x, xt64, t, 2 * 3 * 128 * 128, chunk=2)
    one, _, _ = ref_step(sd, x[:1], xt64[:1], t[:1], 2 * 3 * 128 * 128, chunk=1)
    ck('loss', abs(loss.item() - lref) / lref, 4.5e-7)        # measured 1.6e-7
    errs = grad_errors(eg, ref)
    ctrl = grad_errors(eg, {k: ref[k] - one[k] for k in ref})
    ck.require('238 parameter gradients', len(errs) == 238)
    med, p90, worst = stats(errs)
    _METRICS['B1 fp32 path::worst parameters'] = [(e, n) for e, n in errs[-5:]]
    ck('grad median', med, 1.8e-6, stats(ctrl)[0])          # measured 6.2e-7 (control 0.96)
    ck('grad worst', worst, 4e-6, stats(ctrl)[0])            # measured 1.4e-6
    ck.done()


def test_batch_independence_of_the_tensor_core_gradient(c3):
    """B3: the gradient of one micro-batch of 32 in a single pass against the sum of the same engine's gradients over 16 passes
    of 2 images (different wave counts, kernel choices and weight-gradient K-splits; same arithmetic per image)"""
    ck = Checks('B3 batch independence')
    x, t = c3.xs[0], c3.ts[0]
    c3.tr.opt.zero_grad()
    _microbatch(c3, x, t, 1.0)
    one = c3.eng.flat_grad.clone()
    c3.tr.opt.zero_grad()
    parts = []
    for i in range(0, 32, 2):
        _microbatch(c3, x[i:i + 2], t[i:i + 2], 2 / 32)
        if i == 28:
            parts.append(c3.eng.flat_grad.clone())      # 15 of the 16 pairs: the negative control
    many = c3.eng.flat_grad.clone()
    c3.tr.opt.zero_grad()
    eg1, eg16, eg15 = {}, {}, {}
    for n_, (off, k) in c3.eng._offsets.items():
        eg1[n_], eg16[n_], eg15[n_] = one[off:off + k], many[off:off + k], parts[0][off:off + k]
    errs = grad_errors(eg16, eg1)
    ctrl = grad_errors(eg15, eg1)
    med, p90, worst = stats(errs)
    _METRICS['B3 batch independence::worst parameters'] = [(e, n) for e, n in errs[-5:]]
    ck('median', med, 1.2e-4, stats(ctrl)[0])                # measured 4.0e-5 (control 6.8e-2), 25x below the fp64 comparison
    ck('worst', worst, 5e-4, stats(ctrl)[0])                 # measured 1.7e-4
    ck.done()


@pytest.fixture(scope='module')
def step1(c3):
    """B2 + B4: two micro-batches of 32 on the default tensor-core path (loss / 2 each into the same flat gradient), their fp64
    references, then the fused Adam + EMA step with everything it reads snapshotted"""
    s = Config3()
    tr, eng = c3.tr, c3.eng
    tr.opt.zero_grad()
    sd0 = {k: v.detach().clone() for k, v in c3.unet.state_dict().items()}
    N = 32 * 3 * 128 * 128
    s.checks = []
    s.losses = []
    refs = []
    for mb in range(2):
        x, t = c3.xs[mb], c3.ts[mb]
        xt = c3.gd.q_sample(x, t)
        xt64 = blur_per_image(c3.oracle, x.double(), t)
        with torch.no_grad():
            y = c3.unet(xt, t)
            c3.gd.loss_type = 'l1'
            l1 = c3.gd.p_losses(x, t).item()
            c3.gd.loss_type = 'l2'
        loss = _microbatch(c3, x, t, 0.5)
        ref, lref, yref = ref_step(sd0, x, xt64, t, 2 * N)
        s.checks.append(('x_t mb%d max abs' % mb, maxabs(xt, xt64), 3.5e-7,                    # measured 1.2e-7
                         maxabs(xt64, blur_per_image(c3.oracle, x.double(), torch.where(t < 199, t + 1, t - 1)))))
        s.checks.append(('output mb%d' % mb, rel(y, yref), 1.3e-3,                                  # measured 4.6e-4
                          rel(y.roll(1, 0), yref)))
        s.checks.append(('l2 loss mb%d' % mb, abs(loss.item() - 2 * lref) / (2 * lref), 5e-5, None))       # measured 1.8e-5
        l1ref = (x.double() - yref).abs().mean().item()
        s.checks.append(('l1 loss mb%d' % mb, abs(l1 - l1ref) / l1ref, 2e-5,                 # measured 6.8e-6
                          abs(l1ref * 0.99 - l1ref) / l1ref))
        refs.append(ref)
        del xt64, y, yref
    torch.cuda.synchronize()
    s.eng_g = engine_grads(c3.unet)
    s.ref = {k: refs[0][k] + refs[1][k] for k in refs[0]}
    one, _, _ = ref_step(sd0, c3.xs[0][:1], blur_per_image(c3.oracle, c3.xs[0][:1].double(), c3.ts[0][:1]), c3.ts[0][:1], 2 * N, chunk=1)
    s.ctrl_leave_one = {k: s.ref[k] - one[k] for k in s.ref}
    s.ctrl_second = refs[1]
    del refs, one
    # ---- B4: the optimizer step on what it reads
    ema_eng = c3.tr._ema_unet.engine
    s.p0, s.g0 = eng.flat_param.clone(), eng.flat_grad.clone()
    s.m0, s.v0, s.e0 = tr.opt.m.clone(), tr.opt.v.clone(), ema_eng.flat_param.clone()
    s.t0 = tr.opt.t
    tr.opt.step(ema_mode=2, ema_beta=0.995, grad_scale=1.0)
    tr.opt.zero_grad()
    torch.cuda.synchronize()
    s.sd0 = sd0
    yield s
    del s


def test_tensor_core_step_at_the_bench_shape_matches_fp64(c3, step1):
    """B2: default tensor-core path, B = 32 x 2 micro-batches: x_t, the network output and the loss of each micro-batch, and every
    parameter gradient after both backwards against the fp64 reference of the 64 images"""
    ck = Checks('B2 tensor-core step')
    for c in step1.checks:
        ck(*c)
    errs = grad_errors(step1.eng_g, step1.ref)
    med, p90, worst = stats(errs)
    c1 = stats(grad_errors(step1.eng_g, step1.ctrl_leave_one))
    c2 = stats(grad_errors(step1.eng_g, step1.ctrl_second))
    _METRICS['B2 tensor-core step::worst parameters'] = [(e, n) for e, n in errs[-10:]]
    _METRICS['B2 tensor-core step::p90'] = p90
    # measured median 1.02e-3, p90 1.28e-3, worst 2.19e-3 (ups.0.2.fn.fn.to_out.weight); one image left out: median 1.6e-2
    ck('grad median', med, 3e-3, c1[0])
    ck('grad worst', worst, 5e-3, c1[0])
    ck('grad median vs second micro-batch alone', med, 3e-3, c2[0])          # control 1.0
    ck.done()


def test_optimizer_step_matches_torch_adam_in_fp64(c3, step1):
    """B4: the fused Adam + EMA step of the training step against torch.optim.Adam in float64 and the EMA lerp, on the snapshot of
    flat_param / flat_grad / m / v / EMA it read"""
    ck = Checks('B4 optimizer')
    eng, opt = c3.eng, c3.tr.opt
    p = step1.p0.double().clone().requires_grad_(True)
    p.grad = step1.g0.double()
    ta = torch.optim.Adam([p], lr=LR, betas=(F32(0.9), F32(0.999)), eps=1e-8)
    assert step1.t0 == 0
    ta.step()
    pref = p.detach()
    st = ta.state[p]
    d_k = eng.flat_param.double() - step1.p0.double()
    d_r = pref - step1.p0.double()
    wrong = LR * 0.1 * p.grad / (0.001 ** 0.5 * p.grad.abs() + 1e-8)                  # control: no bias correction
    ck('param update (|err| / lr)', (d_k - d_r).abs().max().item() / LR, 1.8e-4,      # measured 6.0e-5 (fp32 rounding of p)
       (wrong + d_r).abs().max().item() / LR)
    ck('exp_avg', rel(opt.m, st['exp_avg']), 7.5e-8,          # measured 2.5e-8
       rel(step1.g0, st['exp_avg']))
    ck('exp_avg_sq', rel(opt.v, st['exp_avg_sq']), 1.2e-7,    # measured 4.1e-8
       rel(step1.g0.double().square(), st['exp_avg_sq']))
    ema = c3.tr._ema_unet.engine.flat_param.double()
    beta = F32(0.995)
    eref = step1.e0.double() * beta + (1 - beta) * eng.flat_param.double()
    ewrong = step1.e0.double() * (1 - beta) + beta * eng.flat_param.double()
    sc = eref.abs().clamp_min(LR)
    ck('ema', ((ema - eref).abs() / sc).max().item(), 3.5e-7,       # measured 1.2e-7
       ((ewrong - eref).abs() / sc).max().item())
    ck.require('packs marked stale', eng._dirty)
    ck.done()


def test_gradient_after_the_step_follows_the_new_weights(c3, step1):
    """B5: the gradient of a third micro-batch at the updated weights against the fp64 reference there (stale forward or
    data-gradient packs would give the gradient at the old weights: the control)"""
    ck = Checks('B5 after the step')
    N = 32 * 3 * 128 * 128
    x, t = c3.xs[2], c3.ts[2]
    c3.tr.opt.zero_grad()
    _microbatch(c3, x, t, 0.5)
    torch.cuda.synchronize()
    eg = engine_grads(c3.unet)
    c3.tr.opt.zero_grad()
    xt64 = blur_per_image(c3.oracle, x.double(), t)
    sd1 = {k: v.detach().clone() for k, v in c3.unet.state_dict().items()}
    ref, _, _ = ref_step(sd1, x, xt64, t, 2 * N)
    errs = grad_errors(eg, ref)
    del ref
    gc.collect()
    old, _, _ = ref_step(step1.sd0, x, xt64, t, 2 * N)
    ctrl = grad_errors(eg, old)
    med, p90, worst = stats(errs)
    _METRICS['B5 after the step::worst parameters'] = [(e, n) for e, n in errs[-10:]]
    ck('grad median', med, 1.7e-3, stats(ctrl)[0])           # measured 5.7e-4 (control: old weights, 1.4)
    ck('grad worst', worst, 2.8e-3, stats(ctrl)[-1])         # measured 9.3e-4
    ck.done()


def test_ema_sampling_with_cuda_graph_matches_fp64_oracle(c3, step1):
    """B6: `ema.sample(batch_size=32, img, t=3)` with CUDA-graph replay (the benchmark's warm-up: cd_blur_step_down at S = 128
    inside a captured graph) against DeblurOracle.sample(t=3) in fp64 with the EMA weights"""
    ck = Checks('B6 sampling')
    ema = c3.tr.ema_model
    x = c3.xs[1]
    eng = ema.denoise_fn.engine
    eng.enable_cuda_graph(True)
    try:
        with torch.no_grad():
            xt, dr, img = ema.sample(batch_size=32, img=x, t=3)
        torch.cuda.synchronize()
    finally:
        eng.enable_cuda_graph(False)
    sd = {k: v.detach().to(DEV, F64) for k, v in ema.denoise_fn.state_dict().items()}
    fn = lambda a, s: UO.unet_forward(sd, a, s.to(a.device, F64))
    kw = dict(image_size=128, channels=3, timesteps=200, kernel_std=0.01, kernel_size=15, blur_routine='Exponential_reflect')
    outs = {}
    for routine in ('x0_step_down', 'default'):
        o = DO.DeblurOracle(fn, sampling_routine=routine, **kw)
        o.kernels2d = [k.double().cuda() for k in o.kernels2d]
        res = [o.sample(batch_size=8, img=x[i:i + 8].double(), t=3) for i in range(0, 32, 8)]
        outs[routine] = [torch.cat([r[j] for r in res]) for j in range(3)]
    r, w = outs['x0_step_down'], outs['default']
    ck('x_t', rel(xt, r[0]), 3.5e-7,                    # measured 1.2e-7
       rel(xt, blur_per_image(c3.oracle, x.double(), torch.full((32,), 1))))
    ck('direct reconstruction', rel(dr, r[1]), 1.6e-3, rel(dr.roll(1, 0), r[1]))      # measured 5.4e-4
    ck('sample (Algorithm 2)', rel(img, r[2]), 1.9e-3, rel(w[2], r[2]))       # measured 6.3e-4
    ck.done()
