"""Data-parallel training on the GPU: the gradient all-reduce that `Trainer._accumulate` overlaps with the backward, and the
training step of two ranks against one process and against float64.

Above one process, the engine's backward declares suffixes of the flat gradient final as it walks the network
(`_grads_ready_from`: after the mid block, after `downs.3`, after `downs.2`) and the trainer all-reduces each one while later
kernels keep writing other parts of the same buffer; what is left, `[0, low)` (the time MLP and the `*.mlp.1.*` conditioning
projections, which the layout puts first), is reduced at the end.  A mark placed before the last write into its range, a
weight-gradient launch moved after a mark or a parameter group laid out inside an already-reduced range would leave the
replicas with partly reduced gradients, and nothing in the images/s would show it.

A. The ready marks on the real engine, in one process: the hook is installed by hand as `_accumulate` installs it on the last
   micro-batch and takes a stream-ordered snapshot of every declared range.  Each snapshot must equal the final gradient bit
   for bit (within one run, so the float atomics of the depthwise weight gradient cannot differ), and the ranges plus
   `[0, low)` must tile the buffer.  Control: the first mark moved down to the coarsest trainable down level, whose backward
   has not run yet.
B. Two ranks on one GPU over gloo (whose CUDA all-reduce waits on an event of the caller's stream, as NCCL does): the
   benchmark's step, `Unet(64, (1, 2, 4, 8))` at 128², two micro-batches of 32 per rank.  The all-reduce inputs are recorded
   on each rank; the replicas must agree bit for bit, the reduced gradient must be the sum of the inputs bit for bit and
   match the same four micro-batches run in one process, the float64 gradient of the global loss, and torch's float64 Adam.
C. B on two GPUs over NCCL, the backend of the benchmark (skipped when fewer than two devices are visible).
D. The DDPM `Model` (32², B = 32 per rank, no dropout) on two gloo ranks: no overlapped ranges, one all-reduce of the
   whole buffer.

Every metric is paired with a negative control (a wrong reference) that must land at least 10x past its bound; bit-for-bit
requirements are exact.  Every bound is at most 3x the value measured on an H100 80GB HBM3 (700 W), which is in the comment
beside it.  Set COLDDIFF_TEST_METRICS=<file> to write all values and controls as JSON.

Measured on that card: the file runs in about 85 s, of which each two-rank spawn takes about 16 s.  Each of the two C3
processes sharing the GPU peaks at 14.5 GiB of device memory (torch.cuda.max_memory_allocated), each `Model` process at
3.4 GiB and the parent process at 17.8 GiB.  The float64 reference of check B4 covers all four micro-batches (128 images at
128²) and takes 8 s, so it runs at the benchmark's A = 2."""
import contextlib
import datetime
import io
import os
import sys
import time

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import unet_oracle as UO
from test_config3_step_gpu import (Checks, _metrics_file, _free_between_tests, _METRICS, C3, LR, F32, rel,  # noqa: F401
                                   ref_step, grad_errors, stats, blur_oracle, blur_per_image)
from test_ddp_gloo import _free_port
from test_model_large_gpu import NET

pytestmark = pytest.mark.gpu

DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT = datetime.timedelta(minutes=4)     # a rank stuck in a collective raises instead of hanging the test


class Checks10(Checks):
    """Checks whose negative controls must land at least 10x past their bounds"""

    def __call__(self, name, value, bound, control=None):
        super().__call__(name, value, bound, control)
        if control is not None and not float(control) > 10 * bound:
            self.fails.append('%s: negative control %.3e is not 10x past the bound %.3e' % (name, control, bound))


def _quiet():
    return contextlib.redirect_stdout(io.StringIO())


def _per_param(eng, flat):
    """flat gradient -> {name: slice} in the engine's layout (packed dense-conv slices on both sides of a comparison)"""
    return {n: flat[off:off + k] for n, (off, k) in eng._offsets.items()}


# ==========================================================================================================================
# A. ready marks on the real engine, one process
# ==========================================================================================================================
# (id, Unet keyword arguments, image side, batch, frozen-parameter predicate, input gradient requested)
A_CASES = [
    ('c3-128', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3), 128, 32, None, False),
    ('32-c3', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3), 32, 32, None, False),
    ('32-c1', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=1), 32, 32, None, False),
    ('mults124-64', dict(dim=64, dim_mults=(1, 2, 4), channels=3), 64, 16, None, False),
    ('no-time-emb', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3, with_time_emb=False), 32, 32, None, False),
    ('residual-dx', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3, residual=True), 32, 32, None, True),
    ('frozen-downs3', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3), 32, 32, lambda n: n.startswith('downs.3.'), False),
    ('frozen-ups', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3), 32, 32, lambda n: n.startswith('ups.'), False),
    ('frozen-time-mlp', dict(dim=64, dim_mults=(1, 2, 4, 8), channels=3), 32, 32, lambda n: n.startswith('time_mlp.'), False),
]


def _a_inputs(cfg, S, B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for _ in range(2):
        x = torch.rand(B, cfg['channels'], S, S, generator=g, device=DEV) * 2 - 1
        t = torch.randint(0, 200, (B,), generator=g, device=DEV)
        gy = torch.randn(B, cfg['channels'], S, S, generator=g, device=DEV) / (B * S * S) ** 0.5
        out.append((x, t, gy))
    return out


def _two_micro_batches(net, batches, need_dx, shift_first_mark_to=None):
    """micro-batch 0 without the hook, micro-batch 1 with it, as Trainer._accumulate runs them at A = 2
    -> (hook calls [(lo, hi, snapshot)], final flat gradient, flat gradient after micro-batch 0).
    shift_first_mark_to: a down group whose start the first mark (`ups.0`) is moved to, declaring it final before its backward"""
    eng = net.engine
    if getattr(eng, 'flat_grad', None) is not None:
        eng.flat_grad.zero_()
    calls, after0 = [], None
    gs = getattr(eng, '_group_start', None)
    saved = None
    if shift_first_mark_to is not None:
        saved = gs['ups.0']
        gs['ups.0'] = gs[shift_first_mark_to]
    try:
        for i, (x, t, gy) in enumerate(batches):
            xin = x.clone().requires_grad_(need_dx)
            y = net(xin, t) if net.time_mlp is not None else net(xin)
            if i == 1:
                def hook(lo, hi):
                    calls.append((lo, hi, eng.flat_grad[lo:hi].clone()))      # stream-ordered: what an all-reduce issued now reads
                eng._ready_mark = eng._grad_total
                eng.grad_ready_hook = hook
            try:
                (y * gy).sum().backward()
            finally:
                eng.grad_ready_hook = None
            if need_dx:
                assert xin.grad is not None and xin.grad.shape == x.shape
            if i == 0:
                after0 = eng.flat_grad.clone()
        torch.cuda.synchronize()
    finally:
        if saved is not None:
            gs['ups.0'] = saved
    return calls, eng.flat_grad.clone(), after0


@pytest.mark.parametrize('case', A_CASES, ids=[c[0] for c in A_CASES])
def test_ready_marks_are_sound_on_the_engine(case):
    """every range the backward declares final equals, bit for bit, the gradient the backward leaves at the end; the ranges and
    `[0, low)` tile the buffer; batched repacks disable the hook without changing the gradient"""
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200 import engine as E
    name, cfg, S, B, frozen, need_dx = case
    ck = Checks10('ready marks %s' % name)
    torch.manual_seed(11)
    with _quiet():
        net = cdm.Unet(**cfg).to(DEV)
    if frozen is not None:
        for n, p in net.named_parameters():
            if frozen(n):
                p.requires_grad_(False)
    batches = _a_inputs(cfg, S, B, seed=S + B + len(name))
    calls, final, after0 = _two_micro_batches(net, batches, need_dx)
    eng = net.engine
    total, gs = eng._grad_total, eng._group_start
    nd = len(eng.levels_down)
    # ---- the ranges: non-empty, descending, contiguous from the end; with [0, low) they cover the buffer once
    rng = [(lo, hi) for lo, hi, _ in calls]
    want = [(gs['ups.0'], total)] + [(gs['downs.%d' % i], gs['downs.%d' % (i + 1)] if i + 1 < nd else gs['ups.0'])
                                     for i in reversed(range(2, nd))]
    ck.require('hook called at every mark: %r, expected %r' % (rng, want), rng == want)
    ck.require('ranges non-empty, descending, contiguous from the end: %r' % rng,
               bool(rng) and rng[0][1] == total and all(lo < hi for lo, hi in rng) and all(a[0] == b[1] for a, b in zip(rng, rng[1:])))
    low = rng[-1][0] if rng else total
    cover = torch.zeros(total, dtype=torch.int32)
    cover[:low] += 1
    for lo, hi in rng:
        cover[lo:hi] += 1
    ck.require('ranges + [0, low) cover the buffer exactly once', bool((cover == 1).all()))
    late = [n for n, _ in net.named_parameters() if n.startswith('time_mlp.') or '.mlp.1.' in n]
    ck.require('end-of-backward gradients lie in [0, low)', all(eng._offsets[n][0] + eng._offsets[n][1] <= low for n in late))
    if not late:
        ck.require('no time embedding: the first down group starts the buffer', gs['downs.0'] == 0)
    # ---- every declared range holds its final values when it is declared
    changed = sum(int((snap != final[lo:hi]).sum()) for lo, hi, snap in calls)
    declared = sum(hi - lo for lo, hi in rng)
    ck.require('every snapshot equals the final gradient bit for bit (%d of %d elements differ)' % (changed, declared), changed == 0)
    # control: the first mark moved to the coarsest down level that has a trainable parameter -- its range is snapshotted
    # before that level's backward ran
    train_names = [n for n, p in net.named_parameters() if p.requires_grad]
    k = max(i for i in range(nd) if any(n.startswith('downs.%d.' % i) for n in train_names))
    c_calls, c_final, _ = _two_micro_batches(net, batches, need_dx, shift_first_mark_to='downs.%d' % k)
    lo0, hi0 = gs['downs.%d' % k], gs['downs.%d' % (k + 1)] if k + 1 < nd else gs['ups.0']
    c_lo, _, c_snap = c_calls[0]
    trainable = torch.zeros(total, dtype=torch.bool, device=DEV)
    for n in train_names:
        off, kk = eng._offsets[n]
        trainable[off:off + kk] = True
    early = (c_snap[lo0 - c_lo:hi0 - c_lo] != c_final[lo0:hi0])[trainable[lo0:hi0]]
    # exact: one changed element gives a fraction of at least 1 / 4e7, above the bound
    ck('fraction of declared-final elements changed after the mark', changed / max(declared, 1), 1e-9,
       early.double().mean().item())
    if frozen is not None:
        ck.require('frozen slices stay zero', all(bool((final[off:off + kk] == 0).all())
                                                   for n, (off, kk) in eng._offsets.items() if frozen(n)))
    # ---- batched repacks: the reference-layout gradients are written at the end, so no range may be declared
    prev = E.batched_repack()
    E.batched_repack(True)
    try:
        b_calls, b_final, _ = _two_micro_batches(net, batches, need_dx)
    finally:
        E.batched_repack(prev)
    ck.require('batched repack: hook never called (%d calls)' % len(b_calls), not b_calls)
    # The default path run twice (the control's run) differs by as much (median 5e-4, worst up to 7e-3 on the same inputs): the
    # weight gradients accumulate with float atomics.  Only the median is bounded; the worst parameters are recorded.
    sel = lambda flat: {n: v for n, v in _per_param(eng, flat).items() if n in train_names}
    ctrl = stats(grad_errors(sel(after0), sel(final)))                          # control: micro-batch 1 missing
    errs = grad_errors(sel(b_final), sel(final))
    _METRICS['ready marks %s::default path run twice (median, p90, worst)' % name] = stats(grad_errors(sel(c_final), sel(final)))
    _METRICS['ready marks %s::batched repack worst parameters' % name] = [(e, n) for e, n in errs[-3:]]
    # measured 4.2e-4 .. 5.8e-4 over the nine cases (control 0.61 .. 0.77)
    ck('batched repack vs the default path: median parameter', stats(errs)[0], 1.2e-3, ctrl[0])
    ck.done()


# ==========================================================================================================================
# B, C, D. two ranks
# ==========================================================================================================================
def _c3_diffusion(seed):
    """the benchmark's network and blur diffusion (the `c3` fixture of test_config3_step_gpu), weights from `seed`"""
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(0)
    with _quiet():
        unet = cdm.Unet(dim=C3['dim'], dim_mults=C3['dim_mults'], channels=C3['channels']).to(DEV)
        unet.load_state_dict(UO.make_unet_state_dict(64, (1, 2, 4, 8), 3, seed=seed))
        gd = cdm.GaussianDiffusion(unet, image_size=128, device_of_kernel='cuda', channels=3, timesteps=C3['timesteps'],
                                   loss_type='l2', kernel_std=C3['kernel_std'], kernel_size=C3['kernel_size'],
                                   blur_routine=C3['blur_routine'], train_routine='Final', sampling_routine=C3['sampling_routine'],
                                   discrete=False).to(DEV)
    return gd


def _model_diffusion(seed):
    """the DDPM Model of the CIFAR-10 driver without dropout, Special_6_routine blur, L1 loss"""
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(seed)
    with _quiet():
        m = cdm.Model(resolution=32, in_channels=3, out_ch=3, dropout=0.0, **NET).to(DEV)
        gd = cdm.GaussianDiffusion(m, image_size=32, device_of_kernel='cuda', channels=3, timesteps=50, loss_type='l1', kernel_std=0.1,
                                   kernel_size=3, blur_routine='Special_6_routine', train_routine='Final',
                                   sampling_routine='x0_step_down').to(DEV)
    return gd


NETS = {'c3': (_c3_diffusion, 128, (3, 4)), 'model': (_model_diffusion, 32, (5, 6))}      # builder, image side, seeds of ranks 0, 1


def _images(net, rank):
    """the two micro-batches of 32 images rank `rank` trains on"""
    S = NETS[net][1]
    g = torch.Generator().manual_seed(2000 + 10 * rank + S)
    return [(torch.rand(32, 3, S, S, generator=g) * 2 - 1).to(DEV) for _ in range(2)]


def _worker(rank, world, port, backend, out_dir, net):
    """one rank: the Trainer's optimizer step on this rank's two micro-batches, with the all-reduce inputs, the micro-batches'
    t, the gradient Adam reads and the optimizer state recorded to out_dir/rank<k>.pt"""
    for p in (ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests')):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank if backend == 'nccl' else 0)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=TIMEOUT)
    try:
        import cold_diffusion_models_b200 as cdm
        build, S, seeds = NETS[net]
        gd = build(seeds[rank])                           # the ranks start from different weights: the Trainer must broadcast
        with _quiet():
            tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=32, train_lr=LR, train_num_steps=10 ** 9,
                             gradient_accumulate_every=2, ema_decay=0.995, fp16=False,
                             results_folder=os.path.join(out_dir, 'results%d' % rank), dataset='synthetic')
        assert tr._world == world and tr._rank == rank
        eng, ema_eng = tr._unet.engine, tr._ema_unet.engine
        p0, e0 = eng.flat_param.clone(), ema_eng.flat_param.clone()
        base, total = eng.flat_grad.data_ptr(), eng.flat_grad.numel()
        ts, pre, snap = [], [], {}
        p_losses = gd.p_losses

        def record_t(x, t):
            ts.append(t.clone())
            return p_losses(x, t)

        all_reduce = torch.distributed.all_reduce

        def record_all_reduce(tensor, *a, **k):
            off = (tensor.data_ptr() - base) // 4
            if 0 <= off < total:
                pre.append((off, tensor.clone()))     # stream-ordered: the values this collective reads
            return all_reduce(tensor, *a, **k)

        step = tr.opt.step

        def snapshot_step(**kw):
            snap.update(grad=eng.flat_grad.clone(), kw=kw)
            step(**kw)

        gd.p_losses, tr.opt.step, torch.distributed.all_reduce = record_t, snapshot_step, record_all_reduce
        xs = _images(net, rank)
        torch.manual_seed(100 + rank)                     # GaussianDiffusion.forward draws t from the global generator
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        try:
            loss = tr.train_step(batches=xs)
            torch.cuda.synchronize()
        finally:
            torch.distributed.all_reduce = all_reduce
            tr.opt.step = step
            del gd.p_losses
        seconds = time.perf_counter() - t0
        cpu = lambda v: v.detach().cpu()
        out = dict(grad=cpu(snap['grad']), grad_scale=float(snap['kw'].get('grad_scale', 1.0)), ema_mode=int(snap['kw']['ema_mode']),
                   pre=[(o, cpu(v)) for o, v in pre], ts=[cpu(t) for t in ts], loss=float(loss.item()),
                   ranges=list(getattr(tr, 'overlapped_ranges', [])), has_ranges='overlapped_ranges' in vars(tr),
                   total=total, group_start=dict(getattr(eng, '_group_start', {})), offsets=dict(eng._offsets),
                   p0=cpu(p0), e0=cpu(e0), params=cpu(eng.flat_param), ema=cpu(ema_eng.flat_param), m=cpu(tr.opt.m),
                   v=cpu(tr.opt.v), opt_t=tr.opt.t, seconds=seconds, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
        torch.save(out, os.path.join(out_dir, 'rank%d.pt' % rank))
    finally:
        dist.destroy_process_group()


def _spawn(net, backend, out_dir):
    t0 = time.perf_counter()
    mp.spawn(_worker, args=(2, _free_port(), backend, str(out_dir), net), nprocs=2, join=True)
    runs = [torch.load(os.path.join(str(out_dir), 'rank%d.pt' % r)) for r in range(2)]
    for r, run in enumerate(runs):
        _METRICS['ranks %s %s::rank %d peak device memory GiB' % (net, backend, r)] = run['peak_gib']
        _METRICS['ranks %s %s::rank %d train_step seconds' % (net, backend, r)] = run['seconds']
    _METRICS['ranks %s %s::spawn seconds' % (net, backend)] = time.perf_counter() - t0
    return runs


_SINGLE = {}


def _single_process(net, runs):
    """the four micro-batches of both ranks, with the t each rank drew, run in this process on the engine from rank 0's
    weights -> (rank 0's gradient, rank 1's gradient), each the sum of loss / 2 over its two micro-batches (cached on the t)"""
    key = (net,) + tuple(tuple(t.tolist()) for run in runs for t in run['ts'])
    if key not in _SINGLE:
        gd = NETS[net][0](NETS[net][2][0])
        core = gd.denoise_fn
        eng = core.engine
        eng.flatten_params()
        out = []
        for r in range(2):
            eng.flat_grad.zero_()
            for x, t in zip(_images(net, r), runs[r]['ts']):
                (gd.p_losses(x, t.to(DEV)) / 2).backward()
            out.append(eng.flat_grad.double().cpu())
        torch.cuda.synchronize()
        _SINGLE[key] = (out, {k: v.detach().cpu() for k, v in core.state_dict().items()}, eng.flat_param.cpu())
        del gd, core, eng
    return _SINGLE[key]


def _assembled(run):
    """this rank's all-reduce inputs placed at their offsets -> (flat gradient, per-element count of collectives covering it)"""
    g = torch.zeros(run['total'])
    cover = torch.zeros(run['total'], dtype=torch.int32)
    for off, v in run['pre']:
        g[off:off + v.numel()] = v
        cover[off:off + v.numel()] += 1
    return g, cover


def _check_replicas(ck, runs, single, bounds):
    """checks 1 + 3: the ranks agree bit for bit, the reduced gradient is the sum of the two ranks' all-reduce inputs bit for bit,
    and every input / the mean gradient matches the single-process run"""
    r0, r1 = runs
    for k in ('grad', 'params', 'ema', 'm', 'v'):
        ck.require('ranks bit-identical: %s' % k, bool(torch.equal(r0[k], r1[k])))
    ck.require('both ranks took one optimizer step at the same grad_scale 1/2',
               r0['opt_t'] == r1['opt_t'] == 1 and r0['grad_scale'] == r1['grad_scale'] == 0.5)
    (g0, g1), _, p_single = single
    ck.require('rank 1 started from rank 0\'s broadcast weights', bool(torch.equal(r1['p0'], r0['p0'])) and
               bool(torch.equal(r0['p0'], p_single)))
    ck.require('EMA weights broadcast too', bool(torch.equal(r1['e0'], r0['e0'])))
    pres = []
    for r, run in enumerate(runs):
        g, cover = _assembled(run)
        ck.require('rank %d: the collectives cover the flat gradient exactly once' % r, bool((cover == 1).all()))
        pres.append(g)
    ck.require('control: the ranks\' own gradients differ', not torch.equal(pres[0], pres[1]))
    # exact: the sum of two fp32 values is correctly rounded whichever rank adds
    ck.require('reduced gradient == sum of the two ranks\' all-reduce inputs, bit for bit', bool(torch.equal(r0['grad'], pres[0] + pres[1])))
    for r, (g, ref) in enumerate(zip(pres, (g0, g1))):
        ck('rank %d all-reduce input vs its micro-batches in one process' % r, rel(g, ref), bounds['input'], rel(g, (g0, g1)[1 - r]))
    mean = (g0 + g1) / 2
    red = r0['grad'].double() * r0['grad_scale']
    ck('reduced gradient x 1/2 vs the single-process mean', rel(red, mean), bounds['mean'], rel(pres[0].double() * 0.5, mean))
    ck('reduced gradient x 1/2 vs the single-process mean (control: the 1/2 missing)', rel(red, mean), bounds['mean'],
       rel(r0['grad'].double(), mean))


# ---- B + C: the benchmark's network ---------------------------------------------------------------------------------------
@pytest.fixture(scope='module', params=['gloo', 'nccl'])
def c3_ranks(request, tmp_path_factory):
    if request.param == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('NCCL needs one device per rank and %d CUDA device is visible; the gloo runs cover the '
                    'two-rank step on one device' % torch.cuda.device_count())
    runs = _spawn('c3', request.param, tmp_path_factory.mktemp('c3_' + request.param))
    yield request.param, runs
    del runs


C3_BOUNDS = dict(input=4e-6, mean=3e-6)            # measured 1.45e-6 (input), 1.01e-6 (mean)


def test_two_ranks_reduce_the_global_gradient(c3_ranks):
    """B1-B3: replicas bit-identical after the step, the overlapped ranges, the reduced gradient against the two ranks' inputs
    and against the same four micro-batches in one process"""
    backend, runs = c3_ranks
    ck = Checks10('c3 ranks %s' % backend)
    single = _single_process('c3', runs)
    _check_replicas(ck, runs, single, C3_BOUNDS)
    for r, run in enumerate(runs):
        rng, gs, total = run['ranges'], run['group_start'], run['total']
        want = [(gs['ups.0'], total), (gs['downs.3'], gs['ups.0']), (gs['downs.2'], gs['downs.3'])]
        ck.require('rank %d: overlapped ranges %r, expected %r' % (r, rng, want), rng == want)
        pre_offsets = [o for o, _ in run['pre']]
        ck.require('rank %d: the ranges are reduced in order, then [0, low)' % r, pre_offsets == [lo for lo, _ in want] + [0])
    ck.done()


@pytest.fixture(scope='module')
def c3_fp64():
    """float64 gradient of the global loss (both ranks' four micro-batches) at rank 0's weights, cached on the t"""
    cache = {}

    def get(runs):
        key = tuple(tuple(t.tolist()) for run in runs for t in run['ts'])
        if key not in cache:
            _, sd0, _ = _single_process('c3', runs)
            oracle = blur_oracle(128)
            x = torch.cat([x for r in range(2) for x in _images('c3', r)])
            t = torch.cat([t for run in runs for t in run['ts']]).to(DEV)
            xt64 = blur_per_image(oracle, x.double(), t)
            N = 32 * 3 * 128 * 128
            t0 = time.perf_counter()
            ref, _, _ = ref_step(sd0, x, xt64, t, 4 * N)
            cache[key] = ref
            _METRICS['c3 fp64 reference seconds'] = time.perf_counter() - t0
            del xt64
        return cache[key]
    yield get
    cache.clear()


def test_two_ranks_gradient_matches_fp64(c3_ranks, c3_fp64):
    """B4: the reduced gradient x 1/2 against float64 autograd of the global loss (mean over the 128 images of both ranks)"""
    backend, runs = c3_ranks
    ck = Checks10('c3 ranks %s fp64' % backend)
    ref = c3_fp64(runs)
    gd = _c3_diffusion(3)
    eng = gd.denoise_fn.engine
    eng.flatten_params()

    def by_name(flat):
        eng.flat_grad.copy_(flat.to(DEV, torch.float32))
        return {n: eng.G[n].detach().double().clone() for n in eng.G}
    r0 = runs[0]
    red = by_name(r0['grad'] * r0['grad_scale'])
    local = by_name(_assembled(r0)[0] * r0['grad_scale'])          # control: rank 0's own gradient in place of the reduced one
    noscale = by_name(r0['grad'])                                   # control: the 1/2 missing
    errs = grad_errors(red, ref)
    med, p90, worst = stats(errs)
    _METRICS['c3 ranks %s fp64::worst parameters' % backend] = [(e, n) for e, n in errs[-10:]]
    ck.require('238 parameter gradients', len(errs) == 238)
    c_local, c_noscale = stats(grad_errors(local, ref)), stats(grad_errors(noscale, ref))
    # measured median 1.03e-3, p90 1.28e-3, worst 3.56e-3 (downs.0.0.ds_conv.weight); controls: rank 0's gradient 0.50, no 1/2 1.0
    ck('grad median', med, 3e-3, c_local[0])
    ck('grad p90', p90, 3.8e-3, c_local[1])
    ck('grad worst', worst, 1e-2, c_local[0])
    ck('grad median (control: the 1/2 missing)', med, 3e-3, c_noscale[0])
    ck.done()


def test_two_ranks_optimizer_step_matches_torch_adam_in_fp64(c3_ranks):
    """B5: Adam + the EMA copy of step 0 on both ranks against torch.optim.Adam in float64 on the averaged gradient"""
    backend, runs = c3_ranks
    ck = Checks10('c3 ranks %s adam' % backend)
    r0 = runs[0]
    ck.require('step 0 copies the EMA (ema_mode 1)', r0['ema_mode'] == 1)
    p = r0['p0'].double().clone().requires_grad_(True)
    p.grad = r0['grad'].double() * r0['grad_scale']
    ta = torch.optim.Adam([p], lr=LR, betas=(F32(0.9), F32(0.999)), eps=1e-8)
    ta.step()
    st = ta.state[p]
    d_r = p.detach() - r0['p0'].double()
    d_k = r0['params'].double() - r0['p0'].double()
    wrong = -LR * 0.1 * p.grad / (0.001 ** 0.5 * p.grad.abs() + 1e-8)                  # control: no bias correction
    ck('param update (max |err| / lr)', (d_k - d_r).abs().max().item() / LR, 1.8e-4,    # measured 6.0e-5 (fp32 rounding of p)
       (wrong - d_r).abs().max().item() / LR)
    ck('exp_avg', rel(r0['m'], st['exp_avg']), 7.5e-8, rel(p.grad, st['exp_avg']))                 # measured 2.5e-8
    ck('exp_avg_sq', rel(r0['v'], st['exp_avg_sq']), 8.9e-8, rel(p.grad.square(), st['exp_avg_sq']))   # measured 3.0e-8
    ck.require('EMA == the new weights', bool(torch.equal(r0['ema'], r0['params'])))
    ck.done()


# ---- D: the DDPM Model ----------------------------------------------------------------------------------------------------
MODEL_BOUNDS = dict(input=2.2e-7, mean=1.8e-7)     # measured 7.7e-8 (input), 6.0e-8 (mean)


def test_model_two_gloo_ranks_take_one_all_reduce(tmp_path):
    """D: the Model's engine declares no ready ranges, so the step all-reduces the whole flat gradient once at the end; the
    replicas stay bit-identical and the reduced gradient matches the single-process sum"""
    ck = Checks10('model ranks gloo')
    runs = _spawn('model', 'gloo', tmp_path)
    for r, run in enumerate(runs):
        ck.require('rank %d: overlapped_ranges never set' % r, not run['has_ranges'])
        ck.require('rank %d: one all-reduce of the whole buffer' % r, [o for o, _ in run['pre']] == [0] and
                   run['pre'][0][1].numel() == run['total'])
    _check_replicas(ck, runs, _single_process('model', runs), MODEL_BOUNDS)
    ck.done()
