"""Time the blur degradation kernels and the deblurring model above 128².

    python tools/blur_shapes.py [--json FILE]
    python tools/blur_shapes.py --size 512 [--json FILE]

- cd_blur_apply (per-sample t) and cd_blur_step_down at S = 128, 256, 512, B = 32, C = 3: microseconds per launch, GFLOP/s
  (4 S^3 FLOP per plane and product), and the bytes the launch must move computed from the shapes, with the bound this implies.
  S = 128 is the one-CTA-per-plane kernel; above it the row-strip kernel, which reads X and A_t from L2 once per 32-row strip.
- One training step of `Unet(64, (1, 2, 4, 8))` at 256² (B = 8, 16 and 32, one micro-batch, Adam + EMA): images/s and the
  peak device memory of the step, each batch size in a process of its own.
- One reverse step of `sample` (x0_step_down) at the same size and batch.
- With --size 512: only the training step and the reverse step at 512², B = 1, 2, 4, 8, 10 and 12 (the kernels are skipped).
  The reverse step runs in the same process as the training step, as in a Trainer that samples while it trains.  A batch
  size whose training step runs out of device memory is reported as not fitting, and the larger ones are not tried.  Then
  the largest batch that trains and samples in one process runs once more with gradient_accumulate_every = 2 (twice the
  images per optimizer step).

Every number is printed with the card name and power limit read in the same run.  A run without a GPU stops."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import cold_diffusion_models_b200 as cdm  # noqa: E402
from cold_diffusion_models_b200._lib import call, ptr, stream  # noqa: E402
from cold_diffusion_models_b200.degradation import build_blur_operators  # noqa: E402

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12          # H100 SXM data sheet (700 W): HBM3 bandwidth, dense FP32


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return name, pl


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps            # microseconds


def kernels(res):
    B, Cc, T = 32, 3, 200
    for S in (128, 256, 512):
        ops = build_blur_operators('Exponential_reflect', T, 15, 0.01, S)[0].cuda()
        x = torch.rand(B, Cc, S, S, device='cuda') * 2 - 1
        xt = torch.rand_like(x)
        out = torch.empty_like(x)
        t = torch.randint(0, T - 1, (B,), device='cuda')
        planes = B * Cc
        nstrip = 1 if S <= 128 else (S + 31) // 32
        for name, fn, products, planes_io in (
                ('cd_blur_apply', lambda: call('cd_blur_apply', ptr(x), ptr(out), ptr(ops), ptr(t), 0, B, Cc, S, T, 0, 0, stream()), 1, 2),
                ('cd_blur_step_down', lambda: call('cd_blur_step_down', ptr(xt), ptr(x), ptr(out), ptr(ops), 100, 99, B, Cc, S, T, 0,
                                                   stream()), 2, 3)):
            us = timed(fn, 50)
            flop = 4.0 * S ** 3 * planes * products
            hbm = 4.0 * S * S * planes * planes_io + 4.0 * S * S * B * products     # planes in/out + the operators of the batch
            # L2 -> SM: every CTA reads its plane and operator(s) (the strip kernel once per strip and product)
            l2 = 4.0 * S * S * planes * nstrip * 2 * products + 4.0 * S * S * planes
            t_fl, t_hbm = flop / FP32_FLOPS, hbm / HBM_BPS
            r = dict(kernel=name, S=S, B=B, C=Cc, us=us, gflops=flop / us / 1e3, hbm_bytes=hbm, l2_bytes=l2,
                     bound='fp32 compute' if t_fl > t_hbm else 'HBM', share_of_bound=max(t_fl, t_hbm) / (us * 1e-6))
            res['kernels'].append(r)
            print('%-18s S=%3d  %9.1f us  %8.0f GFLOP/s  HBM %6.1f MB  L2->SM %7.1f MB  bound: %s (%.0f%% of it)' % (
                name, S, us, r['gflops'], hbm / 1e6, l2 / 1e6, r['bound'], 100 * r['share_of_bound']))
        del ops, x, xt, out
        torch.cuda.empty_cache()


def model(res, S, B, A=1):
    """one batch size per process: the caching allocator and the engine's shape-keyed buffers of an earlier batch size would
    otherwise still be allocated and count towards this one's peak"""
    T = 200
    with contextlib.redirect_stdout(io.StringIO()):
        unet = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
        gd = cdm.GaussianDiffusion(unet, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1',
                                   kernel_std=0.01, kernel_size=15, blur_routine='Exponential_reflect',
                                   sampling_routine='x0_step_down').cuda()
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=2e-5, train_num_steps=10 ** 9,
                         gradient_accumulate_every=A, ema_decay=0.995, fp16=False, results_folder=tempfile.mkdtemp(),
                         dataset='synthetic')
    x = torch.rand(B, 3, S, S, device='cuda') * 2 - 1
    for _ in range(3):
        tr.train_step([x] * A)
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated() / 2 ** 30        # weights, gradients, Adam state, EMA copy, engine buffers
    torch.cuda.reset_peak_memory_stats()
    us = timed(lambda: tr.train_step([x] * A), 10)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    r = dict(B=B, S=S, accumulate=A, step_ms=us / 1e3, images_per_s=A * B / (us * 1e-6), peak_gib=peak, resident_gib=resident,
             reserved_gib=torch.cuda.max_memory_reserved() / 2 ** 30)
    ema = tr.ema_model
    img = gd.opt(x, T)
    step = torch.full((B,), T - 1, dtype=torch.long, device='cuda')

    def reverse():
        with torch.no_grad():
            ema._reverse_step(img, ema.denoise_fn(img, step), T)
    try:
        r['reverse_ms'] = timed(reverse, 10) / 1e3
        rev = '%.2f ms' % r['reverse_ms']
    except torch.cuda.OutOfMemoryError:
        # the EMA model's engine allocates its own forward buffers next to everything the training step keeps
        r['reverse_ms'], rev = None, 'out of device memory beside the training state'
    res['train'].append(r)
    print('train step %d^2 B=%2d x %d: %8.2f ms  %7.1f images/s  peak device memory %.2f GiB (%.2f GiB resident between steps, '
          '%.2f GiB reserved)  reverse step (x0_step_down) %s' % (S, B, A, us / 1e3, r['images_per_s'], peak, resident,
                                                                r['reserved_gib'], rev))


def measure(res, S, B, A):
    """one training step size in a fresh process -> False when it ran out of device memory"""
    with tempfile.NamedTemporaryFile(suffix='.json') as f:
        p = subprocess.run([sys.executable, os.path.abspath(__file__), '--size', str(S), '--batch', str(B), '--accumulate', str(A),
                            '--json', f.name], capture_output=True, text=True)
        sys.stdout.write(p.stdout)
        if p.returncode != 0:
            if 'OutOfMemoryError' not in p.stderr and 'out of memory' not in p.stderr:
                sys.exit(p.stderr)
            res['does_not_fit'] = dict(S=S, B=B, accumulate=A)
            print('train step %d^2 B=%2d x %d: out of device memory' % (S, B, A))
            return False
        res['train'] += json.load(open(f.name))['train']
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json')
    ap.add_argument('--size', type=int, default=256, choices=(256, 512), help='image side of the training step')
    ap.add_argument('--batch', type=int, help='measure the training step at this batch size only')
    ap.add_argument('--accumulate', type=int, default=1, help='gradient_accumulate_every of that step')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('blur_shapes: no CUDA device; nothing is measured')
    name, pl = card()
    print('card: %s, power limit %s' % (name, pl))
    res = dict(card=name, power_limit=pl, kernels=[], train=[])
    if a.batch:
        model(res, a.size, a.batch, a.accumulate)
    else:
        if a.size == 256:
            kernels(res)
        fits = None
        for B in ((8, 16, 32) if a.size == 256 else (1, 2, 4, 8, 10, 12)):
            if not measure(res, a.size, B, 1):
                break
            if res['train'][-1]['reverse_ms'] is not None:
                fits = B                    # the largest batch that trains and samples in one process
        if a.size == 512 and fits:
            measure(res, a.size, fits, 2)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
