"""Time guided restoration, `GaussianDiffusion.restore(y, s, weight=..., steps=K)`, against `sample(img=x, t=s, steps=K)` at
config 3: deblurring, Unet(64, (1, 2, 4, 8)), 128², B = 32, T = 200, Exponential_reflect blur, x0_step_down, s = 200,
K = 20 and 200.  Modes, each (mode, K) in a fresh process, with `engine.enable_cuda_graph(True)`:
  sample     sample(img=x, t=200, steps=K): the graphed forward and one update kernel per step
  restore0   restore(y, 200, weight=0, steps=K): the same loop (no backward, graphed forward)
  restore    restore(y, 200, weight=0.05, steps=K): eager autograd forward, input-only backward, the fused guidance kernels
Each row is the median of --iters whole calls after --warmup, CUDA events around each call, every call started from an idle
device.  "guidance kernels" is the device time of one step's cd_blur_guide_grad + cd_blur_guided_step, from CUDA events around
50 launches of each, and its share of the step.  "peak" is torch.cuda.max_memory_allocated over the timed calls.  Prints the
card and its power limit with the table.

usage: python tools/restore_timing.py [--iters 3] [--warmup 1] [--out timing.json]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))

from model_graph_timing import card, timed  # noqa: E402

S, B, T, s = 128, 32, 200, 200
RUNS = [(m, K) for K in (20, 200) for m in ('sample', 'restore0', 'restore')]
WEIGHT = 0.05


def kernel_ms(fn, n=50):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def run_one(mode, K, iters, warmup):
    import torch
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200._lib import call, ptr, stream
    import ctypes as C
    assert torch.cuda.is_available(), "restore_timing.py measures on a CUDA device"
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        net = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
        gd = cdm.GaussianDiffusion(net, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1',
                                   train_routine='Final', sampling_routine='x0_step_down', kernel_std=0.01, kernel_size=15,
                                   blur_routine='Exponential_reflect').cuda()
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.rand(B, 3, S, S, generator=g, device='cuda') * 2 - 1
    y = gd.opt(x, s)
    net.engine.enable_cuda_graph(True)
    if mode == 'sample':
        fn = lambda: gd.sample(batch_size=B, img=x, t=s, steps=K)
    else:
        w = 0.0 if mode == 'restore0' else WEIGHT
        fn = lambda: gd.restore(y, s, weight=w, steps=K)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms, host_ms = timed(fn, iters, warmup)
    peak = torch.cuda.max_memory_allocated()
    row = dict(mode=mode, K=K, ms=ms, host_ms=host_ms, ms_per_step=ms / K, peak_gib=peak / 2 ** 30)
    if mode == 'restore':
        a, b, gg, out = (torch.randn_like(x) for _ in range(4))
        ops = gd._ops_cum
        row['guide_grad_ms'] = kernel_ms(lambda: call('cd_blur_guide_grad', ptr(a), ptr(y), ptr(out), ptr(None), ptr(ops), s - 1,
                                                      B, 3, S, T, stream()))
        row['guided_step_ms'] = kernel_ms(lambda: call('cd_blur_guided_step', ptr(a), ptr(b), ptr(gg), C.c_float(WEIGHT), ptr(out),
                                                       ptr(ops), 99, 89, B, 3, S, T, stream()))
        row['step_down_ms'] = kernel_ms(lambda: call('cd_blur_step_down', ptr(a), ptr(b), ptr(out), ptr(ops), 99, 89, B, 3, S, T,
                                                     0, stream()))
        row['guidance_share'] = (row['guide_grad_ms'] + row['guided_step_ms']) / row['ms_per_step']
    net.engine.enable_cuda_graph(False)
    return [row]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--out', default=None)
    ap.add_argument('--run', default=None, help='run one (mode, K) in this process (internal), e.g. restore:20')
    ap.add_argument('--json', default=None, help='with --run: write its result here')
    a = ap.parse_args()
    if a.run:
        mode, K = a.run.split(':')
        with open(a.json, 'w') as f:
            json.dump(run_one(mode, int(K), a.iters, a.warmup), f)
        return
    rows = []
    for mode, K in RUNS:
        with tempfile.NamedTemporaryFile(suffix='.json') as f:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--run', '%s:%d' % (mode, K), '--json', f.name,
                                '--iters', str(a.iters), '--warmup', str(a.warmup)], capture_output=True, text=True)
            if p.returncode != 0:
                raise RuntimeError('%s:%d failed:\n%s' % (mode, K, p.stderr[-3000:]))
            with open(f.name) as fh:
                rows += json.load(fh)
    info = dict(card=card(), iters=a.iters, warmup=a.warmup, weight=WEIGHT, rows=rows)
    print('card (name, power limit, max SM clock): %s' % info['card'])
    print('| call | K | time | per step | host | peak memory |')
    print('|---|---|---|---|---|---|')
    for r in rows:
        print('| %s | %d | %.1f ms | %.2f ms | %.1f ms | %.2f GiB |' % (r['mode'], r['K'], r['ms'], r['ms_per_step'], r['host_ms'],
                                                                   r['peak_gib']))
    for r in rows:
        if 'guide_grad_ms' in r:
            print('K = %d: cd_blur_guide_grad %.1f us, cd_blur_guided_step %.1f us (cd_blur_step_down %.1f us), guidance share of '
                  'the step %.1f %%' % (r['K'], 1e3 * r['guide_grad_ms'], 1e3 * r['guided_step_ms'], 1e3 * r['step_down_ms'],
                                        100 * r['guidance_share']))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
