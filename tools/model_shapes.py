"""Time the DDPM `Model` at 256² and the GroupNorm kernels of its 256² level.

    python tools/model_shapes.py [--one-cta] [--json FILE]

- cd_groupnorm_fwd / cd_groupnorm_bwd (GroupNorm(32) + swish, with the time-conditioning row) on 256² planes, C = 128 and 256,
  B = 1, 8 and 32: microseconds per call with CUDA events, and the bytes a call must move (forward: x read twice, y written
  once; backward: x read three times, dy twice, dx written once) over that time.  Planes of this size take the split-plane
  kernels.  With --one-cta the same calls also run the one-CTA-per-image kernels (groupnorm_kernel / groupnorm_bwd_kernel),
  which the library keeps for planes of at most 128 x 128 pixels: the tool compiles elementwise.cu and model2_bwd.cu once more
  into a temporary directory with a launcher of its own, so the library itself has no switch for it.
- One training step of `Model(ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2, attn_resolutions=(16,))` in the deblurring
  GaussianDiffusion at 256² (one micro-batch, Adam + EMA) and one reverse step of `sample` (x0_step_down) of the EMA model,
  B = 1, 2, 4, 8, 16, ...: images/s and peak device memory, each batch size in a process of its own, until a batch size does
  not train and sample in one process.

Every number is printed with the card name and power limit read in the same run.  A run without a GPU stops."""
import argparse
import contextlib
import ctypes as C
import io
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import cold_diffusion_models_b200 as cdm  # noqa: E402
from cold_diffusion_models_b200._lib import call, ptr, stream  # noqa: E402

CSRC = os.path.join(ROOT, 'cold_diffusion_models_b200', 'csrc')
S = 256
NET = dict(ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2, attn_resolutions=(16,))

_PROBE = {'elementwise.cu': r'''
extern "C" int probe_gn_fwd(const float* x, int x_ld, int B, int HW, int C, int groups, const float* cond, int cond_ld,
                            const float* gamma, const float* beta, float eps, int swish, float* y, int y_ld, void* st) {
  groupnorm_kernel<<<B, 512, sizeof(float) * 2 * groups, static_cast<cudaStream_t>(st)>>>(x, x_ld, HW, C, groups, cond,
      cond_ld, gamma, beta, eps, swish, y, y_ld);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}''', 'model2_bwd.cu': r'''
extern "C" int probe_gn_bwd(const float* x, int x_ld, int B, int HW, int C, int groups, const float* cond, int cond_ld,
                            const float* gamma, const float* beta, float eps, int swish, const float* dy, int dy_ld, float* dx,
                            int dx_ld, float* dgamma, float* dbeta, float* dcond, int dcond_ld, void* st) {
  groupnorm_bwd_kernel<<<B, 512, sizeof(float) * (4 * groups + 2 * C), static_cast<cudaStream_t>(st)>>>(x, x_ld, HW, C, groups,
      cond, cond_ld, gamma, beta, eps, swish, dy, dy_ld, dx, dx_ld, dgamma, dbeta, dcond, dcond_ld);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}'''}


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


def one_cta_probe(tmp):
    """the one-CTA GroupNorm kernels behind launchers of this tool, compiled from the library's sources into `tmp`"""
    libs = []
    for unit, launcher in _PROBE.items():
        src = os.path.join(tmp, 'probe_' + unit)
        with open(src, 'w') as f:
            f.write('#include "%s"\n%s\n' % (os.path.join(CSRC, unit), launcher))
        so = src[:-3] + '.so'
        subprocess.run(['nvcc', '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xcompiler', '-fPIC', '-shared',
                        '-I' + CSRC, src, '-L' + CSRC, '-lcolddiff', '-Xlinker', '-rpath=' + CSRC, '-o', so], check=True)
        libs.append(C.CDLL(so))
    return libs[0].probe_gn_fwd, libs[1].probe_gn_bwd


def groupnorm(res, probe):
    fwd1, bwd1 = probe if probe else (None, None)
    for Cc in (128, 256):
        for B in (1, 8, 32):
            HW = S * S
            g = torch.Generator(device='cuda').manual_seed(1)
            x, dy = (torch.randn(B * HW, Cc, device='cuda', generator=g) for _ in range(2))
            y, dx = torch.empty_like(x), torch.empty_like(x)
            cond = torch.randn(B, Cc, device='cuda', generator=g)
            gamma, beta = torch.ones(Cc, device='cuda'), torch.zeros(Cc, device='cuda')
            dg, db, dc = torch.zeros(Cc, device='cuda'), torch.zeros(Cc, device='cuda'), torch.zeros(B, Cc, device='cuda')
            fa = (ptr(x), Cc, B, C.c_int64(HW), Cc, 32, ptr(cond), Cc, ptr(gamma), ptr(beta), C.c_float(1e-6), 1, ptr(y), Cc, stream())
            ba = (ptr(x), Cc, B, C.c_int64(HW), Cc, 32, ptr(cond), Cc, ptr(gamma), ptr(beta), C.c_float(1e-6), 1, ptr(dy), Cc,
                  ptr(dx), Cc, ptr(dg), ptr(db), ptr(dc), Cc, stream())
            plane = 4.0 * B * HW * Cc
            r = dict(C=Cc, B=B, fwd_us=timed(lambda: call('cd_groupnorm_fwd', *fa), 20),
                     bwd_us=timed(lambda: call('cd_groupnorm_bwd', *ba), 20))
            line = 'groupnorm 256^2 C=%3d B=%2d  split: fwd %8.1f us (%5.0f GB/s)  bwd %8.1f us (%5.0f GB/s)' % (
                Cc, B, r['fwd_us'], 3 * plane / r['fwd_us'] / 1e3, r['bwd_us'], 6 * plane / r['bwd_us'] / 1e3)
            if probe:
                fa1 = fa[:3] + (HW,) + fa[4:]
                ba1 = ba[:3] + (HW,) + ba[4:]
                r['fwd_one_cta_us'] = timed(lambda: fwd1(*fa1), 5)
                r['bwd_one_cta_us'] = timed(lambda: bwd1(*ba1), 5)
                line += '   one CTA per image: fwd %8.1f us  bwd %8.1f us' % (r['fwd_one_cta_us'], r['bwd_one_cta_us'])
            print(line)
            res['groupnorm'].append(r)
            del x, dy, y, dx
            torch.cuda.empty_cache()


def model(res, B):
    """one batch size per process: the caching allocator and the engine's shape-keyed buffers of an earlier batch size would
    otherwise still be allocated and count towards this one's peak"""
    T = 200
    with contextlib.redirect_stdout(io.StringIO()):
        m = cdm.Model(resolution=S, in_channels=3, out_ch=3, dropout=0.0, **NET).cuda()
        gd = cdm.GaussianDiffusion(m, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1',
                                   kernel_std=0.1, kernel_size=11, blur_routine='Exponential_reflect',
                                   sampling_routine='x0_step_down').cuda()
        tr = cdm.Trainer(gd, None, image_size=S, train_batch_size=B, train_lr=2e-5, train_num_steps=10 ** 9,
                         gradient_accumulate_every=1, ema_decay=0.995, fp16=False, results_folder=tempfile.mkdtemp(),
                         dataset='synthetic')
    x = torch.rand(B, 3, S, S, device='cuda') * 2 - 1
    for _ in range(3):
        tr.train_step([x])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    us = timed(lambda: tr.train_step([x]), 5)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    r = dict(B=B, step_ms=us / 1e3, images_per_s=B / (us * 1e-6), peak_gib=peak)
    ema = tr.ema_model
    img = gd.opt(x, T)
    step = torch.full((B,), T - 1, dtype=torch.long, device='cuda')

    def reverse():
        with torch.no_grad():
            ema._reverse_step(img, ema.denoise_fn(img, step), T)
    r['reverse_ms'] = timed(reverse, 5) / 1e3
    r['peak_with_sampling_gib'] = torch.cuda.max_memory_allocated() / 2 ** 30
    res['train'].append(r)
    print('Model train step 256^2 B=%2d: %8.2f ms  %6.1f images/s  peak device memory %.2f GiB;  reverse step (x0_step_down) '
          '%.2f ms, peak with it %.2f GiB' % (B, r['step_ms'], r['images_per_s'], peak, r['reverse_ms'], r['peak_with_sampling_gib']))


def measure(res, B):
    """one batch size in a fresh process -> False when it ran out of device memory"""
    with tempfile.NamedTemporaryFile(suffix='.json') as f:
        p = subprocess.run([sys.executable, os.path.abspath(__file__), '--batch', str(B), '--json', f.name], capture_output=True,
                           text=True)
        sys.stdout.write(p.stdout)
        if p.returncode != 0:
            if 'OutOfMemoryError' not in p.stderr and 'out of memory' not in p.stderr:
                sys.exit(p.stderr)
            res['does_not_fit'] = B
            print('Model train step 256^2 B=%2d: out of device memory' % B)
            return False
        res['train'] += json.load(open(f.name))['train']
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json')
    ap.add_argument('--one-cta', action='store_true', help='also time the one-CTA-per-image GroupNorm kernels on 256^2 planes')
    ap.add_argument('--batch', type=int, help='measure the training and reverse step at this batch size only')
    ap.add_argument('--max-batch', type=int, default=64, help='largest batch size tried')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('model_shapes: no CUDA device; nothing is measured')
    name, pl = card()
    print('card: %s, power limit %s' % (name, pl))
    res = dict(card=name, power_limit=pl, groupnorm=[], train=[])
    if a.batch:
        model(res, a.batch)
    else:
        with tempfile.TemporaryDirectory() as tmp:
            groupnorm(res, one_cta_probe(tmp) if a.one_cta else None)
        B = 1
        while B <= a.max_batch and measure(res, B):
            res['largest_batch'] = B
            B *= 2
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
