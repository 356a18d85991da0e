"""Time the DDPM `Model` forward eager and replayed from a CUDA graph (`Model.engine.enable_cuda_graph(True)`), and the host-side
schedule of the eager forward alone.  Configurations, each in a fresh process:
  fwd32-B1, fwd32-B16, fwd32-B128  BASELINE config 2's network, Model(ch=128, ch_mult=(1, 2, 2, 2), attn at 16²), at 32²
  fwd128-B16                       the snowification package's celebA `UnetResNet` (the same network at 128²)
  sample-c2                        one full config-2 `sample()` (deblurring, Special_6_routine, T = 50, x0_step_down, B = 128)
Forward rows: CUDA events around each call (from the host's enqueue of the first launch to the end of the last kernel), median
of --iters calls after --warmup; "host" is the wall time of the eager call returning, measured from an idle device, which is
the Python schedule plus the launch API calls (every launch is asynchronous).  The sample row times whole `sample()` calls the
same way.  Prints the card and its power limit with the table.

usage: python tools/model_graph_timing.py [--iters 10] [--warmup 3] [--out timing.json]"""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {'fwd32-B1': (32, 1), 'fwd32-B16': (32, 16), 'fwd32-B128': (32, 128), 'fwd128-B16': (128, 16), 'sample-c2': (32, 128)}


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        import torch
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        import torch
        return torch.cuda.get_device_name()


def timed(fn, iters, warmup):
    """-> (median device-side ms between events around fn, median host ms of fn returning), each call from an idle device"""
    import torch
    dev, host = [], []
    for i in range(warmup + iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        e0.record()
        fn()
        e1.record()
        h1 = time.perf_counter()
        torch.cuda.synchronize()
        if i >= warmup:
            dev.append(e0.elapsed_time(e1))
            host.append((h1 - h0) * 1e3)
    return statistics.median(dev), statistics.median(host)


def run_one(name, iters, warmup):
    import torch
    import cold_diffusion_models_b200 as cdm
    assert torch.cuda.is_available(), "model_graph_timing.py measures on a CUDA device"
    S, B = CONFIGS[name]
    torch.manual_seed(0)
    m = cdm.Model(resolution=S, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2, attn_resolutions=(16,),
                  dropout=0.1).cuda().eval()
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.rand(B, 3, S, S, generator=g, device='cuda') * 2 - 1
    t = torch.randint(0, 50, (B,), generator=g, device='cuda')
    res = dict(config=name, S=S, B=B)
    with torch.no_grad():
        if name == 'sample-c2':
            with contextlib.redirect_stdout(io.StringIO()):
                gd = cdm.GaussianDiffusion(m, image_size=32, device_of_kernel='cuda', channels=3, timesteps=50, loss_type='l1',
                                           kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine', train_routine='Final',
                                           sampling_routine='x0_step_down').cuda()
            fn = lambda: gd.sample(batch_size=B, img=x)        # noqa: E731
            res['eager_ms'], res['eager_host_ms'] = timed(fn, iters, warmup)
            m.engine.enable_cuda_graph(True)
            res['graphed_ms'], res['graphed_host_ms'] = timed(fn, iters, warmup)
        else:
            fn = lambda: m(x, t)                               # noqa: E731
            res['eager_ms'], res['eager_host_ms'] = timed(fn, iters, warmup)
            m.engine.enable_cuda_graph(True)
            res['graphed_ms'], res['graphed_host_ms'] = timed(fn, iters, warmup)
        m.engine.enable_cuda_graph(False)
    res['peak_gib'] = torch.cuda.max_memory_allocated() / 2 ** 30
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--config', default=None, help='run one configuration in this process (internal)')
    ap.add_argument('--json', default=None, help='with --config: write its result here')
    a = ap.parse_args()
    if a.config:
        r = run_one(a.config, a.iters, a.warmup)
        with open(a.json, 'w') as f:
            json.dump(r, f)
        return
    rows = []
    for name in CONFIGS:
        with tempfile.NamedTemporaryFile(suffix='.json') as f:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--config', name, '--json', f.name, '--iters',
                                str(a.iters), '--warmup', str(a.warmup)], capture_output=True, text=True)
            if p.returncode != 0:
                raise RuntimeError('%s failed:\n%s' % (name, p.stderr[-3000:]))
            with open(f.name) as fh:
                rows.append(json.load(fh))
    info = dict(card=card(), iters=a.iters, warmup=a.warmup, rows=rows)
    print('card (name, power limit, max SM clock): %s' % info['card'])
    print('| configuration | eager | eager, host schedule | graphed | graphed, host | speed-up | peak memory |')
    print('|---|---|---|---|---|---|---|')
    for r in rows:
        print('| %s (%d², B = %d) | %.2f ms | %.2f ms | %.2f ms | %.2f ms | %.2fx | %.1f GiB |'
              % (r['config'], r['S'], r['B'], r['eager_ms'], r['eager_host_ms'], r['graphed_ms'], r['graphed_host_ms'],
                 r['eager_ms'] / r['graphed_ms'], r['peak_gib']))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
