"""Time strided sampling, `GaussianDiffusion.sample(..., steps=K)`, with the network forward replayed from its CUDA graph
(`engine.enable_cuda_graph(True)`).  Configurations, each in a fresh process:
  c3  BASELINE config 3: deblurring, Unet(64, (1, 2, 4, 8)), 128², B = 32, T = 200, Exponential_reflect blur, x0_step_down,
      K = 200 (the full loop), 50, 20, 10
  c2  BASELINE config 2: deblurring, the DDPM `Model` (ch 128, ch_mult (1, 2, 2, 2)), 32², B = 128, T = 50, Special_6_routine,
      x0_step_down, K = 50 (the full loop), 10, 5
Each row is the median of --iters whole `sample()` calls after --warmup, CUDA events around each call (from the host's enqueue
of the first launch to the end of the last kernel), every call started from an idle device, as tools/model_graph_timing.py
does.  Speed only: what a smaller K does to sample quality (FID) is not measured here.  Prints the card and its power limit
with the table.

usage: python tools/strided_sampling_timing.py [--iters 5] [--warmup 2] [--out timing.json]"""
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

CONFIGS = {'c3': (128, 32, 200, (200, 50, 20, 10)), 'c2': (32, 128, 50, (50, 10, 5))}


def run_one(name, iters, warmup):
    import torch
    import cold_diffusion_models_b200 as cdm
    assert torch.cuda.is_available(), "strided_sampling_timing.py measures on a CUDA device"
    S, B, T, Ks = CONFIGS[name]
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        if name == 'c3':
            net = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
            kw = dict(kernel_std=0.01, kernel_size=15, blur_routine='Exponential_reflect')
        else:
            net = cdm.Model(resolution=32, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2,
                            attn_resolutions=(16,), dropout=0.1).cuda()
            kw = dict(kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine')
        gd = cdm.GaussianDiffusion(net, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1',
                                   train_routine='Final', sampling_routine='x0_step_down', **kw).cuda()
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.rand(B, 3, S, S, generator=g, device='cuda') * 2 - 1
    net.engine.enable_cuda_graph(True)
    rows = []
    with torch.no_grad():
        for K in Ks:
            ms, host_ms = timed(lambda: gd.sample(batch_size=B, img=x, steps=K), iters, warmup)
            rows.append(dict(config=name, S=S, B=B, T=T, K=K, ms=ms, host_ms=host_ms, ms_per_step=ms / K))
    net.engine.enable_cuda_graph(False)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
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
                rows += json.load(fh)
    info = dict(card=card(), iters=a.iters, warmup=a.warmup, rows=rows)
    print('card (name, power limit, max SM clock): %s' % info['card'])
    print('| configuration | K | sample() | per reverse step | host | vs K = T |')
    print('|---|---|---|---|---|---|')
    full = {r['config']: r['ms'] for r in rows if r['K'] == r['T']}
    for r in rows:
        print('| %s (%d², B = %d, T = %d) | %d | %.1f ms | %.2f ms | %.1f ms | %.2fx |'
              % (r['config'], r['S'], r['B'], r['T'], r['K'], r['ms'], r['ms_per_step'], r['host_ms'], full[r['config']] / r['ms']))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
