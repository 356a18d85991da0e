"""Time the training forward and three kinds of backward of the benchmarked networks:
  full        every parameter trainable, x not differentiated (the training step's backward)
  input-only  every parameter frozen, x.requires_grad (a restoration network used as a differentiable prior)
  half-frozen the down path (downs.* / down.*) frozen, x not differentiated (fine-tuning the rest)
for config 3, Unet(64, (1, 2, 4, 8)) at 128² with B = 32, and Model(ch=128, ch_mult=(1, 2, 2, 2)) at 256² with B = 8.
CUDA events around each pass, after warm-up; the median of --iters runs.  Prints the card and its power limit with the table.

usage: python tools/input_grad_timing.py [--iters 10] [--warmup 3] [--out timing.json]"""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def nets():
    import cold_diffusion_models_b200 as cdm
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
    yield 'Unet config 3, 128², B=32', u, 'downs.', 32, 128
    del u
    torch.cuda.empty_cache()
    m = cdm.Model(resolution=256, in_channels=3, out_ch=3, dropout=0.0, ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2,
                  attn_resolutions=(16,)).cuda()
    yield 'Model 256², B=8', m, 'down.', 8, 256


def time_mode(net, x, t, dy, need_x, iters, warmup):
    fw, bw = [], []
    for i in range(warmup + iters):
        xr = x.detach().requires_grad_(need_x)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        y = net(xr, t)
        e[1].record()
        y.backward(dy)
        e[2].record()
        torch.cuda.synchronize()
        if i >= warmup:
            fw.append(e[0].elapsed_time(e[1]))
            bw.append(e[1].elapsed_time(e[2]))
        del y, xr
    return statistics.median(fw), statistics.median(bw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "input_grad_timing.py measures on a CUDA device"
    rows = []
    for name, net, prefix, B, S in nets():
        g = torch.Generator(device='cuda').manual_seed(1)
        x = torch.rand(B, 3, S, S, generator=g, device='cuda') * 2 - 1
        dy = torch.randn(B, 3, S, S, generator=g, device='cuda') / x.numel()
        t = torch.randint(0, 100, (B,), generator=g, device='cuda')
        res = {}
        for n, p in net.named_parameters():
            p.requires_grad_(True)
        res['forward'], res['full backward'] = time_mode(net, x, t, dy, False, a.iters, a.warmup)
        net.requires_grad_(False)
        _, res['input-only backward'] = time_mode(net, x, t, dy, True, a.iters, a.warmup)
        for n, p in net.named_parameters():
            p.requires_grad_(not n.startswith(prefix))
        _, res['half-frozen backward'] = time_mode(net, x, t, dy, False, a.iters, a.warmup)
        net.requires_grad_(True)
        rows.append((name, res))
    info = dict(card=card(), torch=torch.__version__, iters=a.iters, warmup=a.warmup,
                rows=[dict(network=n, **{k: round(v, 2) for k, v in r.items()}) for n, r in rows])
    print('card (name, power limit, max SM clock): %s' % info['card'])
    print('| network | forward | full backward | input-only backward | half-frozen backward |')
    print('|---|---|---|---|---|')
    for n, r in rows:
        print('| %s | %.1f ms | %.1f ms | %.1f ms | %.1f ms |' % (n, r['forward'], r['full backward'], r['input-only backward'],
                                                                r['half-frozen backward']))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
