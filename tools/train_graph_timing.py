"""Time the training step eager and replayed from a CUDA graph (`Trainer.enable_cuda_graph(True)`).  Configurations, each in a
fresh process, every one B = 32 images per micro-batch (128 for config 2) and gradient_accumulate_every = 2:
  mnist-deblur     the deblurring package's MNIST driver: Unet(64, (1, 2, 4, 8), channels=1) at 32², T = 20, k = 11, σ = 7, Constant
  cifar10-deblur   the same Unet with 3 channels at 32² (the CIFAR-10 drivers)
  c2-model         BASELINE config 2: Model(ch=128, ch_mult=(1, 2, 2, 2), attn at 16², dropout 0.1) at 32², B = 128,
                   T = 50, Special_6_routine
  snow-cifar10     the snowification CIFAR-10 run: SnowificationTrainer with the package's UnetConvNext (Unet(64, (1, 2, 4, 8),
                   residual=False)) at 32², Snow level 1 with random_snow, T = 50; its train() loop calls loss.item() after
                   every step, and so does this row
  c3-celeba128     BASELINE config 3: Unet(64, (1, 2, 4, 8)) at 128², T = 200, k = 15, Exponential_reflect
Per row: "step" is the median interval between CUDA events recorded at the start of consecutive steps run back to back (host
enqueue and device work overlap as in a training loop), over --steps steps after --warmup; "host" is the median wall time of a
train_step call returning, each from an idle device (the Python schedule plus the launch calls); "peak" is
torch.cuda.max_memory_allocated over the mode's steps.  The graphed mode's first step (the capture) is part of its warm-up.
Batches are pinned host tensors copied in by train_step, as a DataLoader with pin_memory delivers them.  Prints the card and
its power limit with the table.

usage: python tools/train_graph_timing.py [--steps 30] [--warmup 5] [--out timing.json]"""
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

CONFIGS = ('mnist-deblur', 'cifar10-deblur', 'c2-model', 'snow-cifar10', 'c3-celeba128')
A = 2


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        import torch
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        import torch
        return torch.cuda.get_device_name()


def build(name, results):
    """-> (trainer, S, C, B, sync_loss)"""
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200 import snowification_diffusion as sn
    common = dict(train_lr=2e-5, gradient_accumulate_every=A, results_folder=results, dataset='synthetic')
    with contextlib.redirect_stdout(io.StringIO()):
        if name in ('mnist-deblur', 'cifar10-deblur'):
            C = 1 if name == 'mnist-deblur' else 3
            net = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=C)
            gd = cdm.GaussianDiffusion(net, image_size=32, device_of_kernel='cuda', channels=C, timesteps=20, loss_type='l1',
                                       kernel_std=7, kernel_size=11, blur_routine='Constant').cuda()
            return cdm.Trainer(gd, None, image_size=32, train_batch_size=32, **common), 32, C, 32, False
        if name == 'c2-model':
            net = cdm.Model(resolution=32, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2,
                            attn_resolutions=(16,), dropout=0.1)
            gd = cdm.GaussianDiffusion(net, image_size=32, device_of_kernel='cuda', channels=3, timesteps=50, loss_type='l1',
                                       kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine').cuda()
            return cdm.Trainer(gd, None, image_size=32, train_batch_size=128, **common), 32, 3, 128, False
        if name == 'snow-cifar10':
            net = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3, residual=False)
            gd = sn.GaussianDiffusion(net, image_size=(32, 32), device_of_kernel='cuda', channels=3, timesteps=50, loss_type='l1',
                                      forward_process_type='Snow', snow_level=1, random_snow=True, batch_size=32).cuda()
            return sn.Trainer(gd, None, train_batch_size=32, **common), 32, 3, 32, True
        if name == 'c3-celeba128':
            net = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3)
            gd = cdm.GaussianDiffusion(net, image_size=128, device_of_kernel='cuda', channels=3, timesteps=200, loss_type='l1',
                                       kernel_std=0.01, kernel_size=15, blur_routine='Exponential_reflect').cuda()
            return cdm.Trainer(gd, None, image_size=128, train_batch_size=32, **common), 128, 3, 32, False
    raise KeyError(name)


def run_one(name, steps, warmup):
    import torch
    assert torch.cuda.is_available(), "train_graph_timing.py measures on a CUDA device"
    torch.manual_seed(0)
    with tempfile.TemporaryDirectory() as results:
        tr, S, C, B, sync_loss = build(name, results)
        g = torch.Generator().manual_seed(1)
        host = [(torch.rand(B, C, S, S, generator=g) * 2 - 1).pin_memory() for _ in range(4 * A)]
        it = [0]

        def step():
            k = it[0] % 4
            it[0] += 1
            loss = tr.train_step(batches=host[k * A:(k + 1) * A])
            if sync_loss:
                loss.item()
        res = dict(config=name, S=S, B=B, A=A)
        for mode, flag in (('eager', False), ('graphed', True)):
            tr.enable_cuda_graph(flag)
            for _ in range(warmup):
                step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
            for i in range(steps):
                ev[i].record()
                step()
            ev[steps].record()
            torch.cuda.synchronize()
            res[mode + '_ms'] = statistics.median(ev[i].elapsed_time(ev[i + 1]) for i in range(steps))
            host_ms = []
            for _ in range(steps):
                torch.cuda.synchronize()
                h0 = time.perf_counter()
                step()
                host_ms.append((time.perf_counter() - h0) * 1e3)
            torch.cuda.synchronize()
            res[mode + '_host_ms'] = statistics.median(host_ms)
            res[mode + '_peak_gib'] = torch.cuda.max_memory_allocated() / 2 ** 30
        tr.enable_cuda_graph(False)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    ap.add_argument('--configs', default=','.join(CONFIGS))
    ap.add_argument('--config', default=None, help='run one configuration in this process (internal)')
    ap.add_argument('--json', default=None, help='with --config: write its result here')
    a = ap.parse_args()
    if a.config:
        r = run_one(a.config, a.steps, a.warmup)
        with open(a.json, 'w') as f:
            json.dump(r, f)
        return
    rows = []
    for name in a.configs.split(','):
        with tempfile.NamedTemporaryFile(suffix='.json') as f:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--config', name, '--json', f.name, '--steps',
                                str(a.steps), '--warmup', str(a.warmup)], capture_output=True, text=True)
            if p.returncode != 0:
                raise RuntimeError('%s failed:\n%s' % (name, p.stderr[-3000:]))
            with open(f.name) as fh:
                rows.append(json.load(fh))
    info = dict(card=card(), steps=a.steps, warmup=a.warmup, rows=rows)
    print('card (name, power limit, max SM clock): %s' % info['card'])
    print('| configuration | eager step | eager host | graphed step | graphed host | eager / graphed | peak eager | peak graphed |')
    print('|---|---|---|---|---|---|---|---|')
    for r in rows:
        print('| %s (%d², %d x %d) | %.2f ms | %.2f ms | %.2f ms | %.2f ms | %.2fx | %.2f GiB | %.2f GiB |'
              % (r['config'], r['S'], r['A'], r['B'], r['eager_ms'], r['eager_host_ms'], r['graphed_ms'], r['graphed_host_ms'],
                 r['eager_ms'] / r['graphed_ms'], r['eager_peak_gib'], r['graphed_peak_gib']))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
