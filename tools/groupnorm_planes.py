"""Time the one-CTA GroupNorm kernels at the planes of the DDPM `Model`, and list the launches of one 32² training step.

    python tools/groupnorm_planes.py [--baseline-lib PATH] [--json FILE]
    python tools/groupnorm_planes.py --launches FILE

- cd_groupnorm_fwd / cd_groupnorm_bwd (GroupNorm(32) + swish with the time-conditioning row) on 32², 64² and 128² planes,
  C = 128 and 256, B = 128 (the batch of the benchmarked 32² training micro-batch and sample).  Planes of this size take the
  one-CTA-per-image kernels (groupnorm_kernel / groupnorm_bwd_kernel).  Microseconds per call with CUDA events, and the bytes a
  call must move (forward: x read twice, y written once; backward: x read three times, dy twice, dx written once) over that
  time.  With --baseline-lib, the same calls of another build of libcolddiff.so run in the same process, the two alternating
  twice, and the largest differences between the two builds' outputs are printed.
- --launches: one training step of the benchmarked 32² configuration (`Model(ch=128, ch_mult=(1, 2, 2, 2))`, 2 micro-batches
  of 128) under torch.profiler after two warm-up steps; writes every kernel launch in order as [name, grid, block] to FILE.

Every timing is printed with the card name and power limit read in the same run.  A run without a GPU stops."""
import argparse
import contextlib
import ctypes as C
import io
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import torch  # noqa: E402

import cold_diffusion_models_b200 as cdm  # noqa: E402
from cold_diffusion_models_b200 import _lib  # noqa: E402
from model_shapes import card, timed  # noqa: E402

B = 128


def _checked(lib, name):
    fn = getattr(lib, name)

    def run(*args):
        rc = fn(*args)
        if rc != 0:
            raise RuntimeError('%s returned %d' % (name, rc))
    return run


def groupnorm(baseline, res):
    libs = [('this', _lib.lib)] + ([('baseline', C.CDLL(os.path.abspath(baseline)))] if baseline else [])
    p = _lib.ptr
    for S in (32, 64, 128):
        for Cc in (128, 256):
            HW = S * S
            g = torch.Generator(device='cuda').manual_seed(1)
            x = torch.randn(B * HW, Cc, device='cuda', generator=g) * 1.5 + 10.0
            dy = torch.randn(B * HW, Cc, device='cuda', generator=g)
            cond = torch.randn(B, Cc, device='cuda', generator=g)
            gamma = 1 + 0.2 * torch.randn(Cc, device='cuda', generator=g)
            beta = 0.1 * torch.randn(Cc, device='cuda', generator=g)
            plane = 4.0 * B * HW * Cc
            r = dict(S=S, C=Cc, B=B)
            outs = {}
            for rep in range(2):
                for tag, lib in libs:
                    y, dx = torch.empty_like(x), torch.empty_like(x)
                    dg, db, dc = torch.zeros(Cc, device='cuda'), torch.zeros(Cc, device='cuda'), torch.zeros(B, Cc, device='cuda')
                    fa = (p(x), Cc, B, C.c_int64(HW), Cc, 32, p(cond), Cc, p(gamma), p(beta), C.c_float(1e-6), 1, p(y), Cc,
                          _lib.stream())
                    ba = (p(x), Cc, B, C.c_int64(HW), Cc, 32, p(cond), Cc, p(gamma), p(beta), C.c_float(1e-6), 1, p(dy), Cc,
                          p(dx), Cc, p(dg), p(db), p(dc), Cc, _lib.stream())
                    fwd, bwd = _checked(lib, 'cd_groupnorm_fwd'), _checked(lib, 'cd_groupnorm_bwd')
                    r.setdefault(tag + '_fwd_us', []).append(timed(lambda: fwd(*fa), 20))
                    dg.zero_(); db.zero_()
                    bwd(*ba)
                    torch.cuda.synchronize()
                    outs[tag] = (y.clone(), dx.clone(), dg.clone(), db.clone(), dc.clone())
                    r.setdefault(tag + '_bwd_us', []).append(timed(lambda: bwd(*ba), 20))
                    del y, dx
            line = 'groupnorm %3d^2 C=%3d B=%d' % (S, Cc, B)
            for tag, _ in libs:
                f, b = min(r[tag + '_fwd_us']), min(r[tag + '_bwd_us'])
                line += '  %s: fwd %7.1f us (%5.0f GB/s) bwd %7.1f us (%5.0f GB/s) [runs %s / %s]' % (
                    tag, f, 3 * plane / f / 1e3, b, 6 * plane / b / 1e3, ' '.join('%.1f' % v for v in r[tag + '_fwd_us']),
                    ' '.join('%.1f' % v for v in r[tag + '_bwd_us']))
            if baseline:
                r['max_abs_diff'] = [(a - b).abs().max().item() for a, b in zip(outs['this'], outs['baseline'])]
                line += '  max |this - baseline| y %.2e dx %.2e dgamma %.2e dbeta %.2e dcond %.2e' % tuple(r['max_abs_diff'])
            print(line, flush=True)
            res['groupnorm'].append(r)
            del x, dy, outs
            torch.cuda.empty_cache()


def launches(path):
    with contextlib.redirect_stdout(io.StringIO()):
        m = cdm.Model(resolution=32, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 2, 2), num_res_blocks=2,
                      attn_resolutions=(16,), dropout=0.1).cuda()
        gd = cdm.GaussianDiffusion(m, image_size=32, device_of_kernel='cuda', channels=3, timesteps=50, loss_type='l1',
                                   kernel_std=0.1, kernel_size=3, blur_routine='Special_6_routine', train_routine='Final',
                                   sampling_routine='x0_step_down').cuda()
        tr = cdm.Trainer(gd, None, image_size=32, train_batch_size=B, train_lr=2e-5, train_num_steps=10 ** 9,
                         gradient_accumulate_every=2, results_folder=tempfile.mkdtemp(), dataset='synthetic')
    xb = [torch.rand(B, 3, 32, 32, device='cuda') * 2 - 1 for _ in range(2)]
    for _ in range(2):
        tr.train_step(batches=xb)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        tr.train_step(batches=xb)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        trace = os.path.join(tmp, 'trace.json')
        prof.export_chrome_trace(trace)
        ev = json.load(open(trace))['traceEvents']
    ks = sorted((e for e in ev if e.get('cat') == 'kernel'), key=lambda e: e['ts'])
    rows = [[e['name'], e['args'].get('grid'), e['args'].get('block')] for e in ks]
    with open(path, 'w') as f:
        json.dump(rows, f, indent=0)
    gn = sum(1 for r in rows if 'groupnorm' in r[0])
    print('%d kernel launches in one training step (%d GroupNorm kernels) -> %s' % (len(rows), gn, path))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--baseline-lib', help='another build of libcolddiff.so to time against, in the same process')
    ap.add_argument('--json')
    ap.add_argument('--launches', help='write the launch list of one 32^2 training step to this file')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('groupnorm_planes: no CUDA device; nothing is measured')
    if a.launches:
        launches(a.launches)
        return
    name, pl = card()
    print('card: %s, power limit %s' % (name, pl))
    res = dict(card=name, power_limit=pl, groupnorm=[])
    groupnorm(a.baseline_lib, res)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
