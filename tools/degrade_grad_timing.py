"""Time the blur degradation against its adjoint (the backward of `degrade` for the deblurring and resolution packages).

    python tools/degrade_grad_timing.py [--json FILE]

cd_blur_apply (per-sample t) and cd_blur_apply_adjoint at S = 128, 256 and 512, B = 32, C = 3, T = 200 Exponential_reflect
operators: microseconds per launch and FP32 TFLOP/s (4 S^3 FLOP per plane, the same for both).  The two kernels do the same
FLOPs and move the same bytes; the adjoint loads the operator transposed into shared memory (one CTA per plane up to 128²)
or as row segments (the row-strip kernels above).  The pair is timed in three alternating rounds, so the spread between
rounds shows next to the difference.  Every number is printed with the card name and power limit read in the same run.
A run without a GPU stops."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from cold_diffusion_models_b200._lib import call, ptr, stream  # noqa: E402
from cold_diffusion_models_b200.degradation import build_blur_operators  # noqa: E402
from blur_shapes import FP32_FLOPS, card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json', default=None)
    ap.add_argument('--reps', type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('degrade_grad_timing.py needs a CUDA device')
    name, pl = card()
    print('%s, power limit %s' % (name, pl))
    res = dict(card=name, power_limit=pl, rows=[])
    B, Cc, T = 32, 3, 200
    for S in (128, 256, 512):
        ops = build_blur_operators('Exponential_reflect', T, 15, 0.01, S)[0].cuda()
        x = torch.rand(B, Cc, S, S, device='cuda') * 2 - 1
        out = torch.empty_like(x)
        t = torch.randint(0, T - 1, (B,), device='cuda')
        fns = {
            'cd_blur_apply': lambda: call('cd_blur_apply', ptr(x), ptr(out), ptr(ops), ptr(t), 0, B, Cc, S, T, 0, 0, stream()),
            'cd_blur_apply_adjoint': lambda: call('cd_blur_apply_adjoint', ptr(x), ptr(out), ptr(ops), ptr(t), 0, B, Cc, S, T, 0,
                                                  stream()),
        }
        rounds = {k: [] for k in fns}
        for _ in range(3):
            for k, fn in fns.items():
                rounds[k].append(timed(fn, args.reps))
        flop = 4.0 * S ** 3 * B * Cc
        for k, us in rounds.items():
            best = min(us)
            r = dict(kernel=k, S=S, B=B, C=Cc, us=best, us_rounds=us, tflops=flop / (best * 1e-6) / 1e12,
                     share_of_fp32_peak=flop / FP32_FLOPS / (best * 1e-6))
            res['rows'].append(r)
            print('%-22s S=%3d  %9.1f us (rounds %s)  %5.1f TFLOP/s  %3.0f%% of the FP32 data-sheet peak' % (
                k, S, best, ' '.join('%.1f' % v for v in us), r['tflops'], 100 * r['share_of_fp32_peak']))
        fwd, adj = min(rounds['cd_blur_apply']), min(rounds['cd_blur_apply_adjoint'])
        print('  S=%d adjoint / forward = %.3f' % (S, adj / fwd))
        del ops, x, out
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
