"""CUDA-event timings of the Lab colour path (`to_lab=True`) of the decolor package at the drivers' shapes, next to the same
work without Lab and to the reference's eager-PyTorch Lab step chain (tests/lab_oracle.py's DecolorLabFP) on the same GPU:

  * cd_chanmix_lab alone (q_sample of a batch at t = T-1, the longest chain) vs the eager chain of T full-tensor passes;
  * one p_losses forward + backward, to_lab on / off;
  * one full sample() (T reverse steps), to_lab on / off.

Shapes: CIFAR-10 (32 x 32, UnetResNet) and CelebA (64 x 64, UnetConvNext), batch 32, T = 20 'Linear' with total removal.
Prints the card's name and power limit with the numbers.  GPU only; writes nothing.

    python tools/lab_decolor_timing.py [--reps N]
"""
import argparse
import contextlib
import io
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch  # noqa: E402


def cuda_ms(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or 'unknown'
    except Exception:
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--batch', type=int, default=32)
    args = ap.parse_args()
    import lab_oracle as LO
    from cold_diffusion_models_b200 import snowification_diffusion as snp
    from cold_diffusion_models_b200.snowification_diffusion.utils import rgb2lab
    assert torch.cuda.is_available(), "needs a CUDA device"
    print('device: %s, power limit: %s' % (torch.cuda.get_device_name(), power_limit()))
    B, T = args.batch, 20

    class Args:
        pass
    rows = []
    for name, S, model in (('CIFAR-10 32x32 UnetResNet', 32, ('UnetResNet', 'cifar10_train')), ('CelebA 64x64 UnetConvNext', 64, ('UnetConvNext', 'celebA'))):
        a = Args()
        a.model, a.dataset = model
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            net = snp.get_model(a).cuda()
        gds = {}
        for lab in (False, True):
            with contextlib.redirect_stdout(io.StringIO()):
                gds[lab] = snp.GaussianDiffusion(net, image_size=S, device_of_kernel='cuda', channels=3, timesteps=T, loss_type='l1',
                                                 forward_process_type='Decolorization', decolor_routine='Linear', decolor_total_remove=True,
                                                 train_routine='Final', sampling_routine='x0_step_down', to_lab=lab).cuda()
        x_rgb = torch.rand(B, 3, S, S, device='cuda') * 2 - 1
        x = {False: x_rgb, True: rgb2lab(x_rgb)}
        t_last = torch.full((B,), T - 1, dtype=torch.long, device='cuda')
        t_rand = torch.randint(0, T, (B,), device='cuda')

        fp = LO.DecolorLabFP(gds[True].forward_process.factors)

        def eager_chain():
            v = x[True]
            with torch.no_grad():
                for i in range(T):
                    v = fp.forward(v, i)
            return v
        rows.append((name, 'q_sample t=T-1: cd_chanmix_lab', cuda_ms(lambda: gds[True].q_sample(x[True], t_last), args.reps)))
        rows.append((name, 'q_sample t=T-1: cd_chanmix (RGB)', cuda_ms(lambda: gds[False].q_sample(x[False], t_last), args.reps)))
        rows.append((name, 'q_sample t=T-1: eager PyTorch Lab chain', cuda_ms(eager_chain, args.reps)))
        for lab in (False, True):
            def step():
                loss = gds[lab].p_losses(x[lab], t_rand)
                loss.backward()
            rows.append((name, 'p_losses fwd+bwd, to_lab=%s' % lab, cuda_ms(step, args.reps)))
        for lab in (False, True):
            rows.append((name, 'sample() %d steps, to_lab=%s' % (T, lab),
                         cuda_ms(lambda: gds[lab].sample(batch_size=B, img=x[lab]), max(3, args.reps // 3), warmup=1)))
        del net, gds
        torch.cuda.empty_cache()
    print('batch %d, T = %d (Linear, total removal), median of CUDA-event times' % (B, T))
    w = max(len(r[0]) for r in rows)
    for shape, what, ms in rows:
        print('%-*s  %-42s %10.3f ms' % (w, shape, what, ms))


if __name__ == '__main__':
    main()
