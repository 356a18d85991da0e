"""ORACLE (test infrastructure only -- never imported by the product path).

CPU fp32 restatement of the reference deblurring `GaussianDiffusion` hot path
(DB = deblurring-diffusion-pytorch/deblurring_diffusion_pytorch/deblurring_diffusion_pytorch.py):
blur-kernel schedule (DB:348-389), q_sample (DB:927-960), p_losses (DB:963-975) and the
Algorithm-1/2 sampling loop `sample` (DB:393-455) / `all_sample` (DB:609-689).

The Gaussian taps come from torchgeometry (not part of the reference and absent from this
image, un-pinned by the reference): restated in `gaussian_1d` from torchgeometry 0.1.2
image/gaussian.py.  PARITY UNPINNED at that single boundary (<= last-ulp differences in
<= 27 taps); everything else in this file is pinned against the real reference by
tests/test_oracle_golden.py.
"""
import numpy as np
import torch
import torch.nn.functional as F


def gaussian_1d(ksize, sigma):
    # torchgeometry 0.1.2 image/gaussian.py::gaussian -- exponent evaluated in Python double,
    # cast to fp32, exp in fp32, normalised in fp32.
    def gauss_fcn(x):
        return -(x - ksize // 2) ** 2 / float(2 * sigma ** 2)
    g = torch.stack([torch.exp(torch.tensor(gauss_fcn(x))) for x in range(ksize)])
    return g / g.sum()


def gaussian_2d(ksize, sigma):
    g = gaussian_1d(ksize, sigma)
    return torch.matmul(g.unsqueeze(-1), g.unsqueeze(-1).t())


def blur_schedule(blur_routine, timesteps, kernel_size, kernel_std):
    """-> list of (ksize, sigma, pad_mode) per step i, DB:363-389.  Unknown routine -> []
    (the reference silently builds no kernels)."""
    out = []
    for i in range(timesteps):
        if blur_routine == 'Incremental':
            out.append((kernel_size, kernel_std * (i + 1), 'circular'))
        elif blur_routine == 'Constant':
            out.append((kernel_size, kernel_std, 'circular'))
        elif blur_routine == 'Constant_reflect':
            out.append((kernel_size, kernel_std, 'reflect'))
        elif blur_routine == 'Exponential_reflect':
            out.append((kernel_size, np.exp(kernel_std * i), 'reflect'))
        elif blur_routine == 'Exponential':
            out.append((kernel_size, np.exp(kernel_std * i), 'circular'))
        elif blur_routine == 'Individual_Incremental':
            ks = 2 * i + 1
            out.append((ks, 2 * ks, 'circular'))
        elif blur_routine == 'Special_6_routine':
            out.append((11, i / 100 + 0.35, 'reflect'))
    return out


class DeblurOracle:
    """Restates GaussianDiffusion(denoise_fn, image_size, channels, timesteps, loss_type,
    kernel_std, kernel_size, blur_routine, train_routine='Final', sampling_routine, discrete)."""

    def __init__(self, denoise_fn, *, image_size, channels=3, timesteps=1000, loss_type='l1',
                 kernel_std=0.1, kernel_size=3, blur_routine='Incremental',
                 sampling_routine='default', discrete=False):
        self.denoise_fn = denoise_fn
        self.image_size, self.channels = image_size, channels
        self.num_timesteps = int(timesteps)
        self.loss_type = loss_type
        self.blur_routine, self.sampling_routine, self.discrete = blur_routine, sampling_routine, discrete
        self.schedule = blur_schedule(blur_routine, self.num_timesteps, kernel_size, kernel_std)
        self.kernels2d = [gaussian_2d(k, s) for (k, s, _) in self.schedule]

    def to(self, device):
        """move the blur taps (the only tensors the oracle owns) -- lets bench.py time this eager-PyTorch restatement on a GPU too"""
        self.kernels2d = [k.to(device) for k in self.kernels2d]
        return self

    def blur_step(self, i, x):
        # nn.Conv2d(C, C, k, padding=(k-1)/2, padding_mode=mode, groups=C, bias=False) DB:351-361
        k, _, mode = self.schedule[i]
        pad = int((k - 1) / 2)
        w = self.kernels2d[i][None, None].repeat(self.channels, 1, 1, 1)
        if pad > 0:
            x = F.pad(x, (pad, pad, pad, pad), mode=mode)
        return F.conv2d(x, w, None, groups=self.channels)

    def _collapse(self, x):
        m = torch.mean(x, [2, 3], keepdim=True)
        return m.expand(x.shape[0], x.shape[1], x.shape[2], x.shape[3])

    def q_sample(self, x_start, t):
        # DB:927-960
        max_iters = int(torch.max(t))
        all_blurs = []
        x = x_start
        for i in range(max_iters + 1):
            x = self.blur_step(i, x)
            if self.discrete and i == (self.num_timesteps - 1):
                x = self._collapse(x)
            all_blurs.append(x)
        all_blurs = torch.stack(all_blurs)
        choose = torch.stack([all_blurs[int(t[b]), b] for b in range(t.shape[0])])       # (DB:947-950: per-sample Python indexing)
        if self.discrete:
            choose = (choose + 1) * 0.5
            choose = choose * 255
            choose = choose.int().float() / 255
            choose = choose * 2 - 1
        return choose

    def p_losses(self, x_start, t):
        # DB:963-975
        x_blur = self.q_sample(x_start, t)
        x_recon = self.denoise_fn(x_blur, t)
        if self.loss_type == 'l1':
            return (x_start - x_recon).abs().mean()
        elif self.loss_type == 'l2':
            return F.mse_loss(x_start, x_recon)
        raise NotImplementedError()

    def degrade(self, img, t):
        # "opt" DB:595-607 / head of sample DB:401-407
        if self.blur_routine == 'Individual_Incremental':
            return self.blur_step(t - 1, img)
        for i in range(t):
            img = self.blur_step(i, img)
        return img

    @torch.no_grad()
    def sample(self, batch_size, img, t=None, noise=None):
        """DB:393-455 (gen_sample DB:526-593 when `noise` -- already scaled by noise_level -- is given).
        Returns (xt, direct_recons, img)."""
        if t is None:
            t = self.num_timesteps
        img = self.degrade(img, t)
        if self.discrete:
            img = self._collapse(img)
        if noise is not None:
            img = img + noise
        xt = img
        direct_recons = None
        while t:
            step = torch.full((batch_size,), t - 1, dtype=torch.long)
            x = self.denoise_fn(img, step)
            if direct_recons is None:
                direct_recons = x
            if self.sampling_routine == 'default':
                if self.blur_routine == 'Individual_Incremental':
                    x = self.blur_step(t - 2, x)  # NB: index -1 at t==1, as in the reference
                else:
                    for i in range(t - 1):
                        x = self.blur_step(i, x)
            elif self.sampling_routine == 'x0_step_down':
                x_times = x
                for i in range(t):
                    x_times = self.blur_step(i, x_times)
                    if self.discrete and i == (self.num_timesteps - 1):
                        x_times = self._collapse(x_times)
                x_sub1 = x
                for i in range(t - 1):
                    x_sub1 = self.blur_step(i, x_sub1)
                x = img - x_times + x_sub1
            img = x
            t -= 1
        return xt, direct_recons, img

    # ---- cover-figure trajectories (DB:691-861), non-'Individual_Incremental' routines ----------------------
    def _cum(self, x, n):
        for i in range(n):
            x = self.blur_step(i, x)
        return x

    def _alg2(self, img, x, times):
        x_times = x
        for i in range(times):
            x_times = self.blur_step(i, x_times)
            if self.discrete and i == (self.num_timesteps - 1):
                x_times = self._collapse(x_times)
        return img - x_times + self._cum(x, times - 1)

    @torch.no_grad()
    def forward_and_backward(self, batch_size, img, t=None, times=None):
        """DB:691-770 with noise_level = 0 -> (Forward, Backward, img)"""
        t = t or self.num_timesteps
        times = times or t
        Forward = [img]
        for i in range(t):
            img = self.blur_step(i, img)
            Forward.append(img)
        if self.discrete:
            img = self._collapse(img)
        Backward = []
        while times:
            step = torch.full((batch_size,), times - 1, dtype=torch.long)
            x = self.denoise_fn(img, step)
            Backward.append(img)
            if self.sampling_routine == 'default':
                x = self._cum(x, times - 1)
            elif self.sampling_routine == 'x0_step_down':
                x = self._alg2(img, x, times)
            img = x
            times -= 1
        return Forward, Backward, img

    @torch.no_grad()
    def forward_and_backward_2(self, batch_size, img):
        """DB:772-861 with noise_level = 0 -> (Forward, Backward_1, Backward_2, img_1, img_2)"""
        T = self.num_timesteps
        Forward = [img]
        for i in range(T):
            img = self.blur_step(i, img)
            Forward.append(img)
        if self.discrete:
            img = self._collapse(img)
        last = img
        outs = []
        for alg in (1, 2):
            img, times, B = last, T, []
            while times:
                step = torch.full((batch_size,), times - 1, dtype=torch.long)
                x = self.denoise_fn(img, step)
                B.append(img)
                img = self._cum(x, times - 1) if alg == 1 else self._alg2(img, x, times)
                times -= 1
            outs.append((B, img))
        return Forward, outs[0][0], outs[1][0], outs[0][1], outs[1][1]
