"""Drop-in `GaussianDiffusion` of denoising_diffusion_pytorch -- the Gaussian-noise ("hot") baseline
(reference: denoising-diffusion-pytorch/denoising_diffusion_pytorch/denoising_diffusion_pytorch.py:308-542, "DN").

Same constructor (no `device_of_kernel`), two-input `forward(x1, x2)`, `q_sample(x_start, x_end, t)`, `sample`,
`gen_sample` ('ddim' / 'x0_step_down'), `all_sample`, `forward_and_backward`; the lerp and the reverse step are
single elementwise kernels (cd_noise_lerp / cd_noise_step) around the same Unet engine."""
import ctypes as C
import torch
from torch import nn

from ._lib import call, ptr, stream
from .autograd import LerpDegrade
from .deblurring import _LossFn
from .strided import reverse_levels


def cosine_beta_schedule(timesteps, s=0.008):
    # DN:295-305 (torch.linspace variant)
    steps = timesteps + 1
    x = torch.linspace(0, steps, steps)
    alphas_cumprod = torch.cos(((x / steps) + s) / (1 + s) * torch.pi * 0.5) ** 2
    alphas_cumprod = alphas_cumprod / alphas_cumprod[0]
    betas = 1 - (alphas_cumprod[1:] / alphas_cumprod[:-1])
    return torch.clip(betas, 0, 0.999)


class GaussianDiffusion(nn.Module):
    def __init__(self, denoise_fn, *, image_size, channels=3, timesteps=1000, loss_type='l1', train_routine='Final',
                 sampling_routine='default', discrete=False):
        super().__init__()
        self.channels = channels
        self.image_size = image_size
        self.denoise_fn = denoise_fn
        self.num_timesteps = int(timesteps)
        self.loss_type = loss_type
        betas = cosine_beta_schedule(timesteps)
        alphas = 1. - betas
        alphas_cumprod = torch.cumprod(alphas, axis=0)
        self.register_buffer('alphas_cumprod', alphas_cumprod)
        self.register_buffer('sqrt_alphas_cumprod', torch.sqrt(alphas_cumprod))
        self.register_buffer('sqrt_one_minus_alphas_cumprod', torch.sqrt(1. - alphas_cumprod))
        self.train_routine = train_routine
        self.sampling_routine = sampling_routine

    # ---- forward process --------------------------------------------------------------------------------------
    def q_sample(self, x_start, x_end, t):
        """DN:517-522; t: (B,) int64"""
        x_start = x_start.contiguous().float(); x_end = x_end.contiguous().float()
        t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
        out = torch.empty_like(x_start)
        with torch.no_grad():
            call('cd_noise_lerp', ptr(x_start), ptr(x_end), ptr(t), 0, ptr(self.sqrt_alphas_cumprod),
                 ptr(self.sqrt_one_minus_alphas_cumprod), C.c_int64(x_start[0].numel()), C.c_int64(x_start.numel()),
                 ptr(out), stream())
        return out

    def degrade(self, x_start, x_end, t):
        """sqrt(alpha_bar_t) x_start + sqrt(1 - alpha_bar_t) x_end: `q_sample`'s values bit for bit (same kernel),
        differentiable with respect to both images"""
        x_start = x_start.contiguous().float(); x_end = x_end.contiguous().float()
        t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
        return LerpDegrade.apply(x_start, x_end, t, 0, self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod, 0)

    def get_x2_bar_from_xt(self, x1_bar, xt, t):
        # DN:377-381 (API parity; the sampling loops use the fused cd_noise_step)
        a = self.sqrt_alphas_cumprod.gather(-1, t).reshape(-1, 1, 1, 1)
        b = self.sqrt_one_minus_alphas_cumprod.gather(-1, t).reshape(-1, 1, 1, 1)
        return (xt - a * x1_bar) / b

    def p_losses(self, x_start, x_end, t):
        if self.train_routine == 'Final':
            x_mix = self.q_sample(x_start=x_start, x_end=x_end, t=t)
            x_recon = self.denoise_fn(x_mix, t)
            if self.loss_type == 'l1':
                loss = _LossFn.apply(x_start, x_recon, 0)
            elif self.loss_type == 'l2':
                loss = _LossFn.apply(x_start, x_recon, 1)
            else:
                raise NotImplementedError()
        return loss

    def forward(self, x1, x2, *args, **kwargs):
        b, c, h, w, device, img_size, = *x1.shape, x1.device, self.image_size
        assert h == img_size and w == img_size, f'height and width of image must be {img_size}'
        t = torch.randint(0, self.num_timesteps, (b,), device=device).long()
        return self.p_losses(x1, x2, t, *args, **kwargs)

    # ---- reverse process --------------------------------------------------------------------------------------
    def _step(self, img, x1_bar, noise, mode, t):
        out = torch.empty_like(img)
        call('cd_noise_step', ptr(img.contiguous()), ptr(x1_bar.contiguous()), ptr(noise), mode, t,
             ptr(self.sqrt_alphas_cumprod), ptr(self.sqrt_one_minus_alphas_cumprod), C.c_int64(img.numel()), ptr(out), stream())
        return out

    def _step_to(self, img, x1_bar, noise, mode, t, s):
        """the reverse step from level t to any level s < t (cd_noise_step_to; s = t - 1 is _step's result bit for bit)"""
        out = torch.empty_like(img)
        call('cd_noise_step_to', ptr(img.contiguous()), ptr(x1_bar.contiguous()), ptr(noise), mode, t, s,
             ptr(self.sqrt_alphas_cumprod), ptr(self.sqrt_one_minus_alphas_cumprod), C.c_int64(img.numel()), ptr(out), stream())
        return out

    def _reverse(self, batch_size, img, t, mode, noise, collect=None):
        direct_recons = None
        while t:
            step = torch.full((batch_size,), t - 1, dtype=torch.long, device=img.device)
            x1_bar = self.denoise_fn(img, step)
            if collect is not None:
                collect(x1_bar, img, step)
            if direct_recons is None:
                direct_recons = x1_bar
            img = self._step(img, x1_bar, noise, mode, t)
            t = t - 1
        return direct_recons, img

    def _reverse_strided(self, batch_size, img, levels, mode, noise):
        """_reverse through the given levels (strided.reverse_levels), one cd_noise_step_to per pair"""
        direct_recons = None
        for hi, lo in zip(levels, levels[1:]):
            step = torch.full((batch_size,), hi - 1, dtype=torch.long, device=img.device)
            x1_bar = self.denoise_fn(img, step)
            if direct_recons is None:
                direct_recons = x1_bar
            img = self._step_to(img, x1_bar, noise, mode, hi, lo)
        return direct_recons, img

    @torch.no_grad()
    def sample(self, batch_size=16, img=None, t=None, *, steps=None):
        """DN:342-375 (always the 'ddim'-style estimate of x2) -> (xt, direct_recons, img).  steps=K: K reverse steps through
        the levels of strided.reverse_levels (cd_noise_step_to) instead of all t (None: every level, the reference's loop)"""
        if t is None:
            t = self.num_timesteps
        levels = None if steps is None else reverse_levels(t, steps)
        self.denoise_fn.eval()
        xt = img
        if levels is None:
            direct_recons, img = self._reverse(batch_size, img.contiguous().float(), t, 0, None)
        else:
            direct_recons, img = self._reverse_strided(batch_size, img.contiguous().float(), levels, 0, None)
        self.denoise_fn.train()
        return xt, direct_recons, img

    @torch.no_grad()
    def gen_sample(self, batch_size=16, img=None, t=None):
        """DN:383-434 -> (noise, direct_recons, img); sampling_routine 'ddim' or 'x0_step_down'"""
        self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        noise = img.contiguous().float()
        direct_recons = None
        out = noise
        if self.sampling_routine == 'ddim':
            direct_recons, out = self._reverse(batch_size, noise, t, 0, None)
        elif self.sampling_routine == 'x0_step_down':
            direct_recons, out = self._reverse(batch_size, noise, t, 1, noise)
        return noise, direct_recons, out

    @torch.no_grad()
    def all_sample(self, batch_size=16, img=None, t=None, times=None, eval=True):
        """DN:474-515 -> (X1_0s, X2_0s, X_ts) as CPU tensors"""
        if eval:
            self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        X1_0s, X2_0s, X_ts = [], [], []

        def collect(x1_bar, cur, step):
            X1_0s.append(x1_bar.detach().cpu())
            X2_0s.append(self.get_x2_bar_from_xt(x1_bar, cur, step).detach().cpu())
            X_ts.append(cur.detach().cpu())
        self._reverse(batch_size, img.contiguous().float(), t, 0, None, collect=collect)
        return X1_0s, X2_0s, X_ts

    @torch.no_grad()
    def forward_and_backward(self, batch_size=16, img=None, t=None, times=None, eval=True):
        """DN:437-472 -> (Forward, Backward, img)"""
        self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        img = img.contiguous().float()
        Forward = [img]
        noise = torch.randn_like(img)
        n_img = img
        for i in range(t):
            step = torch.full((batch_size,), i, dtype=torch.long, device=img.device)
            n_img = self.q_sample(x_start=img, x_end=noise, t=step)
            Forward.append(n_img)
        Backward = []
        _, out = self._reverse(batch_size, n_img, t, 1, noise, collect=lambda x1, cur, s: Backward.append(cur))
        return Forward, Backward, out
