"""Drop-in `GaussianDiffusion` of the defading-GENERATION package (reference:
defading-generation-diffusion-pytorch/defading_diffusion_pytorch/defading_diffusion_pytorch.py:285-568, "DFGEN").

The image fades towards a second image x2 (the driver uses a constant random colour, DFGEN:768-774) with a per-PIXEL
weight: alphas[t] = prod_{i<=t} K_i of the Gaussian fade kernels (DFGEN:313-344), q_sample = alphas[t_b] x1 +
(1 - alphas[t_b]) x2 (DFGEN:543-548).  The reference gathers the (1,S,S) weight planes with a Python loop over the
batch (`extract`, DFGEN:285-294); here q_sample and the Algorithm-2 update are one elementwise kernel each
(cd_fade_lerp / cd_fade_step) indexing the resident [T][S][S] tables per sample; `sample(steps=K)` strides with
cd_fade_step_to."""
import ctypes as C  # noqa: F401
import torch
from torch import nn

from ._lib import call, ptr, stream
from .autograd import LerpDegrade
from .deblurring import _LossFn
from .degradation import gaussian_taps
from .strided import reverse_levels


def get_fade_kernel(dims, std):
    # DFGEN:313-318
    gx, gy = gaussian_taps(dims[0], std[0]), gaussian_taps(dims[1], std[1])
    k = torch.matmul(gx.unsqueeze(-1), gy.unsqueeze(-1).t())
    k = k / torch.max(k)
    k = torch.ones_like(k) - k
    return k[1:, 1:]


def get_kernels_with_schedule(timesteps, size, kernel_std, initial_mask):
    # DFGEN:320-329: cumulative product, entry i = K_0 ... K_i
    out, kers = [], torch.ones((1, size, size))
    for i in range(timesteps):
        s = kernel_std * (i + initial_mask)
        kers = kers * get_fade_kernel((size + 1, size + 1), (s, s))
        out.append(kers)
    return torch.stack(out)


def get_reverse_kernels_with_schedule(timesteps, size, kernel_std, initial_mask):
    # DFGEN:331-342: entry i = product of the first i kernels, list reversed
    out, kers = [], torch.ones((1, size, size))
    for i in range(timesteps):
        out.append(kers)
        s = kernel_std * (i + initial_mask)
        kers = kers * get_fade_kernel((size + 1, size + 1), (s, s))
    out.reverse()
    return torch.stack(out)


class GaussianDiffusion(nn.Module):
    def __init__(self, denoise_fn, *, image_size, channels=3, timesteps=1000, loss_type='l1', train_routine='Final',
                 sampling_routine='default', reverse=False, kernel_std=0.15, initial_mask=11):
        super().__init__()
        self.channels = channels
        self.image_size = image_size
        self.denoise_fn = denoise_fn
        self.num_timesteps = int(timesteps)
        self.loss_type = loss_type
        self.reverse = reverse
        if self.reverse:
            one_minus_alphas = get_reverse_kernels_with_schedule(timesteps, image_size, kernel_std, initial_mask)
            alphas = 1. - one_minus_alphas
        else:
            alphas = get_kernels_with_schedule(timesteps, image_size, kernel_std, initial_mask)
            one_minus_alphas = 1. - alphas
        self.register_buffer('alphas', alphas)                       # (T,1,S,S), reference keys
        self.register_buffer('one_minus_alphas', one_minus_alphas)
        self.train_routine = train_routine
        self.sampling_routine = sampling_routine

    # ---- forward process --------------------------------------------------------------------------------------
    def _lerp(self, x_start, x_end, t):
        x_start = x_start.contiguous().float(); x_end = x_end.contiguous().float()
        B, Cc, H, W = x_start.shape
        assert H == W == self.image_size and x_end.shape == x_start.shape
        out = torch.empty_like(x_start)
        if isinstance(t, int):
            tp, ts = ptr(None), t
        else:
            t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
            tp, ts = ptr(t), 0
        call('cd_fade_lerp', ptr(x_start), ptr(x_end), tp, ts, ptr(self.alphas), ptr(self.one_minus_alphas), B, Cc, H * W,
             ptr(out), stream())
        return out

    def q_sample(self, x_start, x_end, t):
        """DFGEN:543-548; t: (B,) int64"""
        with torch.no_grad():
            return self._lerp(x_start, x_end, t)

    def degrade(self, x_start, x_end, t):
        """alphas[t_b] x_start + one_minus_alphas[t_b] x_end per pixel: `q_sample`'s values bit for bit (same kernel),
        differentiable with respect to both images"""
        x_start = x_start.contiguous().float(); x_end = x_end.contiguous().float()
        B, Cc, H, W = x_start.shape
        assert H == W == self.image_size and x_end.shape == x_start.shape
        if isinstance(t, int):
            return LerpDegrade.apply(x_start, x_end, None, t, self.alphas, self.one_minus_alphas, 1)
        t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
        return LerpDegrade.apply(x_start, x_end, t, 0, self.alphas, self.one_minus_alphas, 1)

    def get_x2_bar_from_xt(self, x1_bar, xt, t):
        # DFGEN:421-425 (API parity; no sampling loop of the reference calls it)
        a = self.alphas.index_select(0, t)
        b = self.one_minus_alphas.index_select(0, t)
        return (xt - a * x1_bar) / (b + 0.00000000000001)

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
    def _reverse(self, batch_size, img, x2, t, collect=None):
        """Algorithm 2 with the end image fixed (DFGEN:397-414): img <- img - D(x1_bar, t-1) + D(x1_bar, t-2)"""
        B, Cc, H, W = img.shape
        direct_recons = None
        while t:
            step = torch.full((batch_size,), t - 1, dtype=torch.long, device=img.device)
            x1_bar = self.denoise_fn(img, step)
            if collect is not None:
                collect(x1_bar, img)
            if direct_recons is None:
                direct_recons = x1_bar
            out = torch.empty_like(img)
            call('cd_fade_step', ptr(img), ptr(x1_bar.contiguous()), ptr(x2), t, ptr(self.alphas), ptr(self.one_minus_alphas),
                 B, Cc, H * W, ptr(out), stream())
            img = out
            t = t - 1
        return direct_recons, img

    def _reverse_strided(self, batch_size, img, x2, levels):
        """_reverse through the given levels (strided.reverse_levels): img <- img - D(x1_bar, hi) + D(x1_bar, lo) in one
        cd_fade_step_to per pair"""
        B, Cc, H, W = img.shape
        direct_recons = None
        for hi, lo in zip(levels, levels[1:]):
            step = torch.full((batch_size,), hi - 1, dtype=torch.long, device=img.device)
            x1_bar = self.denoise_fn(img, step)
            if direct_recons is None:
                direct_recons = x1_bar
            out = torch.empty_like(img)
            call('cd_fade_step_to', ptr(img), ptr(x1_bar.contiguous()), ptr(x2), hi, lo, ptr(self.alphas), ptr(self.one_minus_alphas),
                 B, Cc, H * W, ptr(out), stream())
            img = out
        return direct_recons, img

    @torch.no_grad()
    def sample(self, batch_size=16, img=None, t=None, *, steps=None):
        """DFGEN:385-418 -> (xt, direct_recons, img).  steps=K: K reverse steps through the levels of strided.reverse_levels
        (cd_fade_step_to) instead of all t (None: every level, the reference's loop)"""
        if t is None:
            t = self.num_timesteps
        levels = None if steps is None else reverse_levels(t, steps)
        self.denoise_fn.eval()
        orig = img.contiguous().float()
        if levels is None:
            direct_recons, out = self._reverse(batch_size, orig, orig, t)
        else:
            direct_recons, out = self._reverse_strided(batch_size, orig, orig, levels)
        self.denoise_fn.train()
        return orig, direct_recons, out

    @torch.no_grad()
    def gen_sample(self, batch_size=16, img=None, noise_level=0, t=None):
        """DFGEN:427-457 -> (noise, direct_recons, img)"""
        self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        noise = img.contiguous().float()
        start = noise + torch.randn_like(noise) * noise_level
        direct_recons, out = self._reverse(batch_size, start, noise, t)
        return noise, direct_recons, out

    @torch.no_grad()
    def forward_and_backward(self, batch_size=16, img1=None, img2=None, t=None, times=None, eval=True):
        """DFGEN:459-504 -> (Forward, Backward, img); the backward pass starts from img2 itself"""
        self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        img = img1.contiguous().float()
        noise = img2.contiguous().float()
        Forward = [img]
        for i in range(self.num_timesteps):
            Forward.append(self._lerp(img, noise, i))
        Backward = []
        _, out = self._reverse(batch_size, noise, noise, t, collect=lambda x1, cur: Backward.append(cur))
        return Forward, Backward, out

    @torch.no_grad()
    def all_sample(self, batch_size=16, img=None, t=None, times=None, eval=True):
        """DFGEN:506-541 -> (X1_0s, X_ts)"""
        if eval:
            self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        orig = img.contiguous().float()
        X1_0s, X_ts = [], []

        def collect(x1_bar, cur):
            X1_0s.append(x1_bar)
            X_ts.append(cur)
        self._reverse(batch_size, orig, orig, t, collect=collect)
        return X1_0s, X_ts
