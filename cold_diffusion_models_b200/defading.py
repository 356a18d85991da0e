"""Drop-in `GaussianDiffusion` of defading_diffusion_pytorch (Gaussian-mask inpainting; reference:
defading-diffusion-pytorch/defading_diffusion_pytorch/defading_diffusion_gaussian.py:298-554, "DFG").

Same constructor (`defade_fn`, `kernel_std`, `initial_mask`, `fade_routine`), `q_sample`, `p_losses`, `forward`,
`sample(batch_size, faded_recon_sample, t)`.  The fade is x * prod_i K_i: cumulative masks are tabulated once and
q_sample / the Algorithm-1/2 updates are single elementwise kernels (cd_mask_apply / cd_mask_step_down); the
'Random_*' routines index every sample's own window of the 2S x 2S masks inside the kernel (no Python B x T loop)."""
import ctypes as C
import torch
from torch import nn

from ._lib import call, ptr, stream
from .autograd import MaskDegrade, refuse_grad
from .deblurring import _LossFn
from .degradation import gaussian_taps
from .guided import check_arguments, refuse_restore, restore_loop
from .strided import refuse_strided, reverse_levels


class GaussianDiffusion(nn.Module):
    def __init__(self, defade_fn, *, image_size, device_of_kernel, channels=3, timesteps=1000, loss_type='l1',
                 kernel_std=0.1, initial_mask=11, fade_routine='Incremental', sampling_routine='default', discrete=False):
        super().__init__()
        self.channels = channels
        self.image_size = image_size
        self.defade_fn = defade_fn
        self.device_of_kernel = device_of_kernel
        self.num_timesteps = int(timesteps)
        self.loss_type = loss_type
        self.kernel_std = kernel_std
        self.initial_mask = initial_mask
        self.fade_routine = fade_routine
        self.fade_kernels = self.get_kernels()                       # [T][MS][MS], as in the reference (a plain tensor)
        cum = torch.cumprod(self.fade_kernels, dim=0) if len(self.fade_kernels) else self.fade_kernels
        self.register_buffer('_masks_cum', cum.contiguous(), persistent=False)
        self.sampling_routine = sampling_routine
        self.discrete = discrete

    def get_fade_kernel(self, dims, std):
        # DFG:328-335
        gx, gy = gaussian_taps(dims[0], std[0]), gaussian_taps(dims[1], std[1])
        k = torch.matmul(gx.unsqueeze(-1), gy.unsqueeze(-1).t())
        k = k / torch.max(k)
        k = torch.ones_like(k) - k
        return k[1:, 1:]

    def get_kernels(self):
        # DFG:337-352
        S = self.image_size
        kernels = []
        for i in range(self.num_timesteps):
            if self.fade_routine == 'Incremental':
                s = self.kernel_std * (i + self.initial_mask)
                kernels.append(self.get_fade_kernel((S + 1, S + 1), (s, s)))
            elif self.fade_routine == 'Constant':
                kernels.append(self.get_fade_kernel((S + 1, S + 1), (self.kernel_std, self.kernel_std)))
            elif self.fade_routine == 'Random_Incremental':
                s = self.kernel_std * (i + self.initial_mask)
                kernels.append(self.get_fade_kernel((2 * S + 1, 2 * S + 1), (s, s)))
        return torch.stack(kernels)

    # ---- kernels ----------------------------------------------------------------------------------------------
    def _offsets(self, batch, device):
        if 'Random' not in self.fade_routine:
            return None, None
        rx = torch.randint(0, self.image_size + 1, (batch,), device=device).long()
        ry = torch.randint(0, self.image_size + 1, (batch,), device=device).long()
        return rx, ry

    def _fade(self, x, idx, rx, ry, per_sample_t=None, quantize=False):
        x = x.contiguous().float()
        B, Cc, S, _ = x.shape
        out = torch.empty_like(x)
        call('cd_mask_apply', ptr(x), ptr(out), ptr(self._masks_cum), ptr(per_sample_t), int(idx), ptr(rx), ptr(ry),
             B, Cc, S, self._masks_cum.shape[-1], int(quantize), stream())
        return out

    def q_sample(self, x_start, t, _offsets=None):
        """DFG:495-533"""
        with torch.no_grad():
            rx, ry = _offsets if _offsets is not None else self._offsets(x_start.size(0), x_start.device)
            t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
            return self._fade(x_start, -1, rx, ry, per_sample_t=t, quantize=self.discrete)

    def degrade(self, x_start, t, _offsets=None):
        """D(x_start_b, t_b) = x_start * mask: `q_sample`'s values bit for bit (same kernel, same per-sample windows of the
        'Random_*' routines -- pass the same `_offsets`), differentiable with respect to x_start.  `discrete` (8-bit
        truncation) raises when a gradient is requested."""
        if self.discrete:
            refuse_grad("the `discrete` 8-bit truncation", x_start)
        rx, ry = _offsets if _offsets is not None else self._offsets(x_start.size(0), x_start.device)
        t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
        return MaskDegrade.apply(x_start.contiguous().float(), self._masks_cum, t, rx, ry, self.discrete)

    def p_losses(self, x_start, t):
        x_fade = self.q_sample(x_start=x_start, t=t)
        x_recon = self.defade_fn(x_fade, t)
        if self.loss_type == 'l1':
            return _LossFn.apply(x_start, x_recon, 0)
        elif self.loss_type == 'l2':
            return _LossFn.apply(x_start, x_recon, 1)
        raise NotImplementedError()

    def forward(self, x, *args, **kwargs):
        b, c, h, w, device, img_size, = *x.shape, x.device, self.image_size
        assert h == img_size and w == img_size, f'height and width of image must be {img_size}'
        t = torch.randint(0, self.num_timesteps, (b,), device=device).long()
        return self.p_losses(x, t, *args, **kwargs)

    @torch.no_grad()
    def sample(self, batch_size=16, faded_recon_sample=None, t=None, _offsets=None, *, steps=None):
        """DFG:355-424 -> (xt, direct_recons, recon_sample).  steps=K: K reverse steps through the levels of
        strided.reverse_levels instead of all t (None: every level, the reference's loop); the 'Random_*' routines keep one
        window per sample for the whole loop.  Unknown sampling routines (which leave x as it is) raise ValueError with it."""
        if self.sampling_routine not in ('default', 'x0_step_down'):
            refuse_strided(steps, 'defading', "sampling_routine=%r" % self.sampling_routine)
        if t is None:
            t = self.num_timesteps
        levels = reverse_levels(t, steps)
        x = faded_recon_sample
        rx, ry = _offsets if _offsets is not None else self._offsets(batch_size, x.device)
        x = self._fade(x, t - 1, rx, ry, quantize=self.discrete)
        xt = x
        direct_recons = None
        recon = None
        B, Cc, S, _ = x.shape
        MS = self._masks_cum.shape[-1]
        for hi, lo in zip(levels, levels[1:]):
            step = torch.full((batch_size,), hi - 1, dtype=torch.long, device=x.device)
            recon = self.defade_fn(x, step)
            if direct_recons is None:
                direct_recons = recon
            if self.sampling_routine == 'default':
                x = self._fade(recon, lo - 1, rx, ry)
            elif self.sampling_routine == 'x0_step_down':
                out = torch.empty_like(x)
                call('cd_mask_step_down', ptr(x.contiguous()), ptr(recon.contiguous()), ptr(out), ptr(self._masks_cum),
                     hi - 1, lo - 1, ptr(rx), ptr(ry), B, Cc, S, MS, stream())
                x = out
            recon = x
        return xt, direct_recons, recon

    def restore(self, y, s, *, weight, steps=None, _offsets=None):
        """guided restoration (guided.py) from the observation y = D_s(x) = x * mask_{s-1}, the fade `sample(faded_recon_sample=x,
        t=s)` applies, in each sample's window of the 'Random_*' routines (`_offsets`, as `sample` takes them; drawn when None).
        weight = 0 is `sample`'s final image bit for bit.  Raises ValueError for `discrete` and for the routines
        `sample(steps=K)` refuses."""
        if self.discrete:
            refuse_restore('defading', "discrete=True (the 8-bit truncation has no gradient)")
        if self.sampling_routine not in ('default', 'x0_step_down'):
            refuse_restore('defading', "sampling_routine=%r (no strided form)" % self.sampling_routine)
        check_arguments('defading', y, s, weight, self.num_timesteps, (self.channels, self.image_size, self.image_size))
        s, weight = int(s), float(weight)
        levels = reverse_levels(s, steps)
        y = y.contiguous()
        B, Cc, S, _ = y.shape
        MS = self._masks_cum.shape[-1]
        rx, ry = _offsets if _offsets is not None else self._offsets(B, y.device)

        def guide_grad(x0):
            out = torch.empty_like(x0)
            call('cd_mask_guide_grad', ptr(x0), ptr(y), ptr(out), ptr(self._masks_cum), s - 1, ptr(rx), ptr(ry), B, Cc, S, MS,
                 stream())
            return out

        def step(img, x0, g, hi, lo):
            out = torch.empty_like(img)
            xt = img.contiguous() if self.sampling_routine == 'x0_step_down' else None
            call('cd_mask_guided_step', ptr(xt), ptr(x0.contiguous()), ptr(g), C.c_float(weight), ptr(out), ptr(self._masks_cum),
                 hi - 1, lo - 1, ptr(rx), ptr(ry), B, Cc, S, MS, stream())
            return out

        return restore_loop(self.defade_fn, y, levels, weight, guide_grad, step)

    @torch.no_grad()
    def all_sample(self, batch_size=16, faded_recon_sample=None, t=None, times=None, _offsets=None):
        """DFG:428-494 -> (x0_list, xt_list): every step's reconstruction and the faded sample AFTER that step's update"""
        x = faded_recon_sample
        rx, ry = _offsets if _offsets is not None else self._offsets(batch_size, x.device)
        if t is None:
            t = self.num_timesteps
        if times is None:
            times = t
        x = self._fade(x, t - 1, rx, ry, quantize=self.discrete)
        B, Cc, S, _ = x.shape
        MS = self._masks_cum.shape[-1]
        x0_list, xt_list = [], []
        while times:
            step = torch.full((batch_size,), times - 1, dtype=torch.long, device=x.device)
            recon = self.defade_fn(x, step)
            x0_list.append(recon)
            if self.sampling_routine == 'default':
                x = self._fade(recon, times - 2, rx, ry)
            elif self.sampling_routine == 'x0_step_down':
                out = torch.empty_like(x)
                call('cd_mask_step_down', ptr(x.contiguous()), ptr(recon.contiguous()), ptr(out), ptr(self._masks_cum),
                     times - 1, times - 2, ptr(rx), ptr(ry), B, Cc, S, MS, stream())
                x = out
            xt_list.append(x)
            times -= 1
        return x0_list, xt_list
