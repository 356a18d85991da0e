"""Drop-in `GaussianDiffusion` for deblurring_diffusion_pytorch (reference:
deblurring-diffusion-pytorch/deblurring_diffusion_pytorch/deblurring_diffusion_pytorch.py:311-981, "DB").

Same constructor, attributes, method names and return values as the reference class; the degradation
schedule D(x,t), q_sample, the Algorithm-1/Algorithm-2 sampling loops and the loss run in libcolddiff
(cd_blur_apply / cd_blur_step_down / cd_loss_fwd_bwd) and the restoration network is whatever
`denoise_fn` is (normally cold_diffusion_models_b200.Unet).
"""
import ctypes as C
import torch
from torch import nn
import torch.nn.functional as F  # noqa: F401  (kept for API familiarity; not used on the hot path)

from ._lib import call, ptr, stream
from .autograd import BlurDegrade, refuse_grad
from .degradation import build_blur_operators
from .guided import check_arguments, refuse_restore, restore_loop
from .strided import refuse_strided, reverse_levels


class _LossFn(torch.autograd.Function):
    """loss = mean|x0 - xhat| (l1) or mean (x0 - xhat)^2 (l2) (DB:968-971), gradient produced in the same kernel."""

    @staticmethod
    def forward(ctx, x_start, x_recon, mode):
        x_start = x_start.contiguous(); x_recon = x_recon.contiguous()
        loss = torch.zeros((), device=x_recon.device, dtype=torch.float32)
        dx = torch.empty_like(x_recon) if x_recon.requires_grad else None
        call('cd_loss_fwd_bwd', ptr(x_start), ptr(x_recon), C.c_int64(x_recon.numel()), mode, C.c_float(1.0),
             ptr(loss), ptr(dx), stream())
        ctx.dx = dx
        return loss

    @staticmethod
    def backward(ctx, g):
        dx = ctx.dx
        if dx is None:
            return None, None, None
        return None, dx * g, None


class GaussianDiffusion(nn.Module):
    def __init__(self, denoise_fn, *, image_size, device_of_kernel, channels=3, timesteps=1000, loss_type='l1',
                 kernel_std=0.1, kernel_size=3, blur_routine='Incremental', train_routine='Final',
                 sampling_routine='default', discrete=False):
        super().__init__()
        self.channels = channels
        self.image_size = image_size
        self.denoise_fn = denoise_fn
        self.device_of_kernel = device_of_kernel
        self.num_timesteps = int(timesteps)
        self.loss_type = loss_type
        self.kernel_std = kernel_std
        self.kernel_size = kernel_size
        self.blur_routine = blur_routine
        ops_cum, ops_single, taps, sched = build_blur_operators(blur_routine, self.num_timesteps, kernel_size,
                                                                kernel_std, image_size)
        self._taps, self._sched = taps, sched
        # the reference keeps the step kernels as Conv2d parameters inside the state_dict (DB:341,351-361)
        self.gaussian_kernels = nn.ModuleList(self.get_kernels())
        self.register_buffer('_ops_cum', ops_cum, persistent=False)
        self.register_buffer('_ops_single', ops_single if ops_single is not None else torch.zeros(0), persistent=False)
        self.train_routine = train_routine
        self.sampling_routine = sampling_routine
        self.discrete = discrete

    # ---- reference-compatible kernel containers (never executed) ---------------------------------
    def blur(self, dims, std):
        from .degradation import gaussian_taps
        gx, gy = gaussian_taps(dims[0], std[0]), gaussian_taps(dims[1], std[1])
        return torch.matmul(gx.unsqueeze(-1), gy.unsqueeze(-1).t())

    def get_conv(self, dims, std, mode='circular'):
        kernel = self.blur(dims, std)
        conv = nn.Conv2d(in_channels=self.channels, out_channels=self.channels, kernel_size=dims,
                         padding=int((dims[0] - 1) / 2), padding_mode=mode, bias=False, groups=self.channels)
        with torch.no_grad():
            conv.weight = nn.Parameter(kernel[None, None].repeat(self.channels, 1, 1, 1))
        return conv

    def get_kernels(self):
        return [self.get_conv((k, k), (s, s), mode=m) for (k, s, m) in self._sched]

    # ---- degradation -------------------------------------------------------------------------------
    def _apply_op(self, x, idx, *, per_sample_t=None, single=False, quantize=False, collapse=True):
        """out = A_idx x A_idx^T per plane (idx < 0: identity).  per_sample_t: int64 (B,) indices.
        collapse=False skips the `discrete` mean-collapse at idx == T-1."""
        x = x.contiguous().float()
        B, Cc, H, W = x.shape
        assert H == W == self.image_size and Cc == self.channels
        out = torch.empty_like(x)
        ops = self._ops_single if single else self._ops_cum
        T = self.num_timesteps
        call('cd_blur_apply', ptr(x), ptr(out), ptr(ops), ptr(per_sample_t), int(idx), B, Cc, H, T,
             int(self.discrete and not single and collapse), int(quantize), stream())
        return out

    def _degrade_to(self, img, t):
        """x_t from a clean image: head of sample()/opt() (DB:401-407, 595-607)."""
        if self.blur_routine == 'Individual_Incremental':
            return self._apply_op(img, (t - 1) % self.num_timesteps, single=True)
        return self._apply_op(img, t - 1)

    @torch.no_grad()
    def opt(self, img, t=None):
        if t is None:
            t = self.num_timesteps
        return self._degrade_to(img, t)

    def q_sample(self, x_start, t):
        """DB:927-960: x_{t_b} = D(x_start_b, t_b) per sample (+ `discrete` mean-collapse at T-1 and 8-bit truncation)."""
        with torch.no_grad():
            t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
            return self._apply_op(x_start, -1, per_sample_t=t, quantize=self.discrete)

    def degrade(self, x_start, t):
        """D(x_start_b, t_b): `q_sample`'s values bit for bit (same kernel), differentiable with respect to x_start, with the
        gradient A_t^T g A_t.  For reconstruction guidance and for inverting the degradation by gradient descent; q_sample itself
        stays detached, as the reference's is.  `discrete` (8-bit truncation, zero derivative almost everywhere) raises when a
        gradient is requested."""
        if self.discrete:
            refuse_grad("the `discrete` 8-bit truncation", x_start)
        x = x_start.contiguous().float()
        assert x.shape[1:] == (self.channels, self.image_size, self.image_size)
        t = t.to(device=x.device, dtype=torch.int64).contiguous()
        return BlurDegrade.apply(x, self._ops_cum, t, -1, self.num_timesteps, self.discrete, self.discrete)

    def p_losses(self, x_start, t):
        if self.train_routine == 'Final':
            x_blur = self.q_sample(x_start=x_start, t=t)
            x_recon = self.denoise_fn(x_blur, t)
            if self.loss_type == 'l1':
                loss = _LossFn.apply(x_start, x_recon, 0)
            elif self.loss_type == 'l2':
                loss = _LossFn.apply(x_start, x_recon, 1)
            else:
                raise NotImplementedError()
        return loss

    def forward(self, x, *args, **kwargs):
        b, c, h, w, device, img_size, = *x.shape, x.device, self.image_size
        assert h == img_size and w == img_size, f'height and width of image must be {img_size}'
        t = torch.randint(0, self.num_timesteps, (b,), device=device).long()
        return self.p_losses(x, t, *args, **kwargs)

    # ---- reverse process -----------------------------------------------------------------------------
    def _reverse_step(self, img, x0_hat, t, lo=None):
        """one step of Algorithm 1 ('default') or Algorithm 2 ('x0_step_down') (DB:428-451) from level t to level lo
        (t - 1 unless given: the strided loop of `sample(steps=...)`)"""
        T = self.num_timesteps
        if lo is None:
            lo = t - 1
        if self.sampling_routine == 'default':
            if self.blur_routine == 'Individual_Incremental':
                return self._apply_op(x0_hat, (lo - 1) % T, single=True)
            return self._apply_op(x0_hat, lo - 1)
        elif self.sampling_routine == 'x0_step_down':
            return self._step_down(img, x0_hat, t, lo)
        return x0_hat          # unknown routine: the reference leaves x = x0_hat

    def _step_down(self, img, x0_hat, t, lo=None):
        """Algorithm 2: x_{lo} = x_t - D(x0_hat, t) + D(x0_hat, lo) with the cumulative operators, lo = t-1 unless given
        (DB:436-451)"""
        if lo is None:
            lo = t - 1
        out = torch.empty_like(img)
        B, Cc, H, W = img.shape
        call('cd_blur_step_down', ptr(img.contiguous()), ptr(x0_hat.contiguous()), ptr(out), ptr(self._ops_cum),
             t - 1, lo - 1, B, Cc, H, self.num_timesteps, int(self.discrete), stream())
        return out

    def _check_strided(self, steps):
        """the routines whose one-step update has no strided counterpart (ValueError when steps is given): train routines other
        than 'Final' (the network output is the next image), unknown sampling routines (x = x0_hat), and 'default' with
        'Individual_Incremental' blur, whose update applies the single kernel K_{t-2} (K_{T-1} at the last step) rather
        than D(x0_hat, t-1).  Its 'x0_step_down' forms D(x0_hat, s) from the cumulative operators, as q_sample does."""
        if self.train_routine != 'Final':
            refuse_strided(steps, 'deblurring', "train_routine=%r" % self.train_routine)
        if self.sampling_routine not in ('default', 'x0_step_down'):
            refuse_strided(steps, 'deblurring', "sampling_routine=%r" % self.sampling_routine)
        if self.sampling_routine == 'default' and self.blur_routine == 'Individual_Incremental':
            refuse_strided(steps, 'deblurring', "sampling_routine='default' with blur_routine='Individual_Incremental'")

    @torch.no_grad()
    def sample(self, batch_size=16, img=None, t=None, _noise=None, *, steps=None):
        """DB:393-455 -> (xt, direct_recons, img).  steps=K: K reverse steps through the levels of strided.reverse_levels
        instead of all t (None: every level, the reference's loop)"""
        if t is None:
            t = self.num_timesteps
        self._check_strided(steps)
        levels = reverse_levels(t, steps)
        self.denoise_fn.eval()
        img = self._degrade_to(img, t)
        if self.discrete:
            img = torch.mean(img, [2, 3], keepdim=True).expand_as(img).contiguous()
        if _noise is not None:
            img = img + _noise
        xt = img
        direct_recons = None
        for hi, lo in zip(levels, levels[1:]):
            step = torch.full((batch_size,), hi - 1, dtype=torch.long, device=img.device)
            x = self.denoise_fn(img, step)
            if self.train_routine == 'Final':
                if direct_recons is None:
                    direct_recons = x
                x = self._reverse_step(img, x, hi, lo)
            img = x
        self.denoise_fn.train()
        return xt, direct_recons, img

    def restore(self, y, s, *, weight, steps=None):
        """guided restoration (guided.py): Algorithm 2 from the observation y = D_s(x) through the levels of
        strided.reverse_levels(s, steps), each step pulled towards D_s(x0_hat) = y with the guidance weight.  D_s is what
        `sample(img=x, t=s)` applies to x: the cumulative operator s - 1 (Individual_Incremental: the single kernel (s - 1) % T).
        weight = 0 is `sample(img=x, t=s, steps=steps)`'s final image bit for bit.  Raises ValueError for `discrete` and for
        the routines `sample(steps=K)` refuses."""
        if self.discrete:
            refuse_restore('deblurring', "discrete=True (the 8-bit truncation has no gradient)")
        try:
            self._check_strided(1)           # the routines without a strided form
        except ValueError:
            refuse_restore('deblurring', "train_routine=%r, sampling_routine=%r, blur_routine=%r (no strided form)" % (
                self.train_routine, self.sampling_routine, self.blur_routine))
        check_arguments('deblurring', y, s, weight, self.num_timesteps, (self.channels, self.image_size, self.image_size))
        s, weight = int(s), float(weight)
        levels = reverse_levels(s, steps)
        y = y.contiguous()
        B, Cc, S, _ = y.shape
        T = self.num_timesteps
        single = self.blur_routine == 'Individual_Incremental'
        obs_ops, obs_idx = (self._ops_single, (s - 1) % T) if single else (self._ops_cum, s - 1)
        work = torch.empty_like(y) if S > 128 and weight > 0 else None

        def guide_grad(x0):
            out = torch.empty_like(x0)
            call('cd_blur_guide_grad', ptr(x0), ptr(y), ptr(out), ptr(work), ptr(obs_ops), obs_idx, B, Cc, S, T, stream())
            return out

        def step(img, x0, g, hi, lo):
            out = torch.empty_like(img)
            xt = img.contiguous() if self.sampling_routine == 'x0_step_down' else None
            call('cd_blur_guided_step', ptr(xt), ptr(x0.contiguous()), ptr(g), C.c_float(weight), ptr(out), ptr(self._ops_cum),
                 hi - 1, lo - 1, B, Cc, S, T, stream())
            return out

        self.denoise_fn.eval()
        img = restore_loop(self.denoise_fn, y, levels, weight, guide_grad, step)
        self.denoise_fn.train()
        return img

    @torch.no_grad()
    def gen_sample(self, batch_size=16, img=None, t=None, noise_level=0):
        """DB:526-593: `sample` from a noised degraded start (the reference does not switch back to train mode)."""
        if t is None:
            t = self.num_timesteps
        shape = (img.shape[0], self.channels, self.image_size, self.image_size)
        noise = torch.randn(shape, device=img.device) * noise_level
        return self.sample(batch_size=batch_size, img=img, t=t, _noise=noise)

    gen_sample_2 = gen_sample      # DB:457-524 computes the same thing

    @torch.no_grad()
    def all_sample(self, batch_size=16, img=None, t=None, times=None, eval=True):
        """DB:609-689 -> (X_0s, X_ts)"""
        if eval:
            self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        if times is None:
            times = t
        img = self._degrade_to(img, t)
        X_0s, X_ts = [], []
        noise = None
        if self.discrete:
            img = torch.mean(img, [2, 3], keepdim=True).expand_as(img).contiguous()
            noise = torch.randn_like(img) * 0.001
            img = img + noise
        while times:
            step = torch.full((batch_size,), times - 1, dtype=torch.long, device=img.device)
            x = self.denoise_fn(img, step)
            X_0s.append(x)
            X_ts.append(img)
            if self.train_routine == 'Final':
                if self.blur_routine == 'Individual_Incremental' and self.sampling_routine in ('default', 'x0_step_down'):
                    if times - 2 >= 0:          # NB: the reference blurs `img`, not x (DB:646-647, 655-657)
                        x = self._apply_op(img, times - 2, single=True)
                else:
                    x = self._reverse_step(img, x, times)
            img = x
            times = times - 1
        if self.discrete:
            img = img - noise
        X_0s.append(img)
        self.denoise_fn.train()
        return X_0s, X_ts

    def _range_operator(self, start, t):
        """K_{t-1} ... K_{start} as a one-entry operator table (host float64 product, cached): the partial blur of
        `sample_from_blur(start=...)`, DB:877-879"""
        from .degradation import blur_matrix
        import numpy as np
        key = (start, t)
        cache = self.__dict__.setdefault('_range_ops', {})
        if key not in cache:
            S = self.image_size
            A = np.eye(S, dtype=np.float64)
            for i in range(start, t):
                k, sgm, mode = self._sched[i]
                A = blur_matrix(self._taps[i].double().numpy(), S, mode) @ A
            cache[key] = torch.from_numpy(A.astype(np.float32))[None].contiguous().to(self._ops_cum.device)
        return cache[key]

    @torch.no_grad()
    def sample_from_blur(self, batch_size=16, img=None, t=None, times=None, eval=True, start=None):
        """DB:863-925 -> (xt, direct_recons, img): blur with the kernels start .. t-1 only, then the reverse process from t"""
        if eval:
            self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        if start is None:
            start = 0
        img = img.contiguous().float()
        if start < t:
            if start == 0 and self.blur_routine != 'Individual_Incremental':
                img = self._apply_op(img, t - 1, collapse=False)
            else:
                B, Cc, H, W = img.shape
                out = torch.empty_like(img)
                call('cd_blur_apply', ptr(img), ptr(out), ptr(self._range_operator(start, t)), ptr(None), 0, B, Cc, H, 1, 0, 0, stream())
                img = out
        if self.discrete:
            img = torch.mean(img, [2, 3], keepdim=True).expand_as(img).contiguous()
        xt = img
        direct_recons = None
        while t:
            step = torch.full((batch_size,), t - 1, dtype=torch.long, device=img.device)
            x = self.denoise_fn(img, step)
            if self.train_routine == 'Final':
                if direct_recons is None:
                    direct_recons = x
                x = self._reverse_step(img, x, t)
            img = x
            t = t - 1
        return xt, direct_recons, img

    def _forward_trajectory(self, img, t):
        """[x, D(x,1), ..., D(x,t)] of the cover figures: each entry from the cumulative operator in one launch
        (the reference chains t convolutions, DB:707-711); no `discrete` collapse inside the forward pass."""
        return [img] + [self._apply_op(img, i, collapse=False) for i in range(t)]

    @torch.no_grad()
    def forward_and_backward(self, batch_size=16, img=None, noise_level=0, t=None, times=None, eval=True):
        """DB:691-770 -> (Forward, Backward, img)"""
        if eval:
            self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        if times is None:
            times = t
        img = img.contiguous().float()
        if self.blur_routine == 'Individual_Incremental':
            Forward = [img]
            img = self._apply_op(img, (t - 1) % self.num_timesteps, single=True)
        else:
            Forward = self._forward_trajectory(img, t)
            img = Forward[-1]
        Backward = []
        if self.discrete:
            img = torch.mean(img, [2, 3], keepdim=True).expand_as(img).contiguous()
            img = img + torch.randn_like(img) * noise_level
        while times:
            step = torch.full((batch_size,), times - 1, dtype=torch.long, device=img.device)
            x = self.denoise_fn(img, step)
            Backward.append(img)
            if self.train_routine == 'Final':
                if self.blur_routine == 'Individual_Incremental' and self.sampling_routine in ('default', 'x0_step_down'):
                    if times - 2 >= 0:          # the reference blurs `img`, not x (DB:735-737, 747-749)
                        x = self._apply_op(img, times - 2, single=True)
                else:
                    x = self._reverse_step(img, x, times)
            img = x
            times = times - 1
        return Forward, Backward, img

    @torch.no_grad()
    def forward_and_backward_2(self, batch_size=16, img=None, noise_level=0, eval=True):
        """DB:772-861 -> (Forward, Backward_1, Backward_2, img_1, img_2): Algorithm 1 and Algorithm 2 from the same start"""
        if eval:
            self.denoise_fn.eval()
        T = self.num_timesteps
        img = img.contiguous().float()
        Forward = self._forward_trajectory(img, T)
        img = Forward[-1]
        if self.discrete:
            img = torch.mean(img, [2, 3], keepdim=True).expand_as(img).contiguous()
            img = img + torch.randn_like(img) * noise_level
        last_img = img
        Backward_1, Backward_2 = [], []
        times = T
        while times:                            # Algorithm 1: x <- D(x0_hat, times-1)   (`img - img + ...`, DB:826)
            step = torch.full((batch_size,), times - 1, dtype=torch.long, device=img.device)
            x = self.denoise_fn(img, step)
            Backward_1.append(img)
            img = self._apply_op(x, times - 2, collapse=False)
            times = times - 1
        img_1 = img
        times, img = T, last_img
        while times:                            # Algorithm 2
            step = torch.full((batch_size,), times - 1, dtype=torch.long, device=img.device)
            x = self.denoise_fn(img, step)
            Backward_2.append(img)
            img = self._step_down(img, x, times)
            times = times - 1
        return Forward, Backward_1, Backward_2, img_1, img
