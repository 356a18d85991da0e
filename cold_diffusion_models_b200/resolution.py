"""Drop-in `GaussianDiffusion` of resolution_diffusion_pytorch (super-resolution cold diffusion; reference:
resolution-diffusion-pytorch/resolution_diffusion_pytorch/resolution_diffusion_pytorch.py:325-767, "RS").

Every degradation step `func[i]` (RS:354-414) is `F.interpolate(size=S-d, mode)` -> `F.interpolate(size=S,
'nearest-exact')` (optionally wrapped in a 3x3 sigma-0.5 reflect blur): linear, separable and identical along both
axes, hence the cumulative degradation of a plane is A_t X A_t^T exactly as for the blur family, and the same kernels
(cd_blur_apply / cd_blur_step_down) execute q_sample and the Algorithm-1/2 loops.  The S x S step operators are
tabulated once at construction by pushing an identity through torch's own interpolate (float64, CPU), so index and
weight conventions (bicubic a=-0.75, align_corners=False, nearest-exact rounding) are the library's by construction.
"""
import ctypes as C
import numpy as np
import torch
from torch import nn
import torch.nn.functional as F

from ._lib import call, ptr, stream
from .autograd import BlurDegrade
from .deblurring import _LossFn
from .degradation import gaussian_taps, blur_matrix
from .guided import check_arguments, refuse_restore, restore_loop
from .strided import refuse_strided, reverse_levels


def step_specs(resolution_routine, timesteps, image_size):
    """(dec_size, mode, do_blur) per step -- RS:389-414 (unknown routine -> [] like the reference)."""
    out = []
    for i in range(timesteps):
        r = resolution_routine
        if r == 'Incremental':
            out.append((i, 'bicubic', False))
        elif r == 'Incremental_bilinear':
            out.append((i, 'bilinear', False))
        elif r == 'Incremental_area':
            out.append((i, 'area', False))
        elif r == 'Incremental_bicubic_with_blur':
            out.append((i, 'bicubic', True))
        elif r == 'Incremental_bilinear_with_blur':
            out.append((i, 'bilinear', True))
        elif r == 'Incremental_area_with_blur':
            out.append((i, 'area', True))
        elif r == 'Incremental_factor_2':
            out.append((image_size - image_size // 2 ** (i + 1), 'bicubic', False))
        elif r == 'Incremental_bilinear_factor_2':
            out.append((image_size - image_size // 2 ** (i + 1), 'bilinear', False))
        elif r == 'Incremental_area_factor_2':
            out.append((image_size - image_size // 2 ** (i + 1), 'area', False))
    return out


def step_matrix(S, dec_size, mode, do_blur, probe_columns=128):
    """1-D operator (S x S, float64) of one RS.transform_func step along an axis.

    The columns are probed `probe_columns` at a time: a batch holds probe_columns x S x S doubles (for the default 17 MB at
    S = 128, 67 MB at 256 and 268 MB at 512; the interpolate outputs add about as much again), where a single batch of all S
    columns would hold S^3 (1.07 GB at S = 512).  Every column is computed by the same interpolate calls whatever the
    batching, so the result does not depend on it.  The batching bounds memory, not time: the work stays S^3 per step
    (0.9 s per step at S = 512 on an 8-core x86 CPU, about 3 minutes for a T = 200 constructor)."""
    # rows of `probe[k]` are all e_k, so the 2-D separable op returns (M e_k)^T in every row (operators preserve constants)
    M = np.empty((S, S), dtype=np.float64)
    eye = torch.eye(S, dtype=torch.float64)
    for k0 in range(0, S, probe_columns):
        k1 = min(S, k0 + probe_columns)
        probe = eye[k0:k1].reshape(k1 - k0, 1, 1, S).expand(k1 - k0, 1, S, S).contiguous()
        x = F.interpolate(probe, size=S - dec_size, mode=mode, antialias=False)  # raises for size 0 like the reference
        x = F.interpolate(x, size=S, mode='nearest-exact', antialias=False)
        M[:, k0:k1] = x[:, 0, 0, :].t().numpy()                                   # M[:, k] = response to e_k
    if do_blur:
        Bm = blur_matrix(gaussian_taps(3, 0.5).double().numpy(), S, 'reflect')
        M = Bm @ M @ Bm
    return M


class GaussianDiffusion(nn.Module):
    def __init__(self, denoise_fn, *, image_size, device_of_kernel, channels=3, timesteps=1000, loss_type='l1',
                 resolution_routine='Incremental', train_routine='Final', sampling_routine='default'):
        super().__init__()
        self.channels = channels
        self.image_size = image_size
        self.denoise_fn = denoise_fn
        self.device_of_kernel = device_of_kernel
        self.num_timesteps = int(timesteps)
        self.loss_type = loss_type
        self.resolution_routine = resolution_routine
        specs = step_specs(resolution_routine, self.num_timesteps, image_size)
        ops = np.zeros((len(specs), image_size, image_size), dtype=np.float32)
        steps = np.zeros((len(specs), image_size, image_size), dtype=np.float32)
        A = np.eye(image_size)
        for i, (d, mode, blur) in enumerate(specs):
            M = step_matrix(image_size, d, mode, blur)
            steps[i] = M.astype(np.float32)
            A = M @ A
            ops[i] = A.astype(np.float32)
        self.register_buffer('_ops_cum', torch.from_numpy(ops), persistent=False)
        self.register_buffer('_ops_step', torch.from_numpy(steps), persistent=False)
        self._nsteps = len(specs)
        self.train_routine = train_routine
        self.sampling_routine = sampling_routine

    # ---- degradation ---------------------------------------------------------------------------------------
    def _apply_op(self, x, idx, per_sample_t=None):
        x = x.contiguous().float()
        B, Cc, H, W = x.shape
        out = torch.empty_like(x)
        call('cd_blur_apply', ptr(x), ptr(out), ptr(self._ops_cum), ptr(per_sample_t), int(idx), B, Cc, H, self.num_timesteps,
             0, 0, stream())
        return out

    @torch.no_grad()
    def _apply_step(self, x, i):
        """func[i]: the single degradation step i alone"""
        x = x.contiguous().float()
        B, Cc, H, W = x.shape
        out = torch.empty_like(x)
        call('cd_blur_apply', ptr(x), ptr(out), ptr(self._ops_step), ptr(None), int(i), B, Cc, H, self.num_timesteps, 0, 0, stream())
        return out

    @property
    def func(self):
        """the reference exposes `func`: a list of per-step callables img -> degraded img (RS:389-414); same here, one launch
        each (built on access so that deep copies of the module bind to the copy)"""
        import functools
        return [functools.partial(self._apply_step, i=i) for i in range(self._nsteps)]

    def get_funcs(self):
        return self.func

    @torch.no_grad()
    def transform_func(self, img, dec_size, mode, do_blur=False):
        """RS:354-387: one pixelation step with explicit parameters (shrink to S - dec_size with `mode`, back with nearest-exact,
        optionally inside a 3x3 sigma-0.5 reflect blur).  The operator is tabulated on first use and applied in one launch."""
        S = img.shape[2]
        key = (S, int(dec_size), mode, bool(do_blur))
        cache = self.__dict__.setdefault('_transform_ops', {})
        if key not in cache:
            cache[key] = torch.from_numpy(step_matrix(S, int(dec_size), mode, bool(do_blur)).astype(np.float32))[None].contiguous().to(img.device)
        x = img.contiguous().float()
        B, Cc, H, W = x.shape
        out = torch.empty_like(x)
        call('cd_blur_apply', ptr(x), ptr(out), ptr(cache[key]), ptr(None), 0, B, Cc, H, 1, 0, 0, stream())
        return out

    def q_sample(self, x_start, t):
        """RS:630-652.  Rows with t_b = -1 (the 'Step' train routine at t = 0, RS:745) were meant to pass through, but the
        reference tests the loop index instead of t (`if step != -1`, RS:645), so they take `all_blurs[-1]`: the level
        max(t) of that batch.  Reproduced here (two index ops on B int64 values, no host sync); when every t is -1 the
        reference raises inside torch.stack -- that case passes the rows through instead."""
        with torch.no_grad():
            t = t.to(device=x_start.device, dtype=torch.int64).contiguous()
            t = torch.where(t < 0, t.max().expand_as(t), t).contiguous()
            return self._apply_op(x_start, -1, per_sample_t=t)

    def degrade(self, x_start, t):
        """D(x_start_b, t_b): `q_sample`'s values bit for bit (same kernel, same level max(t) for the t = -1 rows),
        differentiable with respect to x_start (gradient A_t^T g A_t with the tabulated resize operators)."""
        x = x_start.contiguous().float()
        t = t.to(device=x.device, dtype=torch.int64).contiguous()
        t = torch.where(t < 0, t.max().expand_as(t), t).contiguous()
        return BlurDegrade.apply(x, self._ops_cum, t, -1, self.num_timesteps, 0, 0)

    def _loss(self, a, b):
        if self.loss_type == 'l1':
            return _LossFn.apply(a, b, 0)
        elif self.loss_type == 'l2':
            return _LossFn.apply(a, b, 1)
        raise NotImplementedError()

    def p_losses(self, x_start, t):
        """RS:655-761.  'Final' is the benchmarked path; the research variants are composed from the same kernels
        (their extra elementwise/statistics steps are tiny torch ops)."""
        r = self.train_routine
        if r == 'Final':
            return self._loss(x_start, self.denoise_fn(self.q_sample(x_start, t), t))
        if r == 'Final_small_noise':
            x_start = x_start + 0.001 * torch.randn_like(x_start)
            return self._loss(x_start, self.denoise_fn(self.q_sample(x_start, t), t))
        if r in ('Final_random_mean', 'Final_random_mean_and_actual'):
            loss1 = None
            if r == 'Final_random_mean_and_actual':
                loss1 = self._loss(x_start, self.denoise_fn(self.q_sample(x_start, t), t))
            mean = torch.mean(x_start, [2, 3], keepdim=True)
            x_start = x_start - mean + torch.randn_like(mean)
            loss = self._loss(x_start, self.denoise_fn(self.q_sample(x_start, t), t))
            return loss if loss1 is None else loss1 + loss
        if r == 'Gradient_norm':
            x_blur = self.q_sample(x_start, t)
            grad_pred = self.denoise_fn(x_blur, t)
            gradient = x_blur - x_start
            norm = torch.linalg.norm(gradient.flatten(1), dim=1).reshape(-1, 1, 1, 1)
            return self._loss(gradient / (norm + 1e-5), grad_pred)
        if r == 'Step':
            x_blur = self.q_sample(x_start, t)
            x_blur_sub = self.q_sample(x_start, t - 1)
            return self._loss(x_blur_sub, self.denoise_fn(x_blur, t))
        raise UnboundLocalError("local variable 'loss' referenced before assignment")   # what the reference does

    def forward(self, x, *args, **kwargs):
        b, c, h, w, device, img_size, = *x.shape, x.device, self.image_size
        assert h == img_size and w == img_size, f'height and width of image must be {img_size}'
        t = torch.randint(0, self.num_timesteps, (b,), device=device).long()
        return self.p_losses(x, t, *args, **kwargs)

    # ---- reverse process -----------------------------------------------------------------------------------
    def _reverse_step(self, img, x0_hat, t, lo=None):
        """Algorithm 1 / 2 from level t to level lo (t - 1 unless given) with the tabulated cumulative operators"""
        if lo is None:
            lo = t - 1
        if self.sampling_routine == 'default':
            return self._apply_op(x0_hat, lo - 1)
        elif self.sampling_routine == 'x0_step_down':
            out = torch.empty_like(img)
            B, Cc, H, W = img.shape
            call('cd_blur_step_down', ptr(img.contiguous()), ptr(x0_hat.contiguous()), ptr(out), ptr(self._ops_cum),
                 t - 1, lo - 1, B, Cc, H, self.num_timesteps, 0, stream())
            return out
        return x0_hat

    @torch.no_grad()
    def sample(self, batch_size=16, img=None, t=None, *, steps=None):
        """RS:417-459 -> (xt, direct_recons, img).  steps=K: K reverse steps through the levels of strided.reverse_levels
        instead of all t (None: every level, the reference's loop).  Train routines other than 'Final' (the network output is
        the next image) and unknown sampling routines have no strided form: ValueError."""
        if self.train_routine != 'Final':
            refuse_strided(steps, 'resolution', "train_routine=%r" % self.train_routine)
        if self.sampling_routine not in ('default', 'x0_step_down'):
            refuse_strided(steps, 'resolution', "sampling_routine=%r" % self.sampling_routine)
        if t is None:
            t = self.num_timesteps
        levels = reverse_levels(t, steps)
        img = self._apply_op(img, t - 1)
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
        return xt, direct_recons, img

    def restore(self, y, s, *, weight, steps=None):
        """guided restoration (guided.py) from the observation y = D_s(x), D_s = the tabulated cumulative operator s - 1 that
        `sample(img=x, t=s)` applies.  weight = 0 is `sample(img=x, t=s, steps=steps)`'s final image bit for bit.  Raises
        ValueError for the routines `sample(steps=K)` refuses."""
        if self.train_routine != 'Final':
            refuse_restore('resolution', "train_routine=%r (no strided form)" % self.train_routine)
        if self.sampling_routine not in ('default', 'x0_step_down'):
            refuse_restore('resolution', "sampling_routine=%r (no strided form)" % self.sampling_routine)
        check_arguments('resolution', y, s, weight, self.num_timesteps, (self.channels, self.image_size, self.image_size))
        s, weight = int(s), float(weight)
        levels = reverse_levels(s, steps)
        y = y.contiguous()
        B, Cc, S, _ = y.shape
        T = self.num_timesteps
        work = torch.empty_like(y) if S > 128 and weight > 0 else None

        def guide_grad(x0):
            out = torch.empty_like(x0)
            call('cd_blur_guide_grad', ptr(x0), ptr(y), ptr(out), ptr(work), ptr(self._ops_cum), s - 1, B, Cc, S, T, stream())
            return out

        def step(img, x0, g, hi, lo):
            out = torch.empty_like(img)
            xt = img.contiguous() if self.sampling_routine == 'x0_step_down' else None
            call('cd_blur_guided_step', ptr(xt), ptr(x0.contiguous()), ptr(g), C.c_float(weight), ptr(out), ptr(self._ops_cum),
                 hi - 1, lo - 1, B, Cc, S, T, stream())
            return out

        return restore_loop(self.denoise_fn, y, levels, weight, guide_grad, step)

    @torch.no_grad()
    def opt(self, img, t=None):
        if t is None:
            t = self.num_timesteps
        return self._apply_op(img, t - 1)

    def _reverse_loop(self, batch_size, img, times, collect=None):
        direct_recons = None
        while times:
            step = torch.full((batch_size,), times - 1, dtype=torch.long, device=img.device)
            x = self.denoise_fn(img, step)
            if collect is not None:
                collect(x, img)
            if direct_recons is None:
                direct_recons = x
            if self.train_routine == 'Final':
                x = self._reverse_step(img, x, times)
            img = x
            times = times - 1
        return direct_recons, img

    @torch.no_grad()
    def gen_sample(self, batch_size=16, img=None, t=None, times=None, noise_level=0):
        """RS:460-503 -> (xt, direct_recons, img): the reverse process from a given (already degraded) image plus noise"""
        if t is None:
            t = self.num_timesteps
        if times is None:
            times = t
        img = img.contiguous().float()
        img = img + torch.randn_like(img) * noise_level
        direct_recons, out = self._reverse_loop(batch_size, img, times)
        return img, direct_recons, out

    @torch.no_grad()
    def all_sample(self, batch_size=16, img=None, t=None, times=None):
        """RS:505-555 -> (X_0s, X_ts)"""
        if t is None:
            t = self.num_timesteps
        if times is None:
            times = t
        img = self._apply_op(img, t - 1)
        X_0s, X_ts = [], []
        self._reverse_loop(batch_size, img, times, collect=lambda x, cur: (X_0s.append(x), X_ts.append(cur)))
        return X_0s, X_ts

    @torch.no_grad()
    def forward_and_backward(self, batch_size=16, img=None, t=None, times=None, eval=True):
        """RS:558-616 -> (Forward, Backward, img)"""
        if eval:
            self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        if times is None:
            times = t
        img = img.contiguous().float()
        Forward = [img] + [self._apply_op(img, i) for i in range(t)]
        Backward = []
        _, out = self._reverse_loop(batch_size, Forward[-1], times, collect=lambda x, cur: Backward.append(cur))
        return Forward, Backward, out
