"""Drop-in `GaussianDiffusion` + forward processes of the snowification/ (== decolor-diffusion/) package (reference:
snowification/diffusion/diffusion.py:110-447 "SN", snowification/diffusion/forward_process_impl.py:131-372 "FP").

* `DeColorization` (FP:131-218): every step is the per-pixel channel mix f_i I + (1-f_i)/C 11^T; the cumulative mix is a
  [T][C][C] table and D(x, t_b) is ONE kernel with a per-sample step index (cd_chanmix).
* `Snow` (FP:221-372): D depends on the clean image only; the T snow layers are generated on the device (cd_snow_layers:
  scipy.ndimage.zoom's order-1 arithmetic bit for bit, threshold, clip, motion blur of all steps in two launches) from the
  random numbers the host draws exactly as the reference does (numpy generator, seed 123321 unless `random_snow`), and
  applied by cd_snow.  `random_snow=True` regenerates them in `reset_parameters`, as upstream does -- there on the host
  with scipy and T CPU convolutions per p_losses call.
* per-sample masked stepping (`sample_one_step`, `sample_multi_step`, SN:195-256) and the `t == -1` pass-through rows
  of `q_sample` (SN:344-388) become per-sample indices handed to the kernels -- no Python loop over steps, no
  `torch.where` scatter per step.  `sample()` returns the reference's dict {'xt','direct_recons','recon'}.
`to_lab=True` (kornia Lab colour path) is out of scope (SURVEY section 2.1) and raises.
"""
import ctypes as C
import numpy as np
import torch
from torch import nn
import torch.nn.functional as F

from ._lib import call, ptr, stream
from .deblurring import _LossFn
from .degradation import gaussian_taps


class ForwardProcessBase:
    def forward(self, x, i, og=None):
        pass

    @torch.no_grad()
    def reset_parameters(self, batch_size=32):
        pass


class DeColorization(ForwardProcessBase):
    def __init__(self, decolor_routine='Constant', decolor_ema_factor=0.9, decolor_total_remove=False, num_timesteps=50,
                 channels=3, to_lab=False):
        if to_lab:
            raise NotImplementedError("to_lab (kornia Lab colour path) is out of scope of the H100 engine")
        self.decolor_routine, self.decolor_ema_factor = decolor_routine, decolor_ema_factor
        self.decolor_total_remove, self.channels, self.num_timesteps = decolor_total_remove, channels, num_timesteps
        self.to_lab = to_lab
        self.factors = self.get_factors()
        # per-step fp32 mixing matrices exactly as FP:150-157 builds them, cumulative product in float64
        Cn = channels
        eye, ones = torch.eye(Cn), torch.ones((Cn, Cn)) / float(Cn)
        self.step_mats = [f * eye + (1.0 - f) * ones for f in self.factors]
        cum, A = [], np.eye(Cn)
        for M in self.step_mats:
            A = M.double().numpy() @ A
            cum.append(A.astype(np.float32))
        self.mats_cum = torch.from_numpy(np.stack(cum)) if cum else torch.zeros(0, Cn, Cn)

    def get_factors(self):
        # FP:167-187
        T, out = self.num_timesteps, []
        if self.decolor_routine == 'Constant':
            for i in range(T):
                out.append(0.0 if (i == T - 1 and self.decolor_total_remove) else self.decolor_ema_factor)
        elif self.decolor_routine == 'Linear':
            diff, start = 1.0 / T, 1.0
            for i in range(T):
                if i == T - 1 and self.decolor_total_remove:
                    out.append(0.0)
                else:
                    f = 1 - diff / start
                    start = start * f
                    out.append(f)
        return out


_SNOW_LEVELS = {   # FP:261-293: c, (thres start,end), (motion-blur sigma start,end), (brightness start,end)
    1: ((0.1, 0.3, 3, 0.5, 5, 4, 0.8), (0.7, 0.3), (0.5, 5.0), (0.95, 0.7)),
    2: ((0.55, 0.3, 2.5, 0.85, 11, 12, 0.55), (1.15, 0.7), (0.05, 12), (0.95, 0.55)),
    3: ((0.55, 0.3, 2.5, 0.7, 11, 16, 0.4), (1.15, 0.7), (0.05, 16), (0.95, 0.4)),
    4: ((0.55, 0.3, 2.5, 0.55, 11, 20, 0.3), (1.15, 0.55), (0.05, 20), (0.95, 0.3)),
}


class Snow(ForwardProcessBase):
    def __init__(self, image_size=(32, 32), snow_level=1, num_timesteps=50, snow_base_path=None, random_snow=False,
                 single_snow=False, batch_size=32, load_snow_base=False, fix_brightness=False):
        self.num_timesteps, self.random_snow, self.snow_level = num_timesteps, random_snow, snow_level
        self.image_size = image_size if isinstance(image_size, tuple) else (image_size, image_size)
        self.single_snow, self.batch_size, self.fix_brightness = single_snow, batch_size, fix_brightness
        self.generate_snow_layer()

    @torch.no_grad()
    def reset_parameters(self, batch_size=-1):
        if batch_size != -1:
            self.batch_size = batch_size
        if self.random_snow:
            self.generate_snow_layer()

    @torch.no_grad()
    def generate_snow_layer(self):
        """FP:252-355.  The host draws the random numbers exactly as the reference does (numpy global generator: one normal field
        per snow sample, then one uniform for the direction; torch.randperm per step for `single_snow`; seed 123321 unless
        `random_snow`) and keeps only the centre crop that clipped_zoom reads (FP:32-38).  Zoom, threshold, clip and motion blur
        of all T steps run on the device (cd_snow_layers) the first time the layers are needed there: `layers(device)`."""
        if not self.random_snow:
            rstate = np.random.get_state()
            np.random.seed(123321)
        c, thr, mbs, brc = _SNOW_LEVELS[self.snow_level]
        T = self.num_timesteps
        self.snow_thres_list = torch.linspace(thr[0], thr[1], T).tolist()
        self.mb_sigma_list = torch.linspace(mbs[0], mbs[1], T).tolist()
        self.br_coef_list = torch.linspace(brc[0], brc[1], T).tolist()
        h = self.image_size[0]
        if self.image_size[1] != h:
            raise ValueError("snow layers are square upstream (clipped_zoom crops both axes with shape[0]); got %r" % (self.image_size,))
        ch = int(np.ceil(h / c[2]))                                  # clipped_zoom, FP:33-41
        top = (h - ch) // 2
        m = int(round(ch * c[2]))                                    # scipy.ndimage.zoom output size
        self._geom = (ch, m, (m - h) // 2, h)
        nsb = self.batch_size if self.single_snow else 1
        crops = [np.random.normal(size=self.image_size, loc=c[0], scale=c[1])[top:top + ch, top:top + ch] for _ in range(nsb)]
        self._noise = torch.from_numpy(np.ascontiguousarray(np.stack(crops)))          # [SB][ch][ch] float64
        vertical_snow = bool(np.random.uniform() > 0.5)
        flags = torch.full((T, nsb), int(vertical_snow), dtype=torch.uint8)
        taps = []
        for i in range(T):
            taps.append(gaussian_taps(c[4], self.mb_sigma_list[i]))
            if self.single_snow:                                     # FP:340-344: a fresh half of the samples goes vertical
                vidx = torch.randperm(nsb)[:int(nsb / 2)]
                flags[i] = 0
                flags[i, vidx] = 1
        if not self.random_snow:
            np.random.set_state(rstate)
        self._taps = torch.stack(taps).float().contiguous()          # [T][k]
        self._vertical = flags.contiguous()
        self._thres = torch.tensor(self.snow_thres_list, dtype=torch.float32)
        self.br_t = torch.tensor(self.br_coef_list, dtype=torch.float32)
        self._layers = None
        self._dev = None

    def layers(self, dev):
        """[T][SB][3][H][W] fp32 on `dev` (cd_snow's layout), generated there"""
        dev = torch.device(dev)
        if self._layers is None or self._layers.device != dev:
            ch, m, trim, h = self._geom
            T, nsb = self._vertical.shape
            noise, thres, taps, vert = (t.to(dev) for t in (self._noise, self._thres, self._taps, self._vertical))
            base = torch.empty((nsb, h, h), dtype=torch.float32, device=dev)
            out = torch.empty((T, nsb, 3, h, h), dtype=torch.float32, device=dev)
            call('cd_snow_layers', ptr(noise), nsb, ch, m, trim, h, ptr(thres), ptr(taps), int(taps.shape[1]), ptr(vert), T,
                 ptr(base), ptr(out), stream())
            self._layers = out
        return self._layers

    # the reference's attributes (FP:305-306, 349-350: lists of CPU tensors), materialised on request
    @property
    def snow_t(self):
        if self._layers is None:
            self.layers('cuda' if torch.cuda.is_available() else 'cpu')
        return self._layers

    @property
    def snow(self):
        return [l.cpu() for l in self.snow_t]

    @property
    def snow_rot(self):
        return [torch.rot90(l.cpu(), k=2, dims=[2, 3]) for l in self.snow_t]


class GaussianDiffusion(nn.Module):
    def __init__(self, denoise_fn, *, image_size, device_of_kernel, one_shot_denoise_fn=None, channels=3, timesteps=1000,
                 loss_type='l1', kernel_std=0.1, kernel_size=3, forward_process_type='Decolorization',
                 train_routine='Final', sampling_routine='default', start_kernel_std=0.01, target_kernel_std=1.0,
                 decolor_routine='Constant', decolor_ema_factor=0.9, decolor_total_remove=True, snow_level=1,
                 random_snow=False, to_lab=False, order_seed=-1.0, recon_noise_std=0.0, load_snow_base=False,
                 load_path=None, batch_size=32, single_snow=False, fix_brightness=False, results_folder=None):
        super().__init__()
        self.channels = channels
        self.image_size = image_size
        self.denoise_fn = denoise_fn
        self.device_of_kernel = device_of_kernel
        self.num_timesteps = int(timesteps)
        self.loss_type = loss_type
        self.train_routine = train_routine
        self.sampling_routine = sampling_routine
        self.snow_level, self.random_snow, self.batch_size, self.single_snow = snow_level, random_snow, batch_size, single_snow
        self.to_lab = to_lab
        self.recon_noise_std = recon_noise_std
        self.forward_process_type = forward_process_type
        if forward_process_type == 'Decolorization':
            self.forward_process = DeColorization(decolor_routine=decolor_routine, decolor_ema_factor=decolor_ema_factor,
                                                  decolor_total_remove=decolor_total_remove, channels=channels,
                                                  num_timesteps=self.num_timesteps, to_lab=to_lab)
        elif forward_process_type == 'Snow':
            if to_lab:
                raise NotImplementedError("to_lab is out of scope of the H100 engine")
            self.forward_process = Snow(image_size=image_size, snow_level=snow_level, random_snow=random_snow,
                                        num_timesteps=self.num_timesteps, batch_size=batch_size, single_snow=single_snow,
                                        fix_brightness=fix_brightness)
        self._tables = None

    # ---- device tables -----------------------------------------------------------------------------------------
    def _tab(self, dev):
        fp = self.forward_process
        if self._tables is None or self._tables[0] != dev or (isinstance(fp, Snow) and fp._dev is None):
            if isinstance(fp, DeColorization):
                self._tables = (dev, fp.mats_cum.to(dev))
            else:
                self._tables = (dev, fp.layers(dev), fp.br_t.to(dev))
                fp._dev = dev
        return self._tables

    def _degrade(self, src, t_hi, hi_off, xt=None, t_lo=None, lo_off=0):
        """mode 0: D(src, t_hi+hi_off); mode 1 (xt given): xt - D(src, t_hi+hi_off) + D(src, t_lo+lo_off)"""
        src = src.contiguous().float()
        B, Cc, H, W = src.shape
        out = torch.empty_like(src)
        tab = self._tab(src.device)
        mode = 0 if xt is None else 1
        t_hi = t_hi.to(device=src.device, dtype=torch.int64).contiguous()
        t_lo = t_lo.to(device=src.device, dtype=torch.int64).contiguous() if t_lo is not None else None
        xt = xt.contiguous() if xt is not None else None
        if isinstance(self.forward_process, DeColorization):
            call('cd_chanmix', ptr(xt), ptr(src), ptr(out), ptr(tab[1]), ptr(t_hi), ptr(t_lo), hi_off, lo_off, B, Cc,
                 C.c_int64(H * W), mode, stream())
        else:
            sb = tab[1].shape[1]
            call('cd_snow', ptr(xt), ptr(src), ptr(out), ptr(tab[1]), ptr(tab[2]), ptr(t_hi), ptr(t_lo), hi_off, lo_off, B, H, W,
                 sb, int(self.forward_process.fix_brightness), mode, stream())
        return out

    # ---- forward process ------------------------------------------------------------------------------------------
    def q_sample(self, x_start, t, return_total_blur=False):
        """SN:344-388: rows with t_b == -1 pass through; the others get D(x_start_b, t_b)."""
        with torch.no_grad():
            t = t.to(x_start.device)
            if bool((t == -1).any()):
                # reference quirk (SN:373-378): row j of the filtered batch is indexed with the UNFILTERED t[j], and a -1
                # found there selects the last (fully degraded) element
                keep = t != -1
                j = torch.cumsum(keep.long(), 0) - 1                       # filtered row number of every kept row
                tj = t[j.clamp(min=0)]
                tj = torch.where(tj == -1, torch.max(t).expand_as(tj), tj)
                t = torch.where(keep, tj, t)
            out = self._degrade(x_start, t, 0)
            if return_total_blur:
                tmax = torch.where(t == -1, t, torch.max(t).expand_as(t))
                return out, self._degrade(x_start, tmax, 0)
            return out

    def loss_func(self, pred, true):
        if self.loss_type == 'l1':
            return _LossFn.apply(pred, true, 0)
        elif self.loss_type == 'l2':
            return _LossFn.apply(pred, true, 1)
        elif self.loss_type == 'sqrt':
            return _LossFn.apply(pred, true, 0).sqrt()
        raise NotImplementedError()

    def prediction_step_t(self, img, t, init_pred=None):
        return self.denoise_fn(img, t)

    def p_losses(self, x_start, t, t_pred=None):
        self.forward_process.reset_parameters()
        if self.train_routine == 'Final':
            x_blur = self.q_sample(x_start=x_start, t=t)
            return self.loss_func(x_start, self.denoise_fn(x_blur, t))
        elif self.train_routine == 'Step_Gradient':
            x_blur, x_blur_sub = self.q_sample(x_start, t), self.q_sample(x_start, t - 1)
            return self.loss_func(x_blur_sub - x_blur, self.denoise_fn(x_blur, t))
        elif self.train_routine == 'Step':
            x_blur, x_blur_sub = self.q_sample(x_start, t), self.q_sample(x_start, t - 1)
            return self.loss_func(x_blur_sub, self.denoise_fn(x_blur, t))
        raise UnboundLocalError("local variable 'loss' referenced before assignment")

    def forward(self, x, *args, **kwargs):
        b, c, h, w, device, img_size, = *x.shape, x.device, self.image_size
        img_w, img_h = img_size if type(img_size) is tuple else (img_size, img_size)
        assert h == img_h and w == img_w, f'height and width of image must be {img_size}'
        t = torch.randint(0, self.num_timesteps, (b,), device=device).long()
        return self.p_losses(x, t, None, *args, **kwargs)      # the reference's t_pred is drawn but never used (SN:440-447)

    # ---- reverse process --------------------------------------------------------------------------------------------
    @torch.no_grad()
    def sample_one_step(self, img, t, init_pred=None):
        """SN:195-245 -> (x, direct_recons); t is a per-sample int64 tensor."""
        x = self.prediction_step_t(img, t, init_pred)
        direct_recons = x.clone()
        if self.train_routine in ['Final', 'Final_random_mean', 'Final_small_noise', 'Final_random_mean_and_actual']:
            if self.sampling_routine == 'default':
                x = self._degrade(x, t, -2)                                        # t_b - 1 steps per row
            elif self.sampling_routine == 'x0_step_down':
                src = x
                if self.recon_noise_std > 0.0 and isinstance(self.forward_process, DeColorization):
                    # (Snow ignores its x argument -- FP:361-372 -- so the reconstruction noise only matters for decolor)
                    src = x + torch.normal(0.0, self.recon_noise_std, size=x.size(), device=x.device)
                # x_times_sub_1 is re-cloned from ALL rows each iteration (SN:229-233): rows that finished before the
                # last iteration end with x_times_sub_1 == x_times, i.e. the update leaves them at `img`.
                t_lo = torch.where(t == torch.max(t), t - 1, t)
                x = self._degrade(src, t, -1, xt=img, t_lo=t_lo, lo_off=-1)
        elif self.train_routine == 'Step':
            pass
        elif self.train_routine == 'Step_Gradient':
            x = img + x
        return x, direct_recons

    @torch.no_grad()
    def sample_multi_step(self, img, t_start, t_end):
        """SN:247-256"""
        fp_index = torch.where(t_start > t_end)[0]
        img_new = img.clone()
        while len(fp_index) > 0:
            _, partial = self.sample_one_step(img_new[fp_index], t_start[fp_index])
            img_new[fp_index] = partial
            t_start = t_start - 1
            fp_index = torch.where(t_start > t_end)[0]
        return img_new

    @torch.no_grad()
    def sample(self, batch_size=16, img=None, t=None):
        """SN:259-295 -> {'xt', 'direct_recons', 'recon'}"""
        self.forward_process.reset_parameters(batch_size=batch_size)
        if t is None:
            t = self.num_timesteps
        og_img = img
        tt = torch.full((img.shape[0],), t, dtype=torch.long, device=img.device)
        img = self._degrade(og_img, tt, -1)
        xt = img
        direct_recons = None
        while t:
            step = torch.full((batch_size,), t - 1, dtype=torch.long, device=img.device)
            x, cur = self.sample_one_step(img, step)
            if direct_recons is None:
                direct_recons = cur
            img = x
            t = t - 1
        return {'xt': xt, 'direct_recons': direct_recons, 'recon': img}

    def _total_forward(self, img):
        """forward_process.total_forward: decolor = every channel <- channel mean (FP:198-218, independent of the schedule);
        snow = D(img, T-1) (FP:358-359)"""
        if isinstance(self.forward_process, DeColorization):
            img = img.contiguous().float()
            B, Cc, H, W = img.shape
            mat = torch.full((1, Cc, Cc), 1.0 / Cc, device=img.device, dtype=torch.float32)
            zero = torch.zeros(B, dtype=torch.int64, device=img.device)
            out = torch.empty_like(img)
            call('cd_chanmix', ptr(None), ptr(img), ptr(out), ptr(mat), ptr(zero), ptr(None), 0, 0, B, Cc, C.c_int64(H * W), 0, stream())
            return out
        tt = torch.full((img.shape[0],), self.num_timesteps, dtype=torch.long, device=img.device)
        return self._degrade(img, tt, -1)

    @torch.no_grad()
    def all_sample(self, batch_size=16, img=None, t=None, times=None, res_dict=None):
        """SN:299-339 -> (X_0s, X_ts, init_pred_clone, img_forward_list); lists of CPU tensors.  (The reference does not pass
        the clean image to sample_one_step here, so this helper only works for decolorization there; same here.)"""
        self.forward_process.reset_parameters(batch_size=batch_size)
        if t is None:
            t = self.num_timesteps
        if times is None:
            times = t
        img = self._total_forward(img)
        X_0s, X_ts = [], []
        while times:
            step = torch.full((img.shape[0],), times - 1, dtype=torch.long, device=img.device)
            img, direct_recons = self.sample_one_step(img, step)
            X_0s.append(direct_recons.cpu())
            X_ts.append(img.cpu())
            times = times - 1
        return X_0s, X_ts, None, []

    @torch.no_grad()
    def forward_and_backward(self, batch_size=16, img=None, t=None, times=None, eval=True):
        """SN:450-490 -> (Forward, Backward, img): Algorithm 2 written with q_sample of the prediction"""
        self.denoise_fn.eval()
        if t is None:
            t = self.num_timesteps
        Forward = [img]
        n_img = img
        for i in range(t):
            step = torch.full((batch_size,), i, dtype=torch.long, device=img.device)
            n_img = self.q_sample(x_start=img, t=step)
            Forward.append(n_img)
        Backward = []
        img = n_img
        while t:
            step = torch.full((batch_size,), t - 1, dtype=torch.long, device=img.device)
            x1_bar = self.denoise_fn(img, step)
            Backward.append(img)
            xt_bar = self.q_sample(x_start=x1_bar, t=step)
            xt_sub1_bar = x1_bar
            if t - 1 != 0:
                step2 = torch.full((batch_size,), t - 2, dtype=torch.long, device=img.device)
                xt_sub1_bar = self.q_sample(x_start=xt_sub1_bar, t=step2)
            img = img - xt_bar + xt_sub1_bar
            t = t - 1
        return Forward, Backward, img
