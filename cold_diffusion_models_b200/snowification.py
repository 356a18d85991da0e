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
* `to_lab=True` (Lab colour path): the tensors the process sees hold Lab values.  A decolorization step is then
  rgb2lab(M_i lab2rgb(x)) (FP:189-195), nonlinear because lab2rgb clamps and clips at every step, so D(x, t_b) runs the
  per-step chain per pixel in registers (cd_chanmix_lab) instead of one cumulative matrix.  Snow takes no `to_lab`
  upstream and applies its operator to whatever the tensor holds; for both processes `sample` / `all_sample` convert
  their outputs back with lab2rgb (SN:287-290, 331-336).  `rgb2lab` / `lab2rgb` below are diffusion/utils.py's.
"""
import ctypes as C
import numpy as np
import torch
from torch import nn
import torch.nn.functional as F

from ._lib import call, ptr, stream
from .autograd import ChanmixDegrade, refuse_grad
from .deblurring import _LossFn
from .degradation import gaussian_taps
from .guided import check_arguments, refuse_restore, restore_loop
from .strided import refuse_strided, reverse_levels
from .train_graph import recording


def _lab_convert(image, to_lab, clip=True):
    if not torch.is_tensor(image):
        raise TypeError(f"Input type is not a torch.Tensor. Got {type(image)}")
    if image.dim() < 3 or image.shape[-3] != 3:
        raise ValueError(f"Input size must have a shape of (*, 3, H, W). Got {image.shape}")
    if not image.is_cuda:
        raise RuntimeError("rgb2lab / lab2rgb run on a CUDA device (H100) only; got %s" % image.device)
    x = image.contiguous().float()
    out = torch.empty_like(x)
    B = x.numel() // (3 * x.shape[-1] * x.shape[-2]) if x.numel() else 0
    call('cd_lab_convert', ptr(x), ptr(out), B, C.c_int64(x.shape[-1] * x.shape[-2]), int(to_lab), int(bool(clip)), stream())
    return out


def rgb2lab(image):
    """diffusion/utils.py:113-163: RGB in [-1, 1], shape (*, 3, H, W) -> Lab (L in 0..100), D65 white point"""
    return _lab_convert(image, True)


def lab2rgb(image, clip=True):
    """diffusion/utils.py:166-222: Lab, shape (*, 3, H, W) -> RGB in [-1, 1] (2 rgb - 1; rgb clipped to [0, 1] when `clip`)"""
    return _lab_convert(image, False, clip)


class ForwardProcessBase:
    def forward(self, x, i, og=None):
        pass

    @torch.no_grad()
    def reset_parameters(self, batch_size=32):
        pass


class DeColorization(ForwardProcessBase):
    def __init__(self, decolor_routine='Constant', decolor_ema_factor=0.9, decolor_total_remove=False, num_timesteps=50,
                 channels=3, to_lab=False):
        if to_lab and channels != 3:
            raise ValueError("to_lab needs 3-channel images, got channels=%d" % channels)
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
        # the per-step table of the Lab path (cd_chanmix_lab): Lab steps do not compose into cumulative matrices
        self.mats_step = torch.stack(self.step_mats).contiguous() if self.step_mats else torch.zeros(0, Cn, Cn)

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

    def layers(self, dev, out=None):
        """[T][SB][3][H][W] fp32 on `dev` (cd_snow's layout), generated there.  `out`: generate into this tensor instead of a
        new cached one (the persistent buffer a captured training step reads)"""
        dev = torch.device(dev)
        if out is not None or self._layers is None or self._layers.device != dev:
            ch, m, trim, h = self._geom
            T, nsb = self._vertical.shape
            noise, thres, taps, vert = (t.to(dev) for t in (self._noise, self._thres, self._taps, self._vertical))
            base = torch.empty((nsb, h, h), dtype=torch.float32, device=dev)
            dst = torch.empty((T, nsb, 3, h, h), dtype=torch.float32, device=dev) if out is None else out
            call('cd_snow_layers', ptr(noise), nsb, ch, m, trim, h, ptr(thres), ptr(taps), int(taps.shape[1]), ptr(vert), T,
                 ptr(base), ptr(dst), stream())
            if out is not None:
                return out
            self._layers = dst
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
            # the reference passes no `to_lab` to Snow: the snow operator acts on the tensor as it is (FP:361-372)
            self.forward_process = Snow(image_size=image_size, snow_level=snow_level, random_snow=random_snow,
                                        num_timesteps=self.num_timesteps, batch_size=batch_size, single_snow=single_snow,
                                        fix_brightness=fix_brightness)
        self._tables = None

    # ---- device tables -----------------------------------------------------------------------------------------
    def _tab(self, dev):
        fp = self.forward_process
        if self._tables is None or self._tables[0] != dev or (isinstance(fp, Snow) and fp._dev is None):
            if isinstance(fp, DeColorization):
                self._tables = (dev, (fp.mats_step if self._lab_decolor() else fp.mats_cum).to(dev))
            else:
                self._tables = (dev, fp.layers(dev), fp.br_t.to(dev))
                fp._dev = dev
        return self._tables

    def _lab_decolor(self):
        return self.to_lab and isinstance(self.forward_process, DeColorization)

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
        if self._lab_decolor():
            call('cd_chanmix_lab', ptr(xt), ptr(src), ptr(out), ptr(tab[1]), ptr(t_hi), ptr(t_lo), hi_off, lo_off, B,
                 C.c_int64(H * W), mode, stream())
        elif isinstance(self.forward_process, DeColorization):
            call('cd_chanmix', ptr(xt), ptr(src), ptr(out), ptr(tab[1]), ptr(t_hi), ptr(t_lo), hi_off, lo_off, B, Cc,
                 C.c_int64(H * W), mode, stream())
        else:
            sb = tab[1].shape[1]
            call('cd_snow', ptr(xt), ptr(src), ptr(out), ptr(tab[1]), ptr(tab[2]), ptr(t_hi), ptr(t_lo), hi_off, lo_off, B, H, W,
                 sb, int(self.forward_process.fix_brightness), mode, stream())
        return out

    # ---- forward process ------------------------------------------------------------------------------------------
    @staticmethod
    def _q_sample_index(t):
        """the per-row index q_sample degrades to (-1: the row passes through)"""
        # a captured training step runs the body unconditionally (no host sync): it maps t to itself when no row is -1
        if recording() is not None or bool((t == -1).any()):
            # reference quirk (SN:373-378): row j of the filtered batch is indexed with the UNFILTERED t[j], and a -1
            # found there selects the last (fully degraded) element
            keep = t != -1
            j = torch.cumsum(keep.long(), 0) - 1                       # filtered row number of every kept row
            tj = t[j.clamp(min=0)]
            tj = torch.where(tj == -1, torch.max(t).expand_as(tj), tj)
            t = torch.where(keep, tj, t)
        return t

    def q_sample(self, x_start, t, return_total_blur=False):
        """SN:344-388: rows with t_b == -1 pass through; the others get D(x_start_b, t_b)."""
        with torch.no_grad():
            t = self._q_sample_index(t.to(x_start.device))
            out = self._degrade(x_start, t, 0)
            if return_total_blur:
                tmax = torch.where(t == -1, t, torch.max(t).expand_as(t))
                return out, self._degrade(x_start, tmax, 0)
            return out

    def degrade(self, x_start, t):
        """`q_sample(x_start, t)`'s values bit for bit.  Decolorization (without Lab) is a per-pixel C x C mix M_t and is
        differentiable with respect to x_start (gradient M_t^T g, the same kernel with the transposed table).  Snow and the
        Lab decolor path are nonlinear and clipped: they raise when a gradient is requested."""
        if not isinstance(self.forward_process, DeColorization):
            refuse_grad("snow (nonlinear and clipped)", x_start)
            return self.q_sample(x_start, t)
        if self._lab_decolor():
            refuse_grad("the Lab decolor path (nonlinear and clipped)", x_start)
            return self.q_sample(x_start, t)
        x = x_start.contiguous().float()
        t = self._q_sample_index(t.to(x.device)).to(dtype=torch.int64).contiguous()
        mats = self._tab(x.device)[1]
        if self.__dict__.get('_mats_t', (None,))[0] is not mats:
            self._mats_t = (mats, mats.transpose(1, 2).contiguous())
        return ChanmixDegrade.apply(x, mats, self._mats_t[1], t)

    def _stage_random_snow(self, draws, dev):
        """captured training step: reset_parameters() redraws the snow layers on the host, which a graph cannot do.  The draws
        and the layer generation run before every replay (`draws.stage()`), into a buffer that lives with the graph; the
        captured cd_snow reads it through the tables set here."""
        fp = self.forward_process
        h = fp.image_size[0]
        nsb = fp._vertical.shape[1]
        layers = draws.buffer((self.num_timesteps, nsb, 3, h, h))
        br = draws.buffer(tuple(fp.br_t.shape), init=fp.br_t)

        def regenerate():
            fp.reset_parameters()
            fp.layers(dev, out=layers)
        draws.host_call(regenerate)
        self._tables = (dev, layers, br)
        fp._dev = dev

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
        draws = recording()
        if draws is None:
            self.forward_process.reset_parameters()
        elif isinstance(self.forward_process, Snow) and self.forward_process.random_snow:
            self._stage_random_snow(draws, x_start.device)
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
    _FINAL_ROUTINES = ('Final', 'Final_random_mean', 'Final_small_noise', 'Final_random_mean_and_actual')

    @torch.no_grad()
    def sample_one_step(self, img, t, init_pred=None, _t_lo=None):
        """SN:195-245 -> (x, direct_recons); t is a per-sample int64 tensor.  _t_lo (the strided loop of `sample(steps=...)`):
        the network time of the level to step down to, per sample, in place of t - 1; the update then indexes D with
        _t_lo - 1 where the one-step update indexes it with t - 2 (the reference's offsets)."""
        x = self.prediction_step_t(img, t, init_pred)
        direct_recons = x.clone()
        if self.train_routine in self._FINAL_ROUTINES:
            if self.sampling_routine == 'default':
                if _t_lo is not None:
                    x = self._degrade(x, _t_lo, -1)
                else:
                    x = self._degrade(x, t, -2)                                    # t_b - 1 steps per row
            elif self.sampling_routine == 'x0_step_down':
                src = x
                if self.recon_noise_std > 0.0 and isinstance(self.forward_process, DeColorization):
                    # (Snow ignores its x argument -- FP:361-372 -- so the reconstruction noise only matters for decolor)
                    src = x + torch.normal(0.0, self.recon_noise_std, size=x.size(), device=x.device)
                # x_times_sub_1 is re-cloned from ALL rows each iteration (SN:229-233): rows that finished before the
                # last iteration end with x_times_sub_1 == x_times, i.e. the update leaves them at `img`.
                t_lo = torch.where(t == torch.max(t), t - 1, t) if _t_lo is None else _t_lo
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
    def sample(self, batch_size=16, img=None, t=None, *, steps=None):
        """SN:259-295 -> {'xt', 'direct_recons', 'recon'}.  steps=K: K reverse steps through the levels of
        strided.reverse_levels instead of all t (None: every level, the reference's loop), with the one-step update's index
        offsets and per-sample snow layers.  The 'Step' / 'Step_Gradient' train routines (the network output is the next image
        or the step to it) and unknown sampling routines have no strided form: ValueError."""
        if self.train_routine not in self._FINAL_ROUTINES:
            refuse_strided(steps, 'snowification', "train_routine=%r" % self.train_routine)
        if self.sampling_routine not in ('default', 'x0_step_down'):
            refuse_strided(steps, 'snowification', "sampling_routine=%r" % self.sampling_routine)
        if t is None:
            t = self.num_timesteps
        levels = reverse_levels(t, steps)
        self.forward_process.reset_parameters(batch_size=batch_size)
        og_img = img
        tt = torch.full((img.shape[0],), t, dtype=torch.long, device=img.device)
        img = self._degrade(og_img, tt, -1)
        xt = img
        direct_recons = None
        for hi, lo in zip(levels, levels[1:]):
            step = torch.full((batch_size,), hi - 1, dtype=torch.long, device=img.device)
            t_lo = None if steps is None else torch.full((batch_size,), lo - 1, dtype=torch.long, device=img.device)
            x, cur = self.sample_one_step(img, step, _t_lo=t_lo)
            if direct_recons is None:
                direct_recons = cur
            img = x
        if self.to_lab:                                                             # SN:287-290
            xt, direct_recons, img = lab2rgb(xt), lab2rgb(direct_recons), lab2rgb(img)
        return {'xt': xt, 'direct_recons': direct_recons, 'recon': img}

    def restore(self, y, s, *, weight, steps=None):
        """guided restoration (guided.py) for decolorization without Lab, from the observation y = D_s(x) = M_{s-1} x per pixel,
        the mix `sample(img=x, t=s)` applies.  The updates index D one step lower, as `sample_one_step` does: 'default' x_lo =
        M_{lo-2} x0_hat - weight g, 'x0_step_down' x_lo = x_hi - M_{hi-2} x0_hat + M_{lo-2} x0_hat - weight g (index < 0:
        identity).  weight = 0 is `sample(img=x, t=s, steps=steps)['recon']` bit for bit.  Raises ValueError for snow and the
        Lab path (nonlinear and clipped) and for the routines `sample(steps=K)` refuses."""
        if not isinstance(self.forward_process, DeColorization):
            refuse_restore('snowification', "snow (nonlinear and clipped)")
        if self.to_lab:
            refuse_restore('snowification', "the Lab decolor path (nonlinear and clipped)")
        if self.train_routine not in self._FINAL_ROUTINES:
            refuse_restore('snowification', "train_routine=%r (no strided form)" % self.train_routine)
        if self.sampling_routine not in ('default', 'x0_step_down'):
            refuse_restore('snowification', "sampling_routine=%r (no strided form)" % self.sampling_routine)
        hw = tuple(self.image_size) if isinstance(self.image_size, tuple) else (self.image_size, self.image_size)
        check_arguments('snowification', y, s, weight, self.num_timesteps, (self.channels,) + hw)
        s, weight = int(s), float(weight)
        levels = reverse_levels(s, steps)
        y = y.contiguous()
        B, Cc, H, W = y.shape
        mats = self._tab(y.device)[1]
        level = lambda n: torch.full((B,), n, dtype=torch.long, device=y.device)
        t_obs = level(s)

        def guide_grad(x0):
            out = torch.empty_like(x0)
            call('cd_chanmix_guide_grad', ptr(x0), ptr(y), ptr(out), ptr(mats), ptr(t_obs), -1, B, Cc, C.c_int64(H * W), stream())
            return out

        def step(img, x0, g, hi, lo):
            out = torch.empty_like(img)
            x0 = x0.contiguous()
            t_hi, t_lo = level(hi - 1), level(lo - 1)
            if self.sampling_routine == 'default':
                call('cd_chanmix_guided', ptr(None), ptr(x0), ptr(g), C.c_float(weight), ptr(out), ptr(mats), ptr(t_lo),
                     ptr(None), -1, 0, B, Cc, C.c_int64(H * W), 0, stream())
                return out
            if self.recon_noise_std > 0.0:                     # as sample_one_step
                x0 = x0 + torch.normal(0.0, self.recon_noise_std, size=x0.size(), device=x0.device)
            call('cd_chanmix_guided', ptr(img.contiguous()), ptr(x0), ptr(g), C.c_float(weight), ptr(out), ptr(mats),
                 ptr(t_hi), ptr(t_lo), -1, -1, B, Cc, C.c_int64(H * W), 1, stream())
            return out

        return restore_loop(self.denoise_fn, y, levels, weight, guide_grad, step)

    def _total_forward(self, img):
        """forward_process.total_forward: decolor = every channel <- channel mean (FP:198-218, independent of the schedule),
        in Lab mode rgb2lab(mean(lab2rgb(img))); snow = D(img, T-1) (FP:358-359)"""
        if isinstance(self.forward_process, DeColorization):
            img = img.contiguous().float()
            B, Cc, H, W = img.shape
            mat = torch.full((1, Cc, Cc), 1.0 / Cc, device=img.device, dtype=torch.float32)
            zero = torch.zeros(B, dtype=torch.int64, device=img.device)
            out = torch.empty_like(img)
            if self.to_lab:                      # a one-step chain with the mean matrix
                call('cd_chanmix_lab', ptr(None), ptr(img), ptr(out), ptr(mat), ptr(zero), ptr(None), 0, 0, B, C.c_int64(H * W), 0,
                     stream())
            else:
                call('cd_chanmix', ptr(None), ptr(img), ptr(out), ptr(mat), ptr(zero), ptr(None), 0, 0, B, Cc, C.c_int64(H * W), 0,
                     stream())
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
            if self.to_lab:                      # SN:331-336 converts the CPU copies; same values, converted on the device
                X_0s.append(lab2rgb(direct_recons).cpu())
                X_ts.append(lab2rgb(img).cpu())
            else:
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
