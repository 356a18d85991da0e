"""Drop-in `Trainer` for the *_diffusion_pytorch packages (reference: DB:1057-1236) on the H100 engine.

Same constructor keywords, attributes (`model`, `ema_model`, `opt`, `dl`, `ds`, `step`) and methods
(`train`, `save`, `load`, `step_ema`, `reset_parameters`) and the same checkpoint format
{'step','model','ema'} with reference state_dict keys.  What differs is execution:

  * one process per GPU (torchrun); gradients live in ONE flat fp32 buffer that is all-reduced with a single
    NCCL call per optimizer step (the reference's nn.DataParallel re-broadcasts all parameters and reduce-adds
    all gradients every micro-step, DB:1192 + celebA_128.py:102);
  * Adam (torch defaults, DB:1117) + the EMA update (DB:73-81,1134-1138) + gradient zeroing are one fused
    multi-tensor kernel (cd_adam_ema_step) over flat parameter / moment / EMA buffers;
  * parameters and EMA parameters are views of flat buffers, so `state_dict()` stays reference-shaped.
"""
import copy
import ctypes as C
from functools import partial  # noqa: F401
from pathlib import Path

import torch
from torch.utils import data

from ._lib import call, ptr, stream
from .evaluation import EvaluationMixin, SnowEvaluationMixin


def cycle(dl):
    while True:
        for d in dl:
            yield d


def _unwrap(m):
    return m.module if hasattr(m, 'module') else m


class SyntheticImages(data.Dataset):
    """x ~ U(-1,1) fp32 NCHW images of the configured shape (matches ToTensor()*2-1, DB:994-995)."""

    def __init__(self, image_size, channels=3, length=1 << 30, seed=1234):
        self.shape = (channels, image_size, image_size)
        self.length = length
        self.seed = seed

    def __len__(self):
        return self.length

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed + i)
        return torch.rand(self.shape, generator=g) * 2 - 1


class ImageFolderDataset(data.Dataset):
    """folder of images -> (C,H,W) fp32 in [-1,1] (reference Dataset / Dataset_Aug1, DB:983-1026)."""

    def __init__(self, folder, image_size, exts=('jpg', 'jpeg', 'png'), augment=False):
        from torchvision import transforms
        self.paths = [p for ext in exts for p in Path(f'{folder}').glob(f'**/*.{ext}')]
        ops_ = []
        if augment:
            ops_ += [transforms.Resize((int(image_size * 1.12), int(image_size * 1.12))), transforms.RandomCrop(image_size),
                     transforms.RandomHorizontalFlip()]
        else:
            ops_ += [transforms.Resize((int(image_size * 1.12), int(image_size * 1.12))), transforms.CenterCrop(image_size)]
        ops_ += [transforms.ToTensor(), transforms.Lambda(lambda t: (t * 2) - 1)]
        self.transform = transforms.Compose(ops_)

    def __len__(self):
        return len(self.paths)

    def __getitem__(self, index):
        from PIL import Image
        return self.transform(Image.open(self.paths[index]))


class DeviceImageDataset:
    """The reference's Dataset / Dataset_Aug1 (DB:983-1026: Resize to 1.12 x S, then CenterCrop or RandomCrop + RandomHorizontalFlip,
    ToTensor()*2-1) with the decoded, resized uint8 images resident in HBM: a 202k-image CelebA-128 set is 12.4 GB of the H100's 80 GB.
    Decoding and the one-time resize run once on the host (PIL, like the reference's transforms); every batch is one gather
    kernel (cd_augment_u8) with per-sample crop windows and flips drawn on the host -- no DataLoader workers, no H2D copy of
    fp32 images.  Opt-in (`Trainer(..., dataset='device')` / `'device_aug'`)."""

    def __init__(self, folder, image_size, augment=False, exts=('jpg', 'jpeg', 'png'), device='cuda', seed=0):
        import numpy as np
        from PIL import Image
        from torchvision import transforms
        self.image_size, self.augment = image_size, augment
        self.paths = sorted(p for ext in exts for p in Path(f'{folder}').glob(f'**/*.{ext}'))
        rs = int(image_size * 1.12)
        resize = transforms.Resize((rs, rs))
        imgs = [np.asarray(resize(Image.open(p).convert('RGB')), dtype=np.uint8) for p in self.paths]
        self.src = torch.from_numpy(np.stack(imgs)).contiguous().to(device)          # [N][rs][rs][3] uint8
        self.N, self.rs = len(imgs), rs
        self.gen = torch.Generator().manual_seed(seed)
        self._perm, self._pos = torch.randperm(self.N, generator=self.gen), 0

    def __len__(self):
        return self.N

    def _indices(self, B, shuffle):
        """the next B image indices of an endless pass over the set (reshuffled every epoch, like cycle(DataLoader(shuffle)))"""
        out, need = [], B
        while need > 0:
            if self._pos >= self.N:
                self._perm, self._pos = (torch.randperm(self.N, generator=self.gen) if shuffle else torch.arange(self.N)), 0
            take = min(need, self.N - self._pos)
            out.append(self._perm[self._pos:self._pos + take])
            self._pos += take
            need -= take
        return torch.cat(out)

    def batch(self, B, shuffle=True, index=None, oy=None, ox=None, flip=None):
        """-> (B, 3, S, S) fp32 in [-1, 1] on the dataset's device"""
        S, m = self.image_size, self.rs - self.image_size
        index = self._indices(B, shuffle) if index is None else index
        if oy is None:
            if self.augment:                      # torchvision RandomCrop.get_params: i ~ U{0..h-th}, j ~ U{0..w-tw}; flip with p = 0.5
                oy = torch.randint(0, m + 1, (B,), generator=self.gen); ox = torch.randint(0, m + 1, (B,), generator=self.gen)
                flip = (torch.rand(B, generator=self.gen) < 0.5)
            else:                                 # torchvision CenterCrop: int(round((h - th) / 2.))
                c = int(round(m / 2.0))
                oy = torch.full((B,), c); ox = torch.full((B,), c); flip = torch.zeros(B, dtype=torch.bool)
        dev = self.src.device
        index = index.to(dev, torch.int64).contiguous()
        oy, ox, flip = (v.to(dev, torch.int32).contiguous() for v in (oy, ox, flip))
        out = torch.empty(B, 3, S, S, device=dev, dtype=torch.float32)
        call('cd_augment_u8', ptr(self.src), self.N, self.rs, self.rs, ptr(index), ptr(oy), ptr(ox), ptr(flip), B, S, ptr(out), stream())
        return out


class FusedAdamEMA:
    """torch.optim.Adam(lr, betas=(0.9,0.999), eps=1e-8, weight_decay=0) + EMA as one kernel over flat buffers."""

    def __init__(self, engine, ema_engine=None, lr=2e-5, betas=(0.9, 0.999), eps=1e-8):
        self.engine, self.ema_engine = engine, ema_engine
        engine.flatten_params()
        if ema_engine is not None:
            ema_engine.flatten_params()
        self.param_groups = [dict(lr=lr, betas=betas, eps=eps)]
        self.m = torch.zeros_like(engine.flat_param)
        self.v = torch.zeros_like(engine.flat_param)
        self.t = 0

    def zero_grad(self, set_to_none=False):
        self.engine.flat_grad.zero_()

    def step(self, ema_mode=0, ema_beta=0.0, grad_scale=1.0):
        g = self.param_groups[0]
        self.t += 1
        e = self.engine
        ema = self.ema_engine.flat_param if (self.ema_engine is not None and ema_mode) else None
        call('cd_adam_ema_step', ptr(e.flat_param), ptr(e.flat_grad), ptr(self.m), ptr(self.v), ptr(ema),
             C.c_int64(e.flat_param.numel()), C.c_float(g['lr']), C.c_float(g['betas'][0]), C.c_float(g['betas'][1]),
             C.c_float(g['eps']), self.t, int(ema_mode) if ema is not None else 0, C.c_float(ema_beta),
             C.c_float(grad_scale), stream())
        e.mark_weights_dirty()
        if ema is not None:
            self.ema_engine.mark_weights_dirty()

    def state_dict(self):
        return dict(t=self.t, m=self.m, v=self.v, param_groups=self.param_groups)

    def load_state_dict(self, sd):
        self.t = sd['t']; self.m.copy_(sd['m']); self.v.copy_(sd['v'])


_MERGE_MICRO_BATCHES = None


def merge_micro_batches(enable=None):
    """switch: run the gradient_accumulate_every micro-batches of one optimizer step as ONE pass over their concatenation.
    The loss is a mean over equally sized micro-batches (DB:1190-1196: `backwards(loss / accumulate)`), so the gradient is the
    same sum of per-sample terms; what changes is the order of the floating-point additions, the number of launches per step
    (weight repacks, per-launch fixed costs and the per-(batch element, head) kernels run once instead of twice) and the
    wave count of the small-resolution layers.  Needs a network without batch-coupled layers (every Unet / Model here) and
    single-tensor batches of one shape; off by default (COLDDIFF_MERGE_MICRO_BATCHES=1, or tuning.autotune() when it
    reproduces the accumulated gradient and is faster)."""
    global _MERGE_MICRO_BATCHES
    if enable is not None:
        _MERGE_MICRO_BATCHES = bool(enable)
    if _MERGE_MICRO_BATCHES is None:
        import os
        _MERGE_MICRO_BATCHES = os.environ.get('COLDDIFF_MERGE_MICRO_BATCHES', '0') == '1'
    return _MERGE_MICRO_BATCHES


class Trainer(EvaluationMixin, object):
    def __init__(self, diffusion_model, folder, *, ema_decay=0.995, image_size=128, train_batch_size=32, train_lr=2e-5,
                 train_num_steps=100000, gradient_accumulate_every=2, fp16=False, step_start_ema=2000,
                 update_ema_every=10, save_and_sample_every=1000, results_folder='./results', load_path=None,
                 dataset=None, shuffle=True):
        super().__init__()
        if fp16:
            raise NotImplementedError("fp16/apex path of the reference is dead code (fp16=False in every driver)")
        self.model = diffusion_model
        self.ema_decay = ema_decay
        self.ema_model = copy.deepcopy(self.model)
        self.update_ema_every = update_ema_every
        self.step_start_ema = step_start_ema
        self.save_and_sample_every = save_and_sample_every
        self.batch_size = train_batch_size
        self.image_size = image_size
        self.gradient_accumulate_every = gradient_accumulate_every
        self.train_num_steps = train_num_steps

        dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()
        self._world = torch.distributed.get_world_size() if dist_on else 1
        self._rank = torch.distributed.get_rank() if dist_on else 0
        core = _unwrap(self.model)
        self.ds, self.dl = self._make_loader(folder, dataset, shuffle, seed=1234)
        # the restoration network is `denoise_fn` in every package except defading (`defade_fn`, DFG:303)
        net_of = lambda m_: m_.denoise_fn if hasattr(m_, 'denoise_fn') else m_.defade_fn
        self._unet = net_of(core)
        self._ema_unet = net_of(_unwrap(self.ema_model))
        self.opt = FusedAdamEMA(self._unet.engine, self._ema_unet.engine, lr=train_lr)
        self.step = 0
        self.results_folder = Path(results_folder)
        self.results_folder.mkdir(exist_ok=True)
        self.fp16 = fp16
        self.reset_parameters()
        if load_path is not None:
            self.load(load_path)
        self._sync_replicas()

    _aug_datasets = ('mnist', 'cifar10', 'flower', 'celebA', 'AFHQ')     # `dataset` values that select Dataset_Aug1

    def _sync_replicas(self):
        """one process per GPU: every replica starts from rank 0's parameters and EMA weights (the reference's nn.DataParallel
        re-broadcasts them every micro-step, celebA_128.py:102); Adam + EMA then stay bit-identical on all ranks because they
        consume the same all-reduced gradient."""
        if self._world <= 1:
            return
        for eng in (self._unet.engine, self._ema_unet.engine):
            torch.distributed.broadcast(eng.flat_param, src=0)
            eng.mark_weights_dirty()

    def _make_loader(self, folder, dataset, shuffle, seed):
        channels = getattr(_unwrap(self.model), 'channels', 3)
        world, rank = self._world, self._rank
        if folder is None or dataset == 'synthetic':
            # every rank reads its own stream of images (DataParallel scatters one batch; here the global batch is world x B)
            ds = SyntheticImages(self.image_size, channels, seed=seed + 1000003 * rank)
            return ds, cycle(data.DataLoader(ds, batch_size=self.batch_size, shuffle=False, pin_memory=True, num_workers=0,
                                             drop_last=True))
        if dataset in ('device', 'device_aug'):            # images resident in HBM, batches gathered by cd_augment_u8
            ds = DeviceImageDataset(folder, self.image_size, augment=(dataset == 'device_aug'), seed=rank)

            def gen():
                while True:
                    yield ds.batch(self.batch_size, shuffle=shuffle)
            return ds, gen()
        aug = dataset in self._aug_datasets
        print(dataset, "DA used" if aug else "")
        ds = ImageFolderDataset(folder, self.image_size, augment=aug)
        if world > 1:                                      # disjoint shards of every epoch, one per rank
            sampler = data.distributed.DistributedSampler(ds, num_replicas=world, rank=rank, shuffle=shuffle, seed=seed)
            return ds, cycle(data.DataLoader(ds, batch_size=self.batch_size, sampler=sampler, pin_memory=True,
                                             num_workers=8 if aug else 16, drop_last=True))
        return ds, cycle(data.DataLoader(ds, batch_size=self.batch_size, shuffle=shuffle, pin_memory=True,
                                         num_workers=8 if aug else 16, drop_last=True))

    # ---- reference API ------------------------------------------------------------------------------
    def reset_parameters(self):
        self.ema_model.load_state_dict(self.model.state_dict())

    def step_ema(self):
        """stand-alone EMA update (the training loop fuses this into the optimizer kernel)."""
        if self.step < self.step_start_ema:
            self.reset_parameters()
            return
        e, m = self._ema_unet.engine, self._unet.engine
        call('cd_ema_update', ptr(e.flat_param), ptr(m.flat_param), C.c_int64(e.flat_param.numel()),
             C.c_float(self.ema_decay), 2, stream())
        e.mark_weights_dirty()

    def save(self, itrs=None):
        if getattr(self, '_rank', 0) != 0:                 # replicas are identical: rank 0 writes the checkpoint
            return
        d = {'step': self.step, 'model': self.model.state_dict(), 'ema': self.ema_model.state_dict()}
        name = 'model.pt' if itrs is None else f'model_{itrs}.pt'
        torch.save(d, str(self.results_folder / name))

    def load(self, load_path):
        print("Loading : ", load_path)
        d = torch.load(load_path, map_location='cpu')
        self.step = d['step']
        self.model.load_state_dict(_match_prefix(d['model'], self.model))
        self.ema_model.load_state_dict(_match_prefix(d['ema'], self.ema_model))
        if getattr(self, '_world', 1) > 1 and hasattr(self, 'opt'):
            self._sync_replicas()

    # ---- hot loop --------------------------------------------------------------------------------------
    def _next(self):
        return next(self.dl)

    def _loss(self, d):
        return torch.mean(self.model(d))                       # DB:1192

    def _sample_start(self):
        """the image the periodic `sample` starts from (DB:1209)"""
        return next(self.dl).cuda()

    def _periodic_sample(self, og_img):
        """-> (xt, direct_recons, recon) of the EMA model every `save_and_sample_every` steps (DB:1210)"""
        return _unwrap(self.ema_model).sample(batch_size=self.batch_size, img=og_img)

    def train_step(self, batches=None):
        """one optimizer step = gradient_accumulate_every micro-batches (DB:1188-1204). Returns mean loss (tensor)."""
        u_loss = None
        A = self.gradient_accumulate_every
        ds = [batches[i] if batches is not None else self._next() for i in range(A)]
        if (A > 1 and merge_micro_batches() and all(torch.is_tensor(d) for d in ds) and len({tuple(d.shape) for d in ds}) == 1):
            # one pass over the concatenated micro-batches: mean over A * B samples == sum_i mean_i / A
            d = torch.cat([d.cuda(non_blocking=True) for d in ds], dim=0)
            loss = self._loss(d)
            loss.backward()
            u_loss = loss.detach() * A
            ds = []
        eng = self._unet.engine
        works, low = [], [None]
        overlap = self._world > 1 and hasattr(eng, '_grads_ready_from')
        for i, d in enumerate(ds):
            d = tuple(x.cuda(non_blocking=True) for x in d) if isinstance(d, (tuple, list)) else d.cuda(non_blocking=True)
            loss = self._loss(d)
            u_loss = loss.detach() if u_loss is None else u_loss + loss.detach()
            if overlap and i == len(ds) - 1:
                # last micro-batch: every finished suffix of the flat gradient is all-reduced while the backward continues
                # (NCCL runs on its own stream behind the kernels enqueued so far)
                def ready(lo, hi):
                    works.append(torch.distributed.all_reduce(eng.flat_grad[lo:hi], async_op=True))
                    low[0] = lo
                    self.overlapped_ranges.append((lo, hi))
                self.overlapped_ranges = []                  # introspection / tests: the ranges reduced during the backward
                eng._ready_mark = eng._grad_total
                eng.grad_ready_hook = ready
            try:
                (loss / A).backward()
            finally:
                eng.grad_ready_hook = None
        from .engine_bwd import allreduce_mean_
        if works:
            scale = allreduce_mean_(eng.flat_grad[:low[0]], self._world)   # what the backward closed last: conditioning MLPs, finest levels
            for w in works:
                w.wait()
        else:
            scale = allreduce_mean_(eng.flat_grad, self._world)            # one NCCL all-reduce per optimizer step
        ema_mode = 0
        if self.step % self.update_ema_every == 0:
            ema_mode = 1 if self.step < self.step_start_ema else 2
        self.opt.step(ema_mode=ema_mode, ema_beta=self.ema_decay, grad_scale=scale)
        self.opt.zero_grad()
        return u_loss / self.gradient_accumulate_every

    def train(self):
        acc_loss = 0
        while self.step < self.train_num_steps:
            loss = self.train_step()
            if self.step % 100 == 0 and self._rank == 0:
                print(f'{self.step}: {loss.item()}')
            acc_loss = acc_loss + loss
            if self.step != 0 and self.step % self.save_and_sample_every == 0:
                from torchvision import utils
                milestone = self.step // self.save_and_sample_every
                og_img = self._sample_start()
                xt, direct_recons, all_images = self._periodic_sample(og_img)
                for name, img in (('og', og_img), ('recon', all_images), ('direct_recons', direct_recons), ('xt', xt)):
                    if self._rank == 0:
                        utils.save_image((img + 1) * 0.5, str(self.results_folder / f'sample-{name}-{milestone}.png'), nrow=6)
                acc_loss = acc_loss / (self.save_and_sample_every + 1)
                if self._rank == 0:
                    print(f'Mean of last {self.step}: {float(acc_loss)}')
                acc_loss = 0
                self.save()
                if self.step % (self.save_and_sample_every * 100) == 0:
                    self.save(self.step)
            self.step += 1
        print('training completed')


class DenoisingTrainer(Trainer):
    """Trainer of denoising_diffusion_pytorch: forward(x1, x2) with x2 = randn_like(x1) (DN:738-741); the noise is
    drawn on the device instead of on the host."""

    def _loss(self, d):
        return torch.mean(self.model(d, torch.randn_like(d)))

    def _sample_start(self):
        return torch.randn(self.batch_size, getattr(_unwrap(self.model), 'channels', 3), self.image_size, self.image_size,
                           device='cuda')                       # DN:757-762

    _to_show = (2, 4, 16, 64, 128, 256, 384, 448, 480)          # DN:862
    _cover_batches = 5                                          # DN:864


class ResolutionTrainer(Trainer):
    """Trainer of resolution_diffusion_pytorch (RS:842-1200): evaluation in batches of 200 (RS:1017) and its own
    mixture-over-low-resolution-images generation routine."""

    def fid_distance_decrease_from_manifold(self, fid_func, start=0, end=1000, bs=200, sanity_check=1):
        return super().fid_distance_decrease_from_manifold(fid_func, start=start, end=end, bs=bs, sanity_check=sanity_check)

    def sample_as_a_mean_blur_torch_gmm_ablation(self, torch_gmm=None, siz=2, ch=3, clusters=10, sample_at=6, noise=0,
                                                 num_samples=6400, bs=64):
        """mixture over the step-`sample_at` low-resolution images (area-averaged to siz x siz); draws are blown up with
        nearest-exact interpolation and restored by `gen_sample` (RS:1117-1183)"""
        import torch.nn.functional as F
        H, W = self._image_size_hw()
        ema = _unwrap(self.ema_model)
        feats = self._dataset_features(lambda b: F.interpolate(ema.opt(b, t=sample_at), size=siz, mode='area').flatten(1))
        model = self._fit_mixture(torch_gmm, feats, clusters)
        og_x = model.sample(num_datapoints=num_samples).cuda().reshape(num_samples, 3, siz, siz)
        og_x = F.interpolate(og_x, size=(H, W), mode='nearest-exact').float()
        self._generate_to_folders(og_x, ch, bs, noise)
        return model


class DefadingTrainer(Trainer):
    """Trainer of defading_diffusion_pytorch (DFG:654-811): its own defaults and `sample(batch_size, faded_recon_sample)`"""

    def __init__(self, diffusion_model, folder, *, ema_decay=0.995, image_size=128, train_batch_size=32, train_lr=2e-5,
                 train_num_steps=700000, gradient_accumulate_every=2, fp16=False, step_start_ema=2000, update_ema_every=10,
                 save_and_sample_every=10000, results_folder='./results', load_path=None, dataset=None):
        super().__init__(diffusion_model, folder, ema_decay=ema_decay, image_size=image_size, train_batch_size=train_batch_size,
                         train_lr=train_lr, train_num_steps=train_num_steps, gradient_accumulate_every=gradient_accumulate_every,
                         fp16=fp16, step_start_ema=step_start_ema, update_ema_every=update_ema_every,
                         save_and_sample_every=save_and_sample_every, results_folder=results_folder, load_path=load_path,
                         dataset=dataset)

    def _periodic_sample(self, og_img):
        return _unwrap(self.ema_model).sample(batch_size=self.batch_size, faded_recon_sample=og_img)      # DFG:789


class DemixingTrainer(Trainer):
    """Trainer of demixing_diffusion_pytorch: two image folders, forward(x1, x2) on one batch of each (DM:600-772)."""
    _aug_datasets = ('train',)

    def __init__(self, diffusion_model, folder1, folder2, *, ema_decay=0.995, image_size=128, train_batch_size=32, train_lr=2e-5,
                 train_num_steps=100000, gradient_accumulate_every=2, fp16=False, step_start_ema=2000, update_ema_every=10,
                 save_and_sample_every=1000, results_folder='./results', load_path=None, dataset=None, shuffle=True):
        super().__init__(diffusion_model, folder1, ema_decay=ema_decay, image_size=image_size, train_batch_size=train_batch_size,
                         train_lr=train_lr, train_num_steps=train_num_steps, gradient_accumulate_every=gradient_accumulate_every,
                         fp16=fp16, step_start_ema=step_start_ema, update_ema_every=update_ema_every,
                         save_and_sample_every=save_and_sample_every, results_folder=results_folder, load_path=load_path,
                         dataset=dataset, shuffle=shuffle)
        self.ds1, self.dl1 = self.ds, self.dl
        self.ds2, self.dl2 = self._make_loader(folder2, dataset, shuffle, seed=4321)

    def _next(self):
        return next(self.dl1), next(self.dl2)

    def _loss(self, d):
        return torch.mean(self.model(d[0], d[1]))               # DM:726-728

    def _sample_start(self):
        return next(self.dl2).cuda()                            # DM:747

    _to_show = (2, 4, 16, 64, 128, 256, 384, 448, 480)          # DM:844
    _cover_batches = 5                                          # DM:846

    def _eval_batch(self):
        return next(self.dl2).cuda()                            # DM:776: evaluation starts from the second domain

    def _forward_backward(self, noise_level):
        og1, og2 = next(self.dl1).cuda(), next(self.dl2).cuda()                                            # DM:848-852
        F_, B_, final = _unwrap(self.ema_model).forward_and_backward(batch_size=self.batch_size, img1=og1, img2=og2)
        return og1, F_, B_, final


class DefadingGenerationTrainer(Trainer):
    """Trainer of the defading-generation package: the end image x2 is a constant random colour in [-0.5, 0.5)
    per sample (DFGEN:768-776), drawn on the device instead of on the host."""
    _aug_datasets = ('train',)

    def _colour(self, like_batch):
        c = torch.rand((like_batch, 3), device='cuda') - 0.5
        return c[:, :, None, None].expand(like_batch, 3, self.image_size, self.image_size).contiguous()

    def _loss(self, d):
        return torch.mean(self.model(d, self._colour(d.shape[0])))

    def _sample_start(self):
        return self._colour(self.batch_size)                    # DFGEN:796-803

    _to_show = (8, 192, 256, 320, 384, 512, 640, 704, 748)      # DFGEN:913
    _cover_batches = 5                                          # DFGEN:915

    def _eval_batch(self):
        c = self._colour(self.batch_size)
        return c + 0.000001 * torch.randn_like(c)               # DFGEN:833-839

    def _forward_backward(self, noise_level):
        og1 = next(self.dl).cuda()                                                                          # DFGEN:917-928
        F_, B_, final = _unwrap(self.ema_model).forward_and_backward(batch_size=self.batch_size, img1=og1,
                                                                     img2=self._colour(self.batch_size))
        return og1, F_, B_, final


def snow_get_transform(image_size, random_aug=False, resize=False):
    """torchvision transform of snowification/diffusion/get_dataset.py:5-34 (and Dataset.get_transform, SN:502-528)"""
    from torchvision import transforms
    to_pm1 = [transforms.ToTensor(), transforms.Lambda(lambda t: (t * 2) - 1)]
    if image_size[0] == 64:
        return transforms.Compose([transforms.CenterCrop((128, 128)), transforms.Resize(image_size)] + to_pm1)
    if not random_aug:
        return transforms.Compose(([transforms.Resize(image_size)] if resize else []) + [transforms.CenterCrop(image_size)] + to_pm1)
    jitter = transforms.ColorJitter(0.8, 0.8, 0.8, 0.2)
    return transforms.Compose([transforms.RandomResizedCrop(size=image_size), transforms.RandomHorizontalFlip(),
                               transforms.RandomApply([jitter], p=0.8)] + to_pm1)


def get_dataset(name, folder, image_size, random_aug=False):
    """torchvision datasets by name (snowification/diffusion/get_dataset.py:44-57); `download=True` of the reference needs a
    network, the files must already be under `folder` here"""
    from torchvision import datasets
    tf = lambda **k: snow_get_transform(image_size, random_aug=random_aug, **k)
    if name in ('cifar10_train', 'cifar10_test'):
        return datasets.CIFAR10(folder, train=name.endswith('train'), transform=tf())
    if name in ('CelebA_train', 'CelebA_test'):
        return datasets.CelebA(folder, split=name.split('_')[1], transform=tf())
    if name in ('flower_train', 'flower_test'):
        return datasets.Flowers102(folder, split=name.split('_')[1], transform=tf(resize=True))
    return None


class SnowificationTrainer(SnowEvaluationMixin, Trainer):
    """Trainer of snowification/diffusion (== decolor-diffusion/diffusion), SN:563-760: the image size comes from the model,
    torchvision datasets by name, `sample()` returns a dict whose entries are all saved, `save(save_with_time_stamp)`."""

    def __init__(self, diffusion_model, folder, *, ema_decay=0.995, image_size=128, train_batch_size=32, train_lr=2e-5,
                 train_num_steps=100000, gradient_accumulate_every=2, fp16=False, step_start_ema=2000, update_ema_every=10,
                 save_and_sample_every=5000, save_with_time_stamp_every=50000, results_folder='./results', load_path=None,
                 random_aug=False, torchvision_dataset=False, dataset=None, to_lab=False, order_seed=-1):
        if to_lab:
            raise NotImplementedError("to_lab (kornia Lab colour path) is out of scope of the H100 engine")
        core = _unwrap(diffusion_model)
        size = core.image_size
        self._size2 = tuple(size) if isinstance(size, (tuple, list)) else (size, size)
        self.random_aug, self.torchvision_dataset, self.to_lab, self.order_seed = random_aug, torchvision_dataset, to_lab, int(order_seed)
        self.save_with_time_stamp_every = save_with_time_stamp_every
        self.num_timesteps = core.num_timesteps
        self.data_loader = None
        super().__init__(diffusion_model, folder, ema_decay=ema_decay, image_size=self._size2[0], train_batch_size=train_batch_size,
                         train_lr=train_lr, train_num_steps=train_num_steps, gradient_accumulate_every=gradient_accumulate_every,
                         fp16=fp16, step_start_ema=step_start_ema, update_ema_every=update_ema_every,
                         save_and_sample_every=save_and_sample_every, results_folder=results_folder, load_path=load_path,
                         dataset=dataset, shuffle=True)
        self.results_folder.mkdir(parents=True, exist_ok=True)
        self.post_process_func = lambda x: x

    def _make_loader(self, folder, dataset, shuffle, seed):
        if folder is None or dataset == 'synthetic':
            return super()._make_loader(folder, dataset, shuffle, seed)
        if self.torchvision_dataset:
            ds = get_dataset(dataset, folder, self._size2, random_aug=self.random_aug)
        else:
            ds = ImageFolderDataset(folder, self._size2[0])
            ds.transform = snow_get_transform(self._size2, random_aug=self.random_aug) if self._size2[0] != 256 else ds.transform
        loader = data.DataLoader(ds, batch_size=self.batch_size, shuffle=True, pin_memory=True, num_workers=4)
        self.data_loader = loader                               # SN:619: the un-cycled loader `test_from_data` walks

        def gen():
            while True:
                for d in loader:                          # torchvision datasets yield (image, label)
                    yield d[0] if isinstance(d, (list, tuple)) else d
        return ds, gen()

    def _process_item(self, x):
        return x[0] if isinstance(x, (list, tuple)) else x

    def save(self, save_with_time_stamp=False):
        d = {'step': self.step, 'model': self.model.state_dict(), 'ema': self.ema_model.state_dict()}
        name = f'model_{self.step}.pt' if save_with_time_stamp else 'model.pt'
        torch.save(d, str(self.results_folder / name))

    def train(self):
        import time
        start_time = time.time()
        while self.step < self.train_num_steps:
            loss = self.train_step()
            print(f'{self.step}: {loss.item()}')
            if self.step != 0 and self.step % 100 == 0:
                print(f'time for 100 steps: {time.time() - start_time}')
                start_time = time.time()
            if self.step != 0 and self.step % self.save_and_sample_every == 0:
                from torchvision import utils
                milestone = self.step // self.save_and_sample_every
                og_img = self._sample_start()
                sample_dict = _unwrap(self.ema_model).sample(batch_size=self.batch_size, img=og_img)
                sample_dict['og'] = og_img
                print(f'images saved: {sample_dict.keys()}')
                for k, img in sample_dict.items():
                    utils.save_image((img + 1) * 0.5, str(self.results_folder / f'sample-{k}-{milestone}.png'), nrow=6)
                self.save()
            if self.step != 0 and self.step % self.save_with_time_stamp_every == 0:
                self.save(save_with_time_stamp=True)
            self.step += 1


def _match_prefix(sd, model):
    """accept checkpoints saved with or without the DataParallel `module.` prefix (DB:1039-1055)."""
    want = any(k.startswith('module.') for k in model.state_dict().keys())
    have = any(k.startswith('module.') for k in sd.keys())
    if want == have:
        return sd
    if have:
        return {k[len('module.'):]: v for k, v in sd.items()}
    return {'module.' + k: v for k, v in sd.items()}
