"""`Unet` -- the ConvNeXt restoration operator R(x, t) of the reference
(deblurring-diffusion-pytorch/deblurring_diffusion_pytorch/deblurring_diffusion_pytorch.py:191-282, "DB"),
with the reference's constructor, `forward(x, time)` signature and state_dict keys, executed by the
sm_90a engine in engine.py (NHWC activations, tensor-core tap-list convolutions, fused HBM kernels).

The nn.Module tree below only *holds parameters* under the reference's names (so reference checkpoints,
including `module.`-prefixed DataParallel ones, load unchanged); no torch arithmetic runs on the hot path.
"""
import math
import torch
from torch import nn

from .engine import UnetEngine


def exists(x):
    return x is not None


class _Params(nn.Module):
    """parameter container; never called"""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter container: arithmetic runs in libcolddiff (engine.py)")


class LayerNorm(_Params):
    # DB:111-121
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.g = nn.Parameter(torch.ones(1, dim, 1, 1))
        self.b = nn.Parameter(torch.zeros(1, dim, 1, 1))


class ConvNextBlock(_Params):
    # DB:135-165 -- same submodule names/indices: mlp.1, ds_conv, net.0 (LayerNorm), net.1, net.3, res_conv
    def __init__(self, dim, dim_out, *, time_emb_dim=None, mult=2, norm=True):
        super().__init__()
        self.mlp = nn.Sequential(nn.GELU(), nn.Linear(time_emb_dim, dim)) if exists(time_emb_dim) else None
        self.ds_conv = nn.Conv2d(dim, dim, 7, padding=3, groups=dim)
        self.net = nn.Sequential(
            LayerNorm(dim) if norm else nn.Identity(),
            nn.Conv2d(dim, dim_out * mult, 3, padding=1),
            nn.GELU(),
            nn.Conv2d(dim_out * mult, dim_out, 3, padding=1))
        self.res_conv = nn.Conv2d(dim, dim_out, 1) if dim != dim_out else nn.Identity()


class LinearAttention(_Params):
    # DB:167-187
    def __init__(self, dim, heads=4, dim_head=32):
        super().__init__()
        self.scale = dim_head ** -0.5
        self.heads = heads
        hidden_dim = dim_head * heads
        self.to_qkv = nn.Conv2d(dim, hidden_dim * 3, 1, bias=False)
        self.to_out = nn.Conv2d(hidden_dim, dim, 1)


class PreNorm(_Params):
    def __init__(self, dim, fn):
        super().__init__()
        self.fn = fn
        self.norm = LayerNorm(dim)


class Residual(_Params):
    def __init__(self, fn):
        super().__init__()
        self.fn = fn


class SinusoidalPosEmb(_Params):
    def __init__(self, dim):
        super().__init__()
        self.dim = dim


def Upsample(dim):
    return nn.ConvTranspose2d(dim, dim, 4, 2, 1)


def Downsample(dim):
    return nn.Conv2d(dim, dim, 4, 2, 1)


class Unet(nn.Module):
    """Unet(dim, out_dim=None, dim_mults=(1,2,4,8), channels=3, with_time_emb=True, residual=False)  (DB:192-200)"""

    def __init__(self, dim, out_dim=None, dim_mults=(1, 2, 4, 8), channels=3, with_time_emb=True, residual=False):
        super().__init__()
        self.channels = channels
        self.residual = residual
        self.dim = dim
        print("Is Time embed used ? ", with_time_emb)       # the reference prints this (DB:203)

        dims = [channels, *map(lambda m: dim * m, dim_mults)]
        in_out = list(zip(dims[:-1], dims[1:]))
        if with_time_emb:
            time_dim = dim
            self.time_mlp = nn.Sequential(SinusoidalPosEmb(dim), nn.Linear(dim, dim * 4), nn.GELU(),
                                          nn.Linear(dim * 4, dim))
        else:
            time_dim = None
            self.time_mlp = None
        self.downs = nn.ModuleList([])
        self.ups = nn.ModuleList([])
        num_resolutions = len(in_out)
        for ind, (dim_in, dim_out) in enumerate(in_out):
            is_last = ind >= (num_resolutions - 1)
            self.downs.append(nn.ModuleList([
                ConvNextBlock(dim_in, dim_out, time_emb_dim=time_dim, norm=ind != 0),
                ConvNextBlock(dim_out, dim_out, time_emb_dim=time_dim),
                Residual(PreNorm(dim_out, LinearAttention(dim_out))),
                Downsample(dim_out) if not is_last else nn.Identity()]))
        mid_dim = dims[-1]
        self.mid_block1 = ConvNextBlock(mid_dim, mid_dim, time_emb_dim=time_dim)
        self.mid_attn = Residual(PreNorm(mid_dim, LinearAttention(mid_dim)))
        self.mid_block2 = ConvNextBlock(mid_dim, mid_dim, time_emb_dim=time_dim)
        for ind, (dim_in, dim_out) in enumerate(reversed(in_out[1:])):
            is_last = ind >= (num_resolutions - 1)
            self.ups.append(nn.ModuleList([
                ConvNextBlock(dim_out * 2, dim_in, time_emb_dim=time_dim),
                ConvNextBlock(dim_in, dim_in, time_emb_dim=time_dim),
                Residual(PreNorm(dim_in, LinearAttention(dim_in))),
                Upsample(dim_in) if not is_last else nn.Identity()]))
        out_dim = out_dim if exists(out_dim) else channels
        self.final_conv = nn.Sequential(ConvNextBlock(dim, dim), nn.Conv2d(dim, out_dim, 1))
        self._engine = None

    # -- engine plumbing -------------------------------------------------------------------------
    @property
    def engine(self):
        if self._engine is None:
            self._engine = UnetEngine(self)
        return self._engine

    def __deepcopy__(self, memo):
        # the engine (packed weights, workspaces) is per-instance device state: never cloned (Trainer's EMA copy)
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k == '_engine' else copy.deepcopy(v, memo)
        return new

    def _apply(self, fn, *a, **k):
        self._engine = None                     # parameters moved/cast: rebuild packed weights lazily
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, *a, **k):
        r = super().load_state_dict(state_dict, *a, **k)
        if self._engine is not None:
            self._engine.mark_weights_dirty()
        return r

    def forward(self, x, time=None):
        """x: (B, C, H, W) fp32 NCHW on a CUDA device, time: (B,) int64  ->  (B, out_dim, H, W)   (DB:256-282).
        `time` may be omitted only when the network was built with with_time_emb=False (snowification's UnetConvNextBlock
        declares `forward(x, time=None)`)."""
        if not x.is_cuda:
            raise RuntimeError("cold_diffusion_models_b200.Unet runs on a CUDA device (H100) only; got %s" % x.device)
        if time is None:
            if self.time_mlp is not None:
                raise TypeError("Unet.forward: `time` is required when the network has a time embedding")
            time = torch.zeros(x.shape[0], dtype=torch.int64, device=x.device)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            from .autograd import UnetFunction
            return UnetFunction.apply(self, x, time, *self.engine.param_list())
        if self.engine.use_cuda_graph:
            return self.engine.forward_graphed(x, time)
        return self.engine.forward(x, time)
