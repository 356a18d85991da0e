"""cold_diffusion_models_b200 -- H100-native engine for the Cold-Diffusion hot path.

Host code is Python/PyTorch (device memory, streams, torch.distributed); all arithmetic runs in
hand-written sm_90a CUDA behind the C ABI in include/colddiff.h (libcolddiff.so)."""
from . import _lib  # noqa: F401  (raises if the CUDA library has not been built)
from .unet import Unet
from .deblurring import GaussianDiffusion
from .trainer import Trainer
from .model2 import Model

__all__ = ['Unet', 'Model', 'GaussianDiffusion', 'Trainer']
