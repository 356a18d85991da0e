"""snowification/diffusion/utils.py (== decolor-diffusion/diffusion/utils.py:113-222) surface: the Lab conversions of the
`to_lab` path.  `rgb2lab(image)` takes RGB in [-1, 1] and `lab2rgb(image, clip=True)` returns 2 rgb - 1; both take CUDA
tensors of shape (*, 3, H, W) and run as one kernel (cd_lab_convert).  A CPU tensor raises: there is no host fallback."""
from ..snowification import rgb2lab, lab2rgb

__all__ = ['rgb2lab', 'lab2rgb']
