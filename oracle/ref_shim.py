"""Import shim for the UNMODIFIED upstream reference (test infrastructure only).

The reference packages import third-party modules that are absent from this
image (comet_ml, torchgeometry, ...).  This module injects minimal stubs so the
reference classes can be imported FROM a checkout of it ($COLD_REF_ROOT, never copied) and run on
CPU to (a) generate golden vectors for tests/golden and (b) pin oracle/*.py.

torchgeometry restatement (torchgeometry 0.1.2 image/gaussian.py, un-pinned by the
reference; "parity unpinned" at this boundary, see oracle/deblur_oracle.py): gaussian(k, s)[x] =
exp(-(x - k//2)^2 / (2 s^2)) normalised to sum 1; 2-D kernel = outer product.
"""
import sys, types, os, math
import torch

REF_ROOT = os.environ.get("COLD_REF_ROOT", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "..", "reference"))


def _gaussian(window_size, sigma):
    def gauss_fcn(x):
        return -(x - window_size // 2) ** 2 / float(2 * sigma ** 2)
    gauss = torch.stack([torch.exp(torch.tensor(gauss_fcn(x))) for x in range(window_size)])
    return gauss / gauss.sum()


def get_gaussian_kernel(ksize, sigma):
    if not isinstance(ksize, int) or ksize % 2 == 0 or ksize <= 0:
        raise TypeError("ksize must be an odd positive integer. Got {}".format(ksize))
    return _gaussian(ksize, sigma)


def get_gaussian_kernel2d(ksize, sigma):
    if not isinstance(ksize, tuple) or len(ksize) != 2:
        raise TypeError("ksize must be a tuple of length two. Got {}".format(ksize))
    if not isinstance(sigma, tuple) or len(sigma) != 2:
        raise TypeError("sigma must be a tuple of length two. Got {}".format(sigma))
    ksize_x, ksize_y = ksize
    sigma_x, sigma_y = sigma
    kernel_x = get_gaussian_kernel(ksize_x, sigma_x)
    kernel_y = get_gaussian_kernel(ksize_y, sigma_y)
    return torch.matmul(kernel_x.unsqueeze(-1), kernel_y.unsqueeze(-1).t())


def install_stubs():
    if "comet_ml" not in sys.modules:
        m = types.ModuleType("comet_ml")
        class Experiment:  # noqa
            def __init__(self, *a, **k): pass
            def __getattr__(self, n): return lambda *a, **k: None
        m.Experiment = Experiment
        sys.modules["comet_ml"] = m
    if "torchgeometry" not in sys.modules:
        tgm = types.ModuleType("torchgeometry")
        img = types.ModuleType("torchgeometry.image")
        img.get_gaussian_kernel2d = get_gaussian_kernel2d
        img.get_gaussian_kernel = get_gaussian_kernel
        tgm.image = img
        sys.modules["torchgeometry"] = tgm
        sys.modules["torchgeometry.image"] = img
    for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.image", "kornia", "kornia.color", "kornia.color.gray", "kornia.color.rgb", "kornia.color.xyz", "imageio", "pytorch_msssim", "sklearn", "sklearn.mixture", "lpips",
                 "cv2"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                m = types.ModuleType(name)
                m.__path__ = []                      # lets `import pkg.sub` resolve to the stubbed sub-modules
                sys.modules[name] = m
                if name == 'kornia.color' or name == 'kornia':
                    pass
                if name == 'pytorch_msssim':
                    m.ssim = lambda *a, **k: None          # evaluation-only import of the reference (never called here)
                if '.' in name:
                    setattr(sys.modules[name.split('.')[0]], name.split('.')[1], m)


def _rgb_to_grayscale(image):
    # kornia.color.gray.rgb_to_grayscale (un-pinned upstream): 0.299 R + 0.587 G + 0.114 B, keepdim channel
    r, g, b = image[..., 0:1, :, :], image[..., 1:2, :, :], image[..., 2:3, :, :]
    return 0.299 * r + 0.587 * g + 0.114 * b


def import_reference(pkg_dir, module):
    """pkg_dir e.g. 'deblurring-diffusion-pytorch'; module e.g. 'deblurring_diffusion_pytorch'."""
    install_stubs()
    if 'kornia.color.gray' in sys.modules and not hasattr(sys.modules['kornia.color.gray'], 'rgb_to_grayscale'):
        sys.modules['kornia.color.gray'].rgb_to_grayscale = _rgb_to_grayscale
        for modname, fns in (('kornia.color', ('rgb_to_lab', 'lab_to_rgb')), ('kornia.color.rgb', ('linear_rgb_to_rgb', 'rgb_to_linear_rgb')),
                             ('kornia.color.xyz', ('rgb_to_xyz', 'xyz_to_rgb'))):
            for fn in fns:
                setattr(sys.modules[modname], fn, lambda *a, **k: None)   # Lab colour path (--to_lab) is never exercised
    p = os.path.join(REF_ROOT, pkg_dir)
    if not os.path.isdir(p):
        raise RuntimeError("reference not present at %s (set $COLD_REF_ROOT to a checkout of the reference)" % p)
    # each reference directory defines same-named modules; purge before switching
    for k in list(sys.modules):
        if k.split(".")[0] == module:
            del sys.modules[k]
    sys.path.insert(0, p)
    try:
        mod = __import__(module)
    finally:
        sys.path.remove(p)
    return mod


def patch_cuda_noop():
    """Reference sampling loops hard-code .cuda() (DB:421); make it a no-op on CPU."""
    torch.Tensor.cuda = lambda self, *a, **k: self
