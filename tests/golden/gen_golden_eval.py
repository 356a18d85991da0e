"""Goldens of the evaluation path from the UNMODIFIED reference (needs a checkout of the reference):
Frechet distances of `Fid/fid_score.py:calculate_frechet_distance` on seeded Gaussian statistics, including a rank-deficient
pair (fewer observations than dimensions, the situation its eps-retry exists for), and `calculate_activation_statistics` with a
stand-in feature network.  Usage: python tests/golden/gen_golden_eval.py   (deterministic)"""
import os, sys
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), 'oracle'))
import ref_shim  # noqa
sys.path.insert(0, os.path.join(ref_shim.REF_ROOT, 'deblurring-diffusion-pytorch'))
from Fid import fid_score  # noqa  (imports torchvision's inception definition; no weights are loaded)
import scipy.linalg as _sl

# The reference calls scipy.linalg.sqrtm(..., disp=False) and unpacks (sqrt, error estimate); the scipy in this image has
# dropped that keyword.  Compatibility stub (same role as the torchgeometry / comet_ml stubs in ref_shim.py): old calling
# convention on top of the same routine.
_sqrtm = _sl.sqrtm


def _sqrtm_compat(a, disp=True, **kw):
    r = _sqrtm(a, **kw)
    return r if disp else (r, 0.0)


fid_score.linalg.sqrtm = _sqrtm_compat


def main():
    rng = np.random.RandomState(2024)
    out = {}
    cases = {'d8': (8, 200, 200), 'd64': (64, 500, 300), 'd32_rankdef': (32, 20, 500), 'd16_same': (16, 100, 100)}
    for name, (d, n1, n2) in cases.items():
        A = rng.randn(d, d) / np.sqrt(d)
        a1 = rng.randn(n1, d) @ A + rng.randn(d) * 0.3
        a2 = a1.copy() if name.endswith('same') else rng.randn(n2, d) * (0.5 + rng.rand(d)) + rng.randn(d) * 0.1
        m1, s1, m2, s2 = a1.mean(0), np.cov(a1, rowvar=False), a2.mean(0), np.cov(a2, rowvar=False)
        out[name + ':a1'], out[name + ':a2'] = a1, a2
        out[name + ':fid'] = np.float64(fid_score.calculate_frechet_distance(m1, s1, m2, s2))
        print(name, out[name + ':fid'])

    # activation statistics through a stand-in feature network (4-d output, spatial size > 1 -> average pooled)
    torch.manual_seed(5)
    net = torch.nn.Conv2d(3, 12, 3, stride=2)

    class Wrapped(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.net = net

        def forward(self, x):
            return [self.net(x)]
    imgs = torch.rand(23, 3, 16, 16)
    mu, sigma = fid_score.calculate_activation_statistics(imgs[:20], Wrapped(), batch_size=5, dims=12, device='cpu')
    out['acts:w'], out['acts:b'] = net.weight.detach().numpy(), net.bias.detach().numpy()
    out['acts:imgs'], out['acts:mu'], out['acts:sigma'] = imgs.numpy(), mu, sigma
    # ---- FID feature network with a synthetic weight file (the real one is a download) ---------------------------------------
    import torchvision
    from Fid import inception as ref_inception
    from fid_weights import synthetic_state
    shapes = {k: v.shape for k, v in torchvision.models.inception_v3(weights=None, aux_logits=False, num_classes=1008,
                                                                       init_weights=False).state_dict().items()}
    state = synthetic_state(shapes)
    ref_inception.load_state_dict_from_url = lambda *a, **k: state
    net = ref_inception.InceptionV3([0, 1, 2, 3]).eval()
    torch.manual_seed(11)
    fid_imgs = torch.rand(2, 3, 48, 40)
    with torch.no_grad():
        feats = net(fid_imgs)
    out['fid:imgs'] = fid_imgs.numpy()
    for i, f in enumerate(feats):
        out[f'fid:block{i}'] = (f if i == 3 else f.mean((2, 3))).numpy()           # spatial means of the big maps
        print('block', i, tuple(f.shape), float(f.abs().mean()))
    out['fid:block2_edge'] = feats[2][:, :16, 0, :].numpy()                          # border row: where the pooling differs
    torch.manual_seed(12)
    small_in = torch.rand(1, 3, 80, 96)
    with torch.no_grad():
        out['fid:small_in'] = small_in.numpy()
        out['fid:small_block2'] = ref_inception.InceptionV3([2], resize_input=False, normalize_input=False).eval()(small_in)[0].numpy()
    np.savez_compressed(os.path.join(HERE, 'eval_small.npz'), **out)
    print('wrote eval_small.npz')

    # ---- public methods of every package's Trainer (names + parameter names): the evaluation surface ------------------------
    import inspect, json
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), 'oracle'))
    import ref_shim
    api = {}
    for tag, pkg_dir, module in (('deblurring', 'deblurring-diffusion-pytorch', 'deblurring_diffusion_pytorch'),
                                 ('resolution', 'resolution-diffusion-pytorch', 'resolution_diffusion_pytorch'),
                                 ('defading', 'defading-diffusion-pytorch', 'defading_diffusion_pytorch'),
                                 ('denoising', 'denoising-diffusion-pytorch', 'denoising_diffusion_pytorch'),
                                 ('demixing', 'demixing-diffusion-pytorch', 'demixing_diffusion_pytorch'),
                                 ('defading_generation', 'defading-generation-diffusion-pytorch', 'defading_diffusion_pytorch'),
                                 ('snowification', 'snowification', 'diffusion')):
        mod = ref_shim.import_reference(pkg_dir, module)
        api[tag] = {mn: [n for n in inspect.signature(fn).parameters if n != 'self']
                    for mn, fn in inspect.getmembers(mod.Trainer, predicate=inspect.isfunction) if not mn.startswith('_')}
    with open(os.path.join(HERE, 'trainer_api.json'), 'w') as f:
        json.dump(api, f, indent=0, sort_keys=True)
    print('wrote trainer_api.json', {k: len(v) for k, v in api.items()})


if __name__ == '__main__':
    main()
