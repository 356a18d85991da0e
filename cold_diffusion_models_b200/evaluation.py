"""Evaluation path of the reference: the metrics and figure / sample dumps its `*_test.py` drivers call
on a trained model.  Everything here is host-side orchestration over the sampling methods of the diffusion classes (which
run on the CUDA engine); the metrics themselves are small and, like in the reference, computed on the gathered CPU tensors.

Reference pieces this file stands in for:
  * `Trainer.test_from_data / paper_* / sample_as_a_*_gmm* / fid_distance_decrease_from_manifold / save_training_data`
    (deblurring_diffusion_pytorch.py:1160-1181, 1238-1722) -> `EvaluationMixin`
  * `Fid/fid_score.py:149-356` (activation statistics + Frechet distance) -> `get_activations`,
    `calculate_activation_statistics`, `calculate_frechet_distance`, `calculate_fid_given_samples`
  * `pytorch_msssim.ssim` (third party, not part of the reference; restated from its published
    definition: 11-tap sigma-1.5 Gaussian window, 'valid' filtering, K = (0.01, 0.03)) -> `ssim`
  * `pycave.bayes.GaussianMixture` (third party, absent) -> `GaussianMixture` with the constructor / fit / sample surface the
    reference drivers use (celebA_128_test.py:129-138).  Only distributional agreement is possible there (EM from a random
    initialisation), so that class has statistical tests, not goldens.

Differences from the reference, on purpose: `sample_as_a_mean_blur_torch_gmm_ablation` does not stop in `pdb.set_trace()`
(DB:1414-1415); GIFs are written with PIL because `imageio` is not a dependency; the loops that the reference hard-codes to
50 batches / 6400 samples take the count as a keyword with the reference's value as default; the metric routine also
returns what it prints.
"""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F
from torch.utils import data


def _core(m):
    return m.module if hasattr(m, 'module') else m


def create_folder(path):
    os.makedirs(path, exist_ok=True)


# ------------------------------------------------------------------------------------------------------------------------
# metrics
# ------------------------------------------------------------------------------------------------------------------------
def rmse(a, b):
    """root mean squared error over every element (DB:1678)"""
    return torch.sqrt(torch.mean((a - b) ** 2))


def _gauss_window(size, sigma, dtype, device):
    c = torch.arange(size, dtype=dtype, device=device) - size // 2
    g = torch.exp(-(c * c) / (2.0 * sigma * sigma))
    return g / g.sum()


def _window_filter(x, g):
    """separable 'valid' Gaussian filtering of (N, C, H, W); an axis shorter than the window is left unfiltered"""
    C = x.shape[1]
    k = g.numel()
    if x.shape[2] >= k:
        x = F.conv2d(x, g.view(1, 1, k, 1).expand(C, 1, k, 1), groups=C)
    if x.shape[3] >= k:
        x = F.conv2d(x, g.view(1, 1, 1, k).expand(C, 1, 1, k), groups=C)
    return x


def ssim(X, Y, data_range=255, size_average=True, win_size=11, win_sigma=1.5, K=(0.01, 0.03), nonnegative_ssim=False,
         chunk=256):
    """structural similarity of two image batches (N, C, H, W), the quantity the reference reports (DB:1679, 1691, 1703).

    Per channel: local means / variances / covariance under a Gaussian window (no padding), the SSIM map averaged over
    the valid region; then the mean over channels and, with `size_average`, over the batch.  Processed `chunk` images at a
    time so that a whole test set can be scored without a second copy of it."""
    if X.shape != Y.shape:
        raise ValueError(f"Input images should have the same dimensions, but got {tuple(X.shape)} and {tuple(Y.shape)}.")
    if X.dim() != 4:
        raise ValueError(f"Input images should be 4-d tensors (N, C, H, W), but got {tuple(X.shape)}")
    if win_size % 2 != 1:
        raise ValueError("Window size should be odd.")
    C1, C2 = (K[0] * data_range) ** 2, (K[1] * data_range) ** 2
    out = []
    for i in range(0, X.shape[0], chunk):
        x, y = X[i:i + chunk].float(), Y[i:i + chunk].float()
        g = _gauss_window(win_size, win_sigma, x.dtype, x.device)
        mx, my = _window_filter(x, g), _window_filter(y, g)
        vx = _window_filter(x * x, g) - mx * mx
        vy = _window_filter(y * y, g) - my * my
        cxy = _window_filter(x * y, g) - mx * my
        m = ((2 * mx * my + C1) / (mx * mx + my * my + C1)) * ((2 * cxy + C2) / (vx + vy + C2))
        per_channel = m.flatten(2).mean(-1)
        if nonnegative_ssim:
            per_channel = torch.relu(per_channel)
        out.append(per_channel)
    per_channel = torch.cat(out)
    return per_channel.mean() if size_average else per_channel.mean(1)


def get_activations(samples, model, batch_size=50, dims=2048, device='cpu', num_workers=1):
    """(n, dims) float64 features of `samples` (a tensor of images in [0, 1]) under `model` (Fid/fid_score.py:149-196).
    As there, a trailing partial batch is not evaluated and its rows stay uninitialised in the reference; here they are
    dropped from the result instead (documented divergence: garbage rows -> no rows)."""
    if hasattr(model, 'eval'):
        model.eval()
    n = (samples.shape[0] // batch_size) * batch_size
    acts = np.empty((n, dims))
    for s in range(0, n, batch_size):
        with torch.no_grad():
            p = model(samples[s:s + batch_size].to(device))
        p = p[0] if isinstance(p, (list, tuple)) else p
        if p.dim() == 4:
            if p.shape[2] != 1 or p.shape[3] != 1:
                p = F.adaptive_avg_pool2d(p, (1, 1))
            p = p.flatten(1)
        acts[s:s + batch_size] = p.double().cpu().numpy()
    return acts


def calculate_activation_statistics(samples, model, batch_size=50, dims=2048, device='cpu', num_workers=1):
    """mean and covariance (rows = observations) of the features (Fid/fid_score.py:254-277)"""
    a = get_activations(samples, model, batch_size, dims, device, num_workers)
    return np.mean(a, axis=0), np.cov(a, rowvar=False)


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """d^2 = |mu1 - mu2|^2 + Tr(S1 + S2 - 2 (S1 S2)^(1/2))   (Fid/fid_score.py:198-252).

    The reference takes a general matrix square root of the product (scipy `sqrtm`, with an eps-regularised retry and an
    imaginary-part check).  Here the trace term comes from a symmetric problem instead: with R = S1^(1/2) (eigen-
    decomposition of the symmetric PSD S1), S1 S2 is similar to R S2 R, which is symmetric PSD, so
    Tr (S1 S2)^(1/2) = sum_i sqrt(lambda_i(R S2 R)) -- real by construction, no retry needed for singular covariances."""
    mu1, mu2 = np.atleast_1d(np.asarray(mu1, np.float64)), np.atleast_1d(np.asarray(mu2, np.float64))
    s1, s2 = np.atleast_2d(np.asarray(sigma1, np.float64)), np.atleast_2d(np.asarray(sigma2, np.float64))
    assert mu1.shape == mu2.shape, 'Training and test mean vectors have different lengths'
    assert s1.shape == s2.shape, 'Training and test covariances have different dimensions'
    w, V = np.linalg.eigh((s1 + s1.T) * 0.5)
    R = (V * np.sqrt(np.clip(w, 0.0, None))) @ V.T
    M = R @ s2 @ R
    lam = np.linalg.eigvalsh((M + M.T) * 0.5)
    tr_covmean = np.sqrt(np.clip(lam, 0.0, None)).sum()
    d = mu1 - mu2
    return float(d.dot(d) + np.trace(s1) + np.trace(s2) - 2.0 * tr_covmean)


def calculate_fid_given_samples(samples, batch_size=50, device='cuda:0', dims=2048, num_workers=1, model=None):
    """FID between `samples[0]` and `samples[1]` (tensors of images in [0, 1]); Fid/fid_score.py:343-356.

    `model` maps an image batch to (N, dims[, 1, 1]) features.  The reference builds pytorch-fid's InceptionV3 from weights
    it downloads (Fid/inception.py:184-208); there is no network in the deployment this engine targets, so either the
    feature network is handed in (any callable) or $COLDDIFF_FID_WEIGHTS names a local copy of that weight file, from which
    `InceptionV3` below is built."""
    if model is None:
        if os.environ.get('COLDDIFF_FID_WEIGHTS') is None:
            raise RuntimeError("calculate_fid_given_samples needs model=<feature extractor> or $COLDDIFF_FID_WEIGHTS pointing at "
                               "pytorch-fid's InceptionV3 weight file: the reference downloads it (Fid/inception.py), this "
                               "engine does not")
        model = InceptionV3([InceptionV3.BLOCK_INDEX_BY_DIM[dims]]).to(device)
    m1, s1 = calculate_activation_statistics(samples[0], model, batch_size, dims, device, num_workers)
    m2, s2 = calculate_activation_statistics(samples[1], model, batch_size, dims, device, num_workers)
    return calculate_frechet_distance(m1, s1, m2, s2)


# ------------------------------------------------------------------------------------------------------------------------
# Gaussian mixture with the surface of pycave.bayes.GaussianMixture that the reference's drivers use
# ------------------------------------------------------------------------------------------------------------------------
class GaussianMixture:
    """EM for a Gaussian mixture on a (n, d) tensor; float64 on the data's device.

    Constructor arguments follow the calls at DB:1410-1411 / DB:1540-1541: `num_components`, `covariance_type`
    ('full' | 'diag' | 'spherical'), `convergence_tolerance` (stop when the mean negative log-likelihood changes by less),
    `covariance_regularization` (added to the diagonal), `batch_size` / `trainer_params` accepted and ignored (the whole
    data set is resident; one EM step is a handful of batched GEMMs)."""

    def __init__(self, num_components=1, *, covariance_type='diag', init_strategy='kmeans', convergence_tolerance=1e-3,
                 covariance_regularization=1e-6, batch_size=None, trainer_params=None, max_epochs=100, seed=None):
        if covariance_type not in ('full', 'diag', 'spherical'):
            raise ValueError(f"unknown covariance_type {covariance_type!r}")
        self.num_components = int(num_components)
        self.covariance_type = covariance_type
        self.init_strategy = init_strategy
        self.convergence_tolerance = float(convergence_tolerance)
        self.covariance_regularization = float(covariance_regularization)
        self.max_epochs = int(max_epochs)
        self.batch_size, self.trainer_params = batch_size, trainer_params
        self._gen = None if seed is None else int(seed)
        self.weights_ = self.means_ = self.covariances_ = None
        self.converged_, self.num_iter_, self.nll_ = False, 0, float('nan')

    # ---- helpers -----------------------------------------------------------------------------------------
    def _generator(self, device):
        g = torch.Generator(device=device)
        g.manual_seed(self._gen if self._gen is not None else int(torch.randint(0, 2 ** 31 - 1, (1,)).item()))
        return g

    def _init_means(self, X, g):
        n, k = X.shape[0], self.num_components
        first = torch.randint(0, n, (1,), generator=g, device=X.device)
        means = [X[first[0]]]
        d2 = ((X - means[0]) ** 2).sum(1)
        for _ in range(1, k):                                              # k-means++ seeding
            p = d2 / d2.sum() if float(d2.sum()) > 0 else torch.full_like(d2, 1.0 / n)
            j = torch.multinomial(p, 1, generator=g)
            means.append(X[j[0]])
            d2 = torch.minimum(d2, ((X - means[-1]) ** 2).sum(1))
        mu = torch.stack(means)
        if self.init_strategy == 'kmeans':
            for _ in range(10):                                            # a few Lloyd iterations
                a = torch.cdist(X, mu).argmin(1)
                for c in range(k):
                    sel = a == c
                    if sel.any():
                        mu[c] = X[sel].mean(0)
        return mu

    def _full_cov(self):
        """(k, d, d) covariance matrices whatever the parametrisation"""
        if self.covariance_type == 'full':
            return self.covariances_
        d = self.means_.shape[1]
        if self.covariance_type == 'diag':
            return torch.diag_embed(self.covariances_)
        return self.covariances_[:, None, None] * torch.eye(d, dtype=self.means_.dtype, device=self.means_.device)

    def _log_prob(self, X):
        """(n, k) log( pi_c N(x | mu_c, S_c) )"""
        d = X.shape[1]
        L = torch.linalg.cholesky(self._full_cov())
        diff = (X[None] - self.means_[:, None]).transpose(1, 2)            # (k, d, n)
        z = torch.linalg.solve_triangular(L, diff, upper=False)
        maha = (z * z).sum(1).T                                            # (n, k)
        logdet = 2.0 * torch.log(torch.diagonal(L, dim1=1, dim2=2)).sum(1)
        return torch.log(self.weights_)[None] - 0.5 * (maha + logdet[None] + d * math.log(2 * math.pi))

    def _m_step(self, X, r):
        n, d = X.shape
        nk = r.sum(0) + 1e-300
        self.weights_ = nk / n
        self.means_ = (r.T @ X) / nk[:, None]
        reg = self.covariance_regularization
        if self.covariance_type == 'full':
            diff = X[None] - self.means_[:, None]                          # (k, n, d)
            cov = torch.einsum('kn,kni,knj->kij', r.T, diff, diff) / nk[:, None, None]
            self.covariances_ = cov + reg * torch.eye(d, dtype=X.dtype, device=X.device)
        else:
            var = (r.T @ (X * X)) / nk[:, None] - self.means_ ** 2
            var = var.clamp_min(0.0)
            self.covariances_ = (var + reg) if self.covariance_type == 'diag' else (var.mean(1) + reg)

    # ---- public surface ----------------------------------------------------------------------------------
    def fit(self, X):
        X = torch.as_tensor(X).detach().double()
        if X.dim() != 2 or X.shape[0] < self.num_components:
            raise ValueError("fit expects (n, d) data with n >= num_components")
        g = self._generator(X.device)
        mu = self._init_means(X, g)
        a = torch.cdist(X, mu).argmin(1)
        self._m_step(X, F.one_hot(a, self.num_components).double())
        prev = float('inf')
        self.converged_ = False
        for it in range(self.max_epochs):
            lp = self._log_prob(X)
            norm = torch.logsumexp(lp, 1, keepdim=True)
            nll = float(-norm.mean())
            self.num_iter_, self.nll_ = it + 1, nll
            if abs(prev - nll) < self.convergence_tolerance:
                self.converged_ = True
                break
            prev = nll
            self._m_step(X, torch.exp(lp - norm))
        return self

    def score(self, X):
        """mean negative log-likelihood of the rows of X"""
        X = torch.as_tensor(X).detach().double().to(self.means_.device)
        return float(-torch.logsumexp(self._log_prob(X), 1).mean())

    def predict_proba(self, X):
        X = torch.as_tensor(X).detach().double().to(self.means_.device)
        lp = self._log_prob(X)
        return torch.exp(lp - torch.logsumexp(lp, 1, keepdim=True)).float()

    def predict(self, X):
        return self.predict_proba(X).argmax(1)

    def sample(self, num_datapoints):
        """(num_datapoints, d) float32 draws from the fitted mixture"""
        if self.means_ is None:
            raise RuntimeError("sample() before fit()")
        g = self._generator(self.means_.device)
        comp = torch.multinomial(self.weights_, int(num_datapoints), replacement=True, generator=g)
        L = torch.linalg.cholesky(self._full_cov())
        z = torch.randn(int(num_datapoints), self.means_.shape[1], dtype=self.means_.dtype, device=self.means_.device,
                        generator=g)
        return (self.means_[comp] + torch.einsum('nij,nj->ni', L[comp], z)).float()

    def get_params(self):
        return dict(num_components=self.num_components, covariance_type=self.covariance_type,
                    init_strategy=self.init_strategy, convergence_tolerance=self.convergence_tolerance,
                    covariance_regularization=self.covariance_regularization, batch_size=self.batch_size,
                    trainer_params=self.trainer_params)

    def __repr__(self):
        return f"GaussianMixture(num_components={self.num_components}, covariance_type={self.covariance_type!r})"


# ------------------------------------------------------------------------------------------------------------------------
# the Trainer's evaluation methods
# ------------------------------------------------------------------------------------------------------------------------
def _save(img, path, nrow=6):
    from torchvision import utils
    utils.save_image(img, str(path), nrow=nrow)


def _unit(x):
    return (x + 1) * 0.5


def _accepted(fn, **kw):
    """the subset of `kw` that `fn` takes (the packages' sampling methods differ in optional keywords)"""
    import inspect
    names = inspect.signature(fn).parameters
    return {k: v for k, v in kw.items() if k in names}


def _write_gif(path, frame_paths):
    from PIL import Image
    frames = [Image.open(p).convert('RGB') for p in frame_paths]
    if frames:
        frames[0].save(str(path), save_all=True, append_images=frames[1:], duration=100, loop=0)


class EvaluationMixin:
    """mixed into `Trainer`; uses `self.ds / self.dl / self.batch_size / self.results_folder / self.ema_model` only"""

    _to_show = (2, 4, 8, 16, 32, 64, 128, 192, 256)          # DB:1273: trajectory indices shown in the cover-page strips
    _cover_batches = 50                                       # DB:1275 (5 in the two-image packages: DN:864, DM:846)
    _cover_noise = 0.002                                      # DB:1350

    def _ema(self):
        return _core(self.ema_model)

    # hooks the per-package trainers override ---------------------------------------------------------------------
    def _eval_batch(self):
        """the batch an evaluation routine starts from (DB:1240: the next training batch)"""
        b = next(self.dl)
        return (b[0] if isinstance(b, (tuple, list)) else b).cuda()

    def _all_sample(self, og_img, times=None):
        """-> (X_0s, X_ts) of the reverse process from `og_img`.  The packages disagree on this call: defading names the
        image `faded_recon_sample` (DFG:817), denoising returns (X1_0s, X2_0s, X_ts) (DN:515 -- its own trainer unpacks two
        names from it and raises), snowification returns four lists (SN:848); the first and the last-but-optional lists
        are the x0-estimates and the x_t in all of them."""
        fn = self._ema().all_sample
        import inspect
        key = 'img' if 'img' in inspect.signature(fn).parameters else 'faded_recon_sample'
        r = fn(batch_size=og_img.shape[0], **{key: og_img}, **_accepted(fn, times=times))
        if len(r) == 3:
            return r[0], r[2]
        return r[0], r[1]

    def _manifold_order(self, n):
        """order in which `fid_distance_decrease_from_manifold` walks the data set (DB:1576: as stored)"""
        return range(n)

    def _score_view(self, t):
        """what the metrics see of a batch of images (identity; the snow package shrinks large images)"""
        return t

    def _forward_backward(self, noise_level):
        """-> (image shown first, Forward, Backward, final) of one batch (DB:1347-1350)"""
        og_img = self._eval_batch()
        Forward, Backward, final_all = self._ema().forward_and_backward(batch_size=self.batch_size, img=og_img,
                                                                        **_accepted(self._ema().forward_and_backward,
                                                                                    noise_level=noise_level))
        return og_img, Forward, Backward, final_all

    # ---- DB:1160-1181 -----------------------------------------------------------------------------------------
    def add_title(self, path, title):
        """re-writes the image at `path` with a 10 px black frame and a 20 px title bar carrying `title`"""
        import cv2
        img = cv2.imread(str(path))
        framed = cv2.copyMakeBorder(img, 10, 10, 10, 10, cv2.BORDER_CONSTANT, value=[0, 0, 0])
        bar_h = 20
        bar = np.zeros((bar_h, framed.shape[1], 3), np.uint8)
        bar[:] = (255, 0, 180)
        out = cv2.vconcat((bar, framed))
        cv2.putText(out, str(title), (bar.shape[1] // 2, bar_h - 2), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (0, 0, 0), 1, 0)
        cv2.imwrite(str(path), out)

    # ---- DB:1238-1266 -----------------------------------------------------------------------------------------
    def _dump_trajectory(self, X_0s, X_ts, extra_path):
        """every x0-estimate / x_t as a titled 6-column grid `sample-<i>-<extra_path>-{x0,xt}.png` + the two GIFs"""
        frames_0, frames_t = [], []
        for i in range(len(X_0s)):
            p0 = self.results_folder / f'sample-{i}-{extra_path}-x0.png'
            _save(_unit(X_0s[i]), p0)
            self.add_title(p0, str(i))
            frames_0.append(p0)
            if i < len(X_ts):
                pt = self.results_folder / f'sample-{i}-{extra_path}-xt.png'
                _save(_unit(X_ts[i]), pt)
                self.add_title(pt, str(i))
                frames_t.append(pt)
        _write_gif(self.results_folder / f'Gif-{extra_path}-x0.gif', frames_0)
        _write_gif(self.results_folder / f'Gif-{extra_path}-xt.gif', frames_t)

    def test_from_data(self, extra_path, s_times=None):
        """one batch through `all_sample`; originals, titled trajectory grids and GIFs (DB:1238-1266)"""
        og_img = self._eval_batch()
        X_0s, X_ts = self._all_sample(og_img, s_times)
        _save(_unit(og_img), self.results_folder / f'og-{extra_path}.png')
        self._dump_trajectory(X_0s, X_ts, extra_path)
        return X_0s, X_ts

    def test_with_mixup(self, extra_path):
        """the reverse process started from the average of two batches (DFG:843-883)"""
        a, b = self._eval_batch(), self._eval_batch()
        og_img = (a + b) / 2
        X_0s, X_ts = self._all_sample(og_img)
        for name, t in (('og1', a), ('og2', b), ('og', og_img)):
            _save(_unit(t), self.results_folder / f'{name}-{extra_path}.png')
        self._dump_trajectory(X_0s, X_ts, extra_path)

    def test_from_random(self, extra_path):
        """the reverse process started from a batch scaled by 0.9, i.e. slightly off the data manifold (DFG:885-920)"""
        og_img = self._eval_batch() * 0.9
        X_0s, X_ts = self._all_sample(og_img)
        _save(_unit(og_img), self.results_folder / f'og-{extra_path}.png')
        self._dump_trajectory(X_0s, X_ts, extra_path)

    def controlled_direct_reconstruct(self, extra_path):
        """seeded `sample` of one batch, the four grids of the periodic sampler, then a checkpoint (DFG:922-941)"""
        torch.manual_seed(0)
        og_img = self._eval_batch()
        xt, direct_recons, all_images = self._periodic_sample(og_img)
        for name, t in (('og', og_img), ('recon', all_images), ('direct_recons', direct_recons), ('xt', xt)):
            _save(_unit(t), self.results_folder / f'sample-{name}-{extra_path}.png')
        self.save()

    def test_from_data_save_results(self, bs=32, batch_size=100):
        """original / degraded / sampled / direct reconstruction of every image of the data set, one file each, into
        `<results>_orig`, `_blur`, `_deblur`, `_d_deblur` (DFG:1146-1251; whole batches of `batch_size` only, as there)"""
        all_samples = self._dataset_features(lambda b: b.cpu(), batch_size=batch_size)
        folders = {k: f'{self.results_folder}_{k}/' for k in ('orig', 'blur', 'd_deblur', 'deblur')}
        for f in folders.values():
            create_folder(f)
        to3 = lambda t: _unit(t.float().cpu().repeat(1, 3 // t.shape[1], 1, 1))
        n = 0
        for cnt in range(0, all_samples.shape[0], bs):
            og_img = all_samples[cnt:cnt + bs].cuda().float()
            X_0s, X_ts = self._all_sample(og_img, None)
            for key, t in (('orig', og_img), ('blur', X_ts[0]), ('deblur', X_0s[-1]), ('d_deblur', X_0s[0])):
                t = to3(t)
                for i in range(t.shape[0]):
                    _save(t[i], f'{folders[key]}{n + i}.png', nrow=1)
            n += og_img.shape[0]
        return n

    def sample_from_data_save(self, start=0, end=1000, bs=1000):
        """the sampled reconstruction of data-set images start+1 .. end, one file each (DN:1362-1395)"""
        imgs = []
        for idx in range(len(self.ds)):
            if idx > start:
                item = self.ds[idx]
                imgs.append(item[0] if isinstance(item, (tuple, list)) else item)
            if end is not None and idx == end:
                break
        all_samples = torch.stack(imgs)
        create_folder(f'{self.results_folder}/')
        cnt = 0
        while cnt < all_samples.shape[0]:
            og_img = all_samples[cnt:cnt + bs].cuda().float()
            X_0s, X_ts = self._all_sample(og_img, None)
            for i in range(X_0s[-1].shape[0]):
                _save(_unit(X_0s[-1][i]), f'{self.results_folder}/sample-x0-{cnt}.png')
                cnt += 1
        return cnt

    # ---- DB:1712-1722 -----------------------------------------------------------------------------------------
    def save_training_data(self, limit=None):
        create_folder(f'{self.results_folder}/')
        n = len(self.ds) if limit is None else min(limit, len(self.ds))
        for idx in range(n):
            _save(_unit(self.ds[idx]), f'{self.results_folder}/{idx}.png')
            if idx % 1000 == 0:
                print(idx)

    # ---- DB:1269-1388 -----------------------------------------------------------------------------------------
    def _strip(self, k, og, Forward, backwards, finals, cnt, suffixes):
        """one row image per backward trajectory: original | selected forward states | selected backward states | final"""
        import cv2
        rf = self.results_folder

        def as_cv(t, name):
            _save(t, rf / name, nrow=1)
            return cv2.imread(f'{rf}/{name}')
        start = as_cv(og[k], f'og_img_{cnt}.png')
        fwd = [as_cv(_unit(Forward[j][k]), 'temp.png') for j in range(len(Forward)) if j in self._to_show]
        for Backward, final, suf in zip(backwards, finals, suffixes):
            row = [start] + fwd
            row += [as_cv(_unit(Backward[j][k]), 'temp.png') for j in range(len(Backward))
                    if (len(Backward) - j) in self._to_show]
            row.append(as_cv(final[k], f'final{suf}_{cnt}.png'))
            cv2.imwrite(f'{rf}/all{suf}_{cnt}.png', cv2.hconcat(row))

    def paper_showing_diffusion_images_cover_page(self, n_batches=None, noise_level=None):
        cnt = 0
        for _ in range(self._cover_batches if n_batches is None else n_batches):
            og_img, Forward, Backward, final_all = self._forward_backward(self._cover_noise if noise_level is None
                                                                          else noise_level)
            og, final_all = _unit(og_img), _unit(final_all)
            for k in range(Forward[0].shape[0]):
                self._strip(k, og, Forward, [Backward], [final_all], cnt, [''])
                cnt += 1

    def paper_showing_diffusion_images_cover_page_both_sampling(self, n_batches=50, noise_level=0.000):
        cnt = 0
        for _ in range(n_batches):
            og_img = self._eval_batch()
            Forward, B1, B2, f1, f2 = self._ema().forward_and_backward_2(batch_size=self.batch_size, img=og_img,
                                                                         noise_level=noise_level)
            og = _unit(og_img)
            for k in range(Forward[0].shape[0]):
                self._strip(k, og, Forward, [B1, B2], [_unit(f1), _unit(f2)], cnt, ['_1', '_2'])
                cnt += 1

    def paper_showing_diffusion_images(self, s_times=None, n_batches=50, to_show=(0, 2, 4, 8, 16, 32, 64, 80, 88, 92, 96, 98, 99)):
        """selected x_t of the reverse trajectory followed by the final estimate, one strip per image (DN:957-995); every
        x_t is also left behind as x_<steps to go>_<n>.png"""
        import cv2
        rf, cnt = self.results_folder, 0
        for _ in range(n_batches):
            og_img = self._eval_batch()
            X_0s, X_ts = self._all_sample(og_img, s_times)
            for k in range(X_ts[0].shape[0]):
                row = []
                for j in range(len(X_ts)):
                    name = f'x_{len(X_ts) - j}_{cnt}.png'
                    _save(_unit(X_ts[j][k]), rf / name, nrow=1)
                    if j in to_show:
                        row.append(cv2.imread(f'{rf}/{name}'))
                _save(_unit(X_0s[-1][k]), rf / f'x_best_{cnt}.png', nrow=1)
                row.append(cv2.imread(f'{rf}/x_best_{cnt}.png'))
                cv2.imwrite(f'{rf}/all_{cnt}.png', cv2.hconcat(row))
                cnt += 1

    def paper_invert_section_images(self, s_times=None, n_batches=50):
        """degraded | direct reconstruction | sampled reconstruction | original, one strip per image (DN:910-955)"""
        import cv2
        rf, cnt = self.results_folder, 0
        for _ in range(n_batches):
            og_img = self._eval_batch()
            X_0s, X_ts = self._all_sample(og_img, s_times)
            og = _unit(og_img)
            for j in range(og.shape[0] // 3):
                tiles = []
                for name, t in (('blurry_image', _unit(X_ts[0][j:j + 1])), ('direct_recons', _unit(X_0s[0][j:j + 1])),
                                ('sampling_recons', _unit(X_0s[-1][j:j + 1])), ('original', og[j:j + 1])):
                    _save(t, rf / f'{name}_{cnt}.png', nrow=3)
                    tiles.append(cv2.copyMakeBorder(cv2.imread(f'{rf}/{name}_{cnt}.png'), 10, 10, 10, 10,
                                                    cv2.BORDER_CONSTANT, value=[0, 0, 0]))
                cv2.imwrite(f'{rf}/all_{cnt}.png', cv2.hconcat(tiles))
                cnt += 1

    # ---- generation from a mixture fitted to degraded images: DB:1391-1564 ---------------------------------------
    def _dataset_features(self, fn, batch_size=100):
        """fn(batch on the GPU) -> (b, d) features, concatenated over the data set in order (drop_last like the reference)"""
        dl = data.DataLoader(self.ds, batch_size=batch_size, shuffle=False, pin_memory=True, num_workers=0, drop_last=True)
        return torch.cat([fn((b[0] if isinstance(b, (tuple, list)) else b).cuda()) for b in dl], dim=0)

    def _fit_mixture(self, torch_gmm, feats, clusters, batch_size=100, **extra):
        torch_gmm = GaussianMixture if torch_gmm is None else torch_gmm
        model = torch_gmm(num_components=clusters, trainer_params=dict(gpus=1), covariance_type='full',
                          convergence_tolerance=0.001, batch_size=batch_size, **extra)
        model.fit(feats)
        return model

    def _image_size_hw(self):
        s = self.image_size
        return (s, s) if isinstance(s, int) else tuple(s)

    def sample_as_a_mean_blur_torch_gmm_ablation(self, torch_gmm=None, ch=3, clusters=10, noise=0, num_samples=6400, bs=64):
        """fit the mixture to per-image channel means (what a fully blurred image is), draw means, run `gen_sample` from the
        constant images and write x_t / direct reconstruction / sample one file per image (for FID folders)"""
        feats = self._dataset_features(lambda b: torch.mean(b, [2, 3]))
        model = self._fit_mixture(torch_gmm, feats, clusters)
        og_x = model.sample(num_datapoints=num_samples).cuda()[:, :, None, None]
        self._generate_to_folders(og_x, ch, bs, noise)
        return model

    def _generate_to_folders(self, og_x, ch, bs, noise):
        """`gen_sample` from the start images `og_x` (broadcast to ch x H x W), bs at a time; x_t / direct reconstruction /
        sample of every image into `<results>_xt`, `<results>_dir_recons`, `<results>_out` (DB:1425-1456)"""
        H, W = self._image_size_hw()
        folders = {k: f'{self.results_folder}_{k}' for k in ('xt', 'out', 'dir_recons')}
        for f in folders.values():
            create_folder(f)
        cnt = 0
        for j in range(og_x.shape[0] // bs):
            og_img = og_x[j * bs:(j + 1) * bs].expand(bs, ch, H, W).float().contiguous()
            xt, direct_recons, all_images = self._ema().gen_sample(batch_size=bs, img=og_img, noise_level=noise)
            for i in range(all_images.shape[0]):
                _save(_unit(all_images[i]), f"{folders['out']}/sample-x0-{cnt}.png")
                _save(_unit(xt[i]), f"{folders['xt']}/sample-x0-{cnt}.png")
                _save(_unit(direct_recons[i]), f"{folders['dir_recons']}/sample-x0-{cnt}.png")
                cnt += 1

    def sample_as_a_mean_blur_torch_gmm(self, torch_gmm=None, start=0, end=1000, ch=3, clusters=10, num_samples=48,
                                        noise_levels=(0.001, 0.002, 0.003, 0.004), repeats=3):
        feats = self._dataset_features(lambda b: torch.mean(b, [2, 3]))
        model = self._fit_mixture(torch_gmm, feats, clusters)
        H, W = self._image_size_hw()
        rf, i = self.results_folder, 0
        og_x = model.sample(num_datapoints=num_samples).cuda()[:, :, None, None].expand(num_samples, ch, H, W).float()
        og_x = og_x.contiguous()
        for noise in noise_levels:
            for j in range(repeats):
                xt, direct_recons, all_images = self._ema().gen_sample_2(batch_size=num_samples, img=og_x, noise_level=noise)
                for name, t in (('og', og_x), ('recon', all_images), ('direct_recons', direct_recons), ('xt', xt)):
                    _save(_unit(t), rf / f'sample-{name}-{noise}-{i}-{j}.png')
        return model

    def sample_as_a_blur_torch_gmm(self, torch_gmm=None, siz=4, ch=3, clusters=10, sample_at=1, num_samples=48):
        """mixture over the degraded images at step `sample_at`, shrunk to siz x siz; samples are blown back up and
        restored with `sample_from_blur(start=sample_at)`"""
        H, W = self._image_size_hw()

        def feat(b):
            z = self._ema().opt(b, t=sample_at)
            return F.interpolate(z, size=siz, mode='bilinear').flatten(1)
        feats = self._dataset_features(feat)
        model = self._fit_mixture(torch_gmm, feats, clusters, covariance_regularization=0.0001)
        og_x = model.sample(num_datapoints=num_samples).cuda().reshape(num_samples, ch, siz, siz)
        og_img = F.interpolate(og_x, size=(H, W), mode='bilinear').float().contiguous()
        xt, direct_recons, all_images = self._ema().sample_from_blur(batch_size=num_samples, img=og_img, start=sample_at)
        rf = self.results_folder
        for name, t in (('og', og_img), ('recon', all_images), ('direct_recons', direct_recons), ('xt', xt)):
            _save(_unit(t), rf / f'sample-{name}-{sample_at}-{siz}-{clusters}.png')
        return model

    def sample_and_save_for_fid(self, noise=0, num_samples=6400, bs=128):
        """unconditional generation from Gaussian noise images, one file per sample (DN:821-854)"""
        out_folder = f'{self.results_folder}_out'
        create_folder(out_folder)
        H, W = self._image_size_hw()
        ch = getattr(self._ema(), 'channels', 3)
        cnt = 0
        for _ in range(num_samples // bs):
            og_img = torch.randn(bs, ch, H, W).cuda()
            xt, direct_recons, all_images = self._ema().gen_sample(batch_size=bs, img=og_img)
            for i in range(all_images.shape[0]):
                _save(_unit(all_images[i]), f'{out_folder}/sample-x0-{cnt}.png')
                cnt += 1

    # ---- DB:1567-1705 -----------------------------------------------------------------------------------------
    def fid_distance_decrease_from_manifold(self, fid_func, start=0, end=1000, bs=32, sanity_check=1):
        """degrade every test image, restore it both ways (direct x0-estimate, full sampling) and report FID / RMSE / SSIM
        of degraded, sampled and direct reconstructions against the originals.  `fid_func(samples=[a, b])` as in
        `calculate_fid_given_samples`; pass None to skip FID.  Index quirks of the reference are kept: image `start`
        itself is skipped (`idx > start`), `end` is inclusive."""
        imgs = []
        order = self._manifold_order(len(self.ds))
        for idx in range(len(self.ds)):
            if idx > start:
                item = self.ds[int(order[idx])]
                imgs.append(item[0] if isinstance(item, (tuple, list)) else item)
            if idx % 1000 == 0:
                print(idx)
            if end is not None and idx == end:
                break
        all_samples = torch.stack(imgs)
        sets = {'original': [], 'blurred': [], 'deblurred': [], 'direct': []}
        to3 = lambda t: _unit(self._score_view(t.float().cpu()).repeat(1, 3 // t.shape[1], 1, 1))
        for cnt in range(0, all_samples.shape[0], bs):
            og_img = all_samples[cnt:cnt + bs].cuda().float()
            X_0s, X_ts = self._all_sample(og_img, None)
            batch = {'original': to3(og_img), 'blurred': to3(X_ts[0]), 'deblurred': to3(X_0s[-1]), 'direct': to3(X_0s[0])}
            if cnt == 0 and sanity_check:
                create_folder('./sanity_check/')
                for name, key in (('og', 'original'), ('xt', 'blurred'), ('recons', 'deblurred'), ('direct-recons', 'direct')):
                    _save(batch[key][0:32], f'./sanity_check/sample-{name}.png')
            for k in sets:
                sets[k].append(batch[k])
        sets = {k: torch.cat(v, dim=0) for k, v in sets.items()}
        out = {}
        for key, label in (('blurred', 'blurry'), ('deblurred', 'deblurred'), ('direct', 'direct deblurred')):
            fid = fid_func(samples=[sets['original'], sets[key]]) if fid_func is not None else None
            r = rmse(sets['original'], sets[key])
            s = ssim(sets['original'], sets[key], data_range=1, size_average=True)
            out[key] = dict(fid=fid, rmse=float(r), ssim=float(s))
            print(f'The FID of {label} images with original image is {fid}')
            print(f'The RMSE of {label} images with original image is {r}')
            print(f'The SSIM of {label} images with original image is {s}')
            if key != 'blurred' and fid is not None:
                how = 'sampling' if key == 'deblurred' else 'direct sampling'
                print(f"Hence the improvement in FID using {how} is {out['blurred']['fid'] - fid}")
        return out


# ------------------------------------------------------------------------------------------------------------------------
# snowification / decolor package: its Trainer's own evaluation helpers (SN:682-1200)
# ------------------------------------------------------------------------------------------------------------------------
class _RunningMetric:
    """update((prediction, target)) / compute(): mean of a per-image score, the protocol `save_metric` expects (SN:827-833;
    the `metrics` module `create_metric_dict` refers to is never imported by the reference)"""

    def __init__(self, data_range=1.0):
        self.data_range, self.total, self.count = float(data_range), 0.0, 0

    def reset(self):
        self.total, self.count = 0.0, 0

    def _scores(self, pred, target):
        raise NotImplementedError

    def update(self, output):
        pred, target = output
        s = self._scores(pred.detach().float(), target.detach().float())
        self.total += float(s.sum())
        self.count += int(s.numel())

    def compute(self):
        return torch.tensor(self.total / max(self.count, 1))


class PSNR(_RunningMetric):
    def _scores(self, pred, target):
        mse = ((pred - target) ** 2).flatten(1).mean(1)
        return 10.0 * torch.log10(self.data_range ** 2 / (mse + 1e-10))


class SSIM(_RunningMetric):
    def _scores(self, pred, target):
        return ssim(pred, target, data_range=self.data_range, size_average=False)


class SnowEvaluationMixin:
    """overrides of `EvaluationMixin` for the snowification / decolor Trainer"""

    _cover_batches = 50

    @property
    def _to_show(self):                                       # SN:1151-1152: quarter points of the trajectory + the last step
        T = self.num_timesteps
        return tuple(int(T * i / 4) for i in range(4)) + (T - 1,)

    def add_title(self, path, title_texts):
        """like the base one, with several titles spread over the bar (SN:682-705); a plain string is one title"""
        import cv2
        if isinstance(title_texts, (str, int)):
            title_texts = [title_texts]
        img = cv2.imread(str(path))
        framed = cv2.copyMakeBorder(img, 10, 10, 10, 10, cv2.BORDER_CONSTANT, value=[0, 0, 0])
        bar_h = 20
        bar = np.zeros((bar_h, framed.shape[1], 3), np.uint8)
        bar[:] = (255, 0, 180)
        out = cv2.vconcat((bar, framed))
        n = len(title_texts)
        for i, title in enumerate(title_texts):
            x = i * (bar.shape[1] // n) + bar.shape[1] // (n * 2)
            cv2.putText(out, str(title), (x, bar_h - 2), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (0, 0, 0), 1, 0)
        cv2.imwrite(str(path), out)

    def make_transparent(self, path):
        import matplotlib.image as mpimg                       # optional dependency, as in the reference (SN:707-711)
        import matplotlib.pyplot as plt
        plt.imshow(mpimg.imread(path))
        plt.savefig(path, transparent=True)
        plt.close()

    def shift_data_range(self, img):
        return (img + 1.0) / 2

    def create_metric_dict(self):
        return {'PSNR': [PSNR(data_range=1.0) for _ in range(self.num_timesteps)],
                'SSIM': [SSIM(data_range=1.0) for _ in range(self.num_timesteps)]}

    def save_metric(self, metric_dict, prefix=''):
        for k, v in metric_dict.items():
            with open(str(self.results_folder / f'{prefix}-{k}.txt'), 'w') as f:
                f.writelines([f'{str(m.compute().item())}\n' for m in v])

    def save_og_test(self, og_dict, extra_path):
        """writes every entry as a titled grid and replaces it by the grid (SN:810-817)"""
        from torchvision import utils
        for k, img in og_dict.items():
            grid = utils.make_grid(_unit(img.cpu()), nrow=6)
            utils.save_image(grid, str(self.results_folder / f'{k}-{extra_path}.png'))
            self.add_title(str(self.results_folder / f'{k}-{extra_path}.png'), '{k}')      # the literal '{k}', as there
            og_dict[k] = grid

    def save_gif(self, X_0s, X_ts, extra_path, init_recon=None, og=None):
        """per step: the x0-estimate grid and the x_t grid, each next to the original grid (and the first reconstruction
        when given), titled; two GIFs (SN:764-807).  `og` is the grid `save_og_test` left in the dictionary."""
        from torchvision import utils
        rf = self.results_folder
        init_grid = None if init_recon is None else utils.make_grid(_unit(init_recon.cpu()), nrow=6)
        self.gif_len = len(X_0s)
        frames_0, frames_t = [], []
        for i in range(len(X_0s)):
            titles = [str(i)]

            def compose(g):
                if init_grid is not None:
                    return utils.make_grid(torch.stack((g, og, init_grid)), nrow=3), [str(i), 'og', 'init_recon']
                if og is not None:
                    return utils.make_grid(torch.stack((g, og)), nrow=2), [str(i), 'og']
                return g, titles
            for lst, tag, frames in ((X_0s, 'x0', frames_0), (X_ts, 'xt', frames_t)):
                g, titles_ = compose(utils.make_grid(_unit(lst[i].cpu()), nrow=6))
                p = rf / f'sample-{i}-{extra_path}-{tag}.png'
                utils.save_image(g, str(p))
                self.add_title(str(p), titles_)
                frames.append(p)
        _write_gif(rf / f'Gif-{extra_path}-x0.gif', frames_0)
        _write_gif(rf / f'Gif-{extra_path}-xt.gif', frames_t)

    def _plain_batch(self):
        if getattr(self, 'data_loader', None) is not None:
            return self._process_item(next(iter(self.data_loader))).cuda()
        return self._eval_batch()

    def test_from_data(self, extra_path, s_times=None):
        """first batch of the (un-cycled) loader through `all_sample`; originals + titled trajectory grids + GIFs (SN:838-863)"""
        og_img = self._plain_batch()
        og_dict = {'og': og_img}
        X_0s, X_ts, init_recon, img_forward_list = self._ema().all_sample(batch_size=self.batch_size, img=og_img, times=s_times,
                                                                          res_dict=og_dict)
        og_dict['og'] = og_img.cpu()
        self.save_og_test(og_dict, extra_path)
        self.save_gif(X_0s, X_ts, extra_path, init_recon=init_recon, og=og_dict['og'])

    def test_with_mixup(self, extra_path):
        """reverse process from the average of two batches (SN:865-882)"""
        a, b = self._eval_batch(), self._eval_batch()
        og_img = (a + b) / 2
        X_0s, X_ts = self._all_sample(og_img)
        og_dict = {'og1': a, 'og2': b, 'og': og_img}
        self.save_og_test(og_dict, extra_path)
        self.save_gif(X_0s, X_ts, extra_path, og=og_dict['og'])

    def test_from_random(self, extra_path):
        """reverse process from a batch scaled by 0.9 (SN:884-895)"""
        og_img = self._eval_batch() * 0.9
        og_dict = {'og': og_img}
        r = self._ema().all_sample(batch_size=self.batch_size, img=og_img, res_dict=og_dict)
        self.save_og_test(og_dict, extra_path)
        self.save_gif(r[0], r[1], extra_path, og=og_dict['og'])

    def paper_invert_section_images(self, s_times=None, n_batches=20, group=9):
        """3 x 3 grids of degraded | direct | sampled | original (SN:897-958; windows j..j+9 for j < B // 9, as there)"""
        import cv2
        rf, cnt = self.results_folder, 0
        for _ in range(n_batches):
            og_img = self._eval_batch()
            X_0s, X_ts = self._all_sample(og_img, s_times)
            og = _unit(og_img)
            for j in range(og.shape[0] // group):
                tiles = []
                for name, t in (('blurry_image', _unit(X_ts[0][j:j + group])), ('direct_recons', _unit(X_0s[0][j:j + group])),
                                ('sampling_recons', _unit(X_0s[-1][j:j + group])), ('original', og[j:j + group])):
                    _save(t, rf / f'{name}_{cnt}.png', nrow=3)
                    tiles.append(cv2.copyMakeBorder(cv2.imread(f'{rf}/{name}_{cnt}.png'), 10, 10, 10, 10,
                                                    cv2.BORDER_CONSTANT, value=[0, 0, 0]))
                cv2.imwrite(f'{rf}/all_{cnt}.png', cv2.hconcat(tiles))
                cnt += 1

    def paper_showing_diffusion_images(self, s_times=None, n_batches=5, to_show=(0, 1, 2, 4, 8, 16, 24, 32, 40, 44, 46, 48, 49)):
        return EvaluationMixin.paper_showing_diffusion_images(self, s_times=s_times, n_batches=n_batches, to_show=to_show)

    def _manifold_order(self, n):
        return np.random.permutation(n)                        # SN:1008

    def _score_view(self, t):
        return F.interpolate(t, size=64) if t.shape[2] > 256 else t       # SN:1043-1047

    def fid_distance_decrease_from_manifold(self, fid_func, start=0, end=1000, bs=16, sanity_check=0):
        """the base routine over a random permutation of the data set, 16 images at a time, no sanity-check dump; images wider
        than 256 px are scored on 64 px copies (SN:1000-1145)"""
        return EvaluationMixin.fid_distance_decrease_from_manifold(self, fid_func, start=start, end=end, bs=bs,
                                                                   sanity_check=sanity_check)


# ------------------------------------------------------------------------------------------------------------------------
# FID feature network (Fid/inception.py): torchvision's InceptionV3 with the pooling of the TensorFlow FID graph
# ------------------------------------------------------------------------------------------------------------------------
class InceptionV3(torch.nn.Module):
    """Feature maps of the InceptionV3 used for FID (Fid/inception.py:16-164; a vendored copy of pytorch-fid upstream).

    Same constructor, block indices and outputs as there.  The FID graph differs from torchvision's InceptionV3 only in the
    pooling that feeds `branch_pool` of the A / C / E blocks: 3x3 average pooling that does not count the zero padding
    (all of them but the last), 3x3 max pooling in the last block (Fid/inception.py:211-326).  Instead of re-deriving the
    blocks, torchvision's modules are used as they are and the input of each `branch_pool` is corrected by hooks: average
    pooling without the padding equals average pooling with it times 9 / (number of in-image taps), a fixed per-pixel factor;
    the last block's `branch_pool` gets the max-pooled block input instead.

    Weights: `weights_path` (or $COLDDIFF_FID_WEIGHTS) names a local copy of pytorch-fid's
    `pt_inception-2015-12-05-6726825d.pth` (same parameter names as torchvision, 1008 classes).  Nothing is downloaded;
    without a file the constructor raises unless `weights_path=False` (random initialisation, for tests)."""

    DEFAULT_BLOCK_INDEX = 3
    BLOCK_INDEX_BY_DIM = {64: 0, 192: 1, 768: 2, 2048: 3}

    def __init__(self, output_blocks=(DEFAULT_BLOCK_INDEX,), resize_input=True, normalize_input=True, requires_grad=False,
                 use_fid_inception=True, weights_path=None):
        super().__init__()
        import torchvision
        self.resize_input, self.normalize_input = resize_input, normalize_input
        self.output_blocks = sorted(output_blocks)
        self.last_needed_block = max(output_blocks)
        assert self.last_needed_block <= 3, 'Last possible output block index is 3'
        net = torchvision.models.inception_v3(weights=None, aux_logits=False, num_classes=1008 if use_fid_inception else 1000,
                                              init_weights=False)
        if weights_path is None:
            weights_path = os.environ.get('COLDDIFF_FID_WEIGHTS')
        if weights_path is None:
            raise RuntimeError("InceptionV3 needs weights_path=<pt_inception-2015-12-05-6726825d.pth> (or $COLDDIFF_FID_WEIGHTS); "
                               "the reference downloads that file, this engine does not")
        if weights_path is not False:
            net.load_state_dict(torch.load(weights_path, map_location='cpu'))
        pool = lambda: torch.nn.MaxPool2d(kernel_size=3, stride=2)
        stages = [[net.Conv2d_1a_3x3, net.Conv2d_2a_3x3, net.Conv2d_2b_3x3, pool()],
                  [net.Conv2d_3b_1x1, net.Conv2d_4a_3x3, pool()],
                  [net.Mixed_5b, net.Mixed_5c, net.Mixed_5d, net.Mixed_6a, net.Mixed_6b, net.Mixed_6c, net.Mixed_6d, net.Mixed_6e],
                  [net.Mixed_7a, net.Mixed_7b, net.Mixed_7c, torch.nn.AdaptiveAvgPool2d(output_size=(1, 1))]]
        self.blocks = torch.nn.ModuleList(torch.nn.Sequential(*st) for st in stages[:self.last_needed_block + 1])
        if use_fid_inception:
            if self.last_needed_block >= 2:
                for m in (net.Mixed_5b, net.Mixed_5c, net.Mixed_5d, net.Mixed_6b, net.Mixed_6c, net.Mixed_6d, net.Mixed_6e):
                    m.branch_pool.register_forward_pre_hook(self._exclude_padding)
            if self.last_needed_block >= 3:
                net.Mixed_7b.branch_pool.register_forward_pre_hook(self._exclude_padding)
                stash = {}
                net.Mixed_7c.register_forward_pre_hook(lambda mod, args: stash.__setitem__('x', args[0]))
                net.Mixed_7c.branch_pool.register_forward_pre_hook(
                    lambda mod, args: (F.max_pool2d(stash.pop('x'), kernel_size=3, stride=1, padding=1),))
        for p in self.parameters():
            p.requires_grad = requires_grad

    @staticmethod
    def _exclude_padding(module, args):
        """avg_pool2d(3, 1, 1) counted 9 taps everywhere; rescale so that only the taps inside the image count"""
        x = args[0]
        H, W = x.shape[-2:]
        ny = torch.full((H,), 3.0, device=x.device, dtype=x.dtype)
        nx = torch.full((W,), 3.0, device=x.device, dtype=x.dtype)
        ny[0] -= 1; ny[-1] -= 1; nx[0] -= 1; nx[-1] -= 1          # a 1-pixel axis ends at 1 tap, as it should
        return (x * (9.0 / (ny[:, None] * nx[None, :])),)

    def forward(self, inp):
        """inp: (B, 3, H, W) in [0, 1] -> list of the selected blocks' outputs, ascending by index"""
        out, x = [], inp
        if self.resize_input:
            x = F.interpolate(x, size=(299, 299), mode='bilinear', align_corners=False)
        if self.normalize_input:
            x = 2 * x - 1
        for idx, block in enumerate(self.blocks):
            x = block(x)
            if idx in self.output_blocks:
                out.append(x)
            if idx == self.last_needed_block:
                break
        return out
