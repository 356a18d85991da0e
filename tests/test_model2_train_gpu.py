"""GPU parity of the `Model` (DDPM UNet) TRAINING path: every parameter gradient through the real library against the
reference (tests/golden/model2_grads_small.npz), fp32 CUDA-core convolutions tight and tensor-core (TF32) within the north-star
tolerance, plus dropout consistency and one Trainer step.

The host logic of the same schedule is checked on CPU by tests/test_model2_host_logic.py."""
import os
import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu]
G = os.path.join(os.path.dirname(__file__), 'golden')


def load(name):
    z = np.load(os.path.join(G, name + '.npz'))
    return {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def build(dropout=0.1):
    import cold_diffusion_models_b200 as cdm
    g = load('model2_small')
    m = cdm.Model(resolution=16, in_channels=3, out_ch=3, ch=32, ch_mult=(1, 2), num_res_blocks=2, attn_resolutions=(8,), dropout=dropout)
    m.load_state_dict({k[3:]: v for k, v in g.items() if k.startswith('sd:')})
    return m.cuda(), g


def check_grads(m, gg, tol):
    named = dict(m.named_parameters())
    worst = (-1.0, '')
    for k, v in gg.items():
        if k.startswith('grad:'):
            mine = named[k[5:]].grad
        elif k.startswith('gsub:'):
            gr = named[k[5:]].grad.reshape(-1)
            mine = gr[::gr.numel() // 2048]
        else:
            continue
        e = rel(mine, v)
        if (mine.double().cpu() - v.double()).abs().max().item() < 1e-6:     # exact-arithmetic zeros (see test_model2_host_logic.py)
            e = 0.0
        worst = max(worst, (e, k))
    assert worst[0] < tol, worst


@pytest.mark.parametrize('impl', ['simt', 'tc'])
def test_model_gradients_match_reference_golden(impl):
    from cold_diffusion_models_b200.ops import CONV_SIMT, CONV_TC
    m, g = build()
    gg = load('model2_grads_small')
    m.eval()                                               # dropout inactive, as in the golden
    m.conv_impl = CONV_SIMT if impl == 'simt' else CONV_TC
    y = m(g['x'].cuda(), g['t'].cuda())
    assert rel(y, g['y']) < (2e-5 if impl == 'simt' else 1.5e-3)
    if impl == 'simt':
        loss = (gg['target'].cuda() - y).abs().mean()
        assert abs(loss.item() - gg['loss'].item()) < 2e-5
        loss.backward()
        torch.cuda.synchronize()
        check_grads(m, gg, 5e-4)
    else:
        # TF32: compare with the smooth L2 loss against oracle autograd (an L1 loss flips sign() on 1e-4-level forward differences)
        import model2_oracle as MO
        sd = {k[3:]: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in g.items() if k.startswith('sd:')}
        yo = MO.model_forward(sd, g['x'], g['t'], ch=32, num_resolutions=2, num_res_blocks=2)
        ((gg['target'] - yo) ** 2).mean().backward()
        ((gg['target'].cuda() - y) ** 2).mean().backward()
        torch.cuda.synchronize()
        errs = sorted(rel(p.grad, sd[n].grad) for n, p in m.named_parameters() if sd[n].grad.abs().max() > 1e-6)
        assert errs[len(errs) // 2] < 3e-3 and errs[-1] < 3e-2, (errs[len(errs) // 2], errs[-1])


def test_dropout_forward_backward_use_the_same_mask():
    """with dropout active the loss still decreases along the negative gradient (finite-difference check of one direction)"""
    from cold_diffusion_models_b200.ops import CONV_SIMT
    m, g = build(dropout=0.3)
    m.train(); m.conv_impl = CONV_SIMT
    x, t = g['x'].cuda(), g['t'].cuda()
    target = torch.zeros_like(x)
    torch.manual_seed(5)
    loss = ((target - m(x, t)) ** 2).mean()
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    gnorm2 = sum((v.double() ** 2).sum().item() for v in grads.values())
    eps = 1e-3 / gnorm2 ** 0.5
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.add_(grads[n], alpha=-eps)
    m.engine.mark_weights_dirty()
    # second forward under autograd so that the training-mode (dropout) path runs again; same host seeds -> same masks
    torch.manual_seed(5)
    loss2 = ((target - m(x, t)) ** 2).mean()
    predicted = -eps * gnorm2
    assert abs((loss2.item() - loss.item()) - predicted) < 0.2 * abs(predicted)


def test_trainer_step_with_model(tmp_path):
    import cold_diffusion_models_b200 as cdm
    m, g = build()
    gd = cdm.GaussianDiffusion(m, image_size=16, device_of_kernel='cuda', channels=3, timesteps=6, kernel_std=0.1, kernel_size=3,
                               blur_routine='Special_6_routine', sampling_routine='x0_step_down').cuda()
    tr = cdm.Trainer(gd, None, image_size=16, train_batch_size=3, gradient_accumulate_every=2, results_folder=str(tmp_path), dataset='synthetic')
    before = m.engine.flat_param.clone()
    loss = tr.train_step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item() and (m.engine.flat_param - before).abs().max().item() > 0
