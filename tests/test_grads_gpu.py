"""GPU parity of the training step's gradients (loss.backward through the engine) against the gradients the
unmodified reference produced with torch autograd (tests/golden/unet_small.npz)."""
import os
import io
import contextlib
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), 'golden')


def load(name):
    z = np.load(os.path.join(G, name + '.npz'))
    return {k: torch.from_numpy(np.asarray(z[k])) for k in z.files}


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _grads(u, x, t, target, mode):
    from cold_diffusion_models_b200.deblurring import _LossFn
    for p in u.parameters():
        p.grad = None
    u.engine.flat_grad.zero_() if getattr(u.engine, 'flat_grad', None) is not None else None
    y = u(x.cuda(), t.cuda())
    loss = _LossFn.apply(target.cuda(), y, mode)
    loss.backward()
    torch.cuda.synchronize()
    return loss


def _small_unet(sd):
    import cold_diffusion_models_b200 as cdm
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
    u.load_state_dict(sd)
    return u.cuda()


def test_unet_gradients_match_reference_golden_fp32_path():
    """every parameter gradient of the L1 training loss, fp32 CUDA-core convolutions, vs the gradients the unmodified
    reference produced with torch autograd."""
    from cold_diffusion_models_b200.ops import CONV_SIMT
    g = load('unet_small')
    sd = {k[3:]: v for k, v in g.items() if k.startswith('sd:')}
    u = _small_unet(sd)
    u.engine.conv_impl = CONV_SIMT
    loss = _grads(u, g['x'], g['t'], g['target'], 0)
    assert abs(loss.item() - g['loss'].item()) < 1e-5
    worst = (0.0, None)
    for n, p in u.named_parameters():
        assert p.grad is not None, n
        if ('grad:' + n) in g:
            e = rel(p.grad, g['grad:' + n])
        else:
            gr = p.grad.reshape(-1)
            stride = gr.numel() // 2048
            e = rel(gr[::stride], g['gsub:' + n])
            assert abs(gr.double().norm().item() / g['gnorm:' + n].item() - 1) < 2e-4, n
        worst = max(worst, (e, n))
        assert e < 2e-4, (n, e)
    print('worst relative gradient error (fp32 path): %.3e at %s' % worst)


def test_unet_gradients_tf32_path_vs_oracle_autograd():
    """tensor-core (TF32) forward + data-gradient convolutions vs the fp32 CPU oracle's autograd, with the smooth L2 loss
    (the L1 loss' sign() gradient flips on 1e-4-level forward differences, which would mask what is being tested).
    The reference's own GPU path also runs convolutions in TF32 (torch.backends.cudnn.allow_tf32 defaults to True)."""
    import unet_oracle as UO
    g = load('unet_small')
    sd = {k[3:]: v for k, v in g.items() if k.startswith('sd:')}
    ref = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    y = UO.unet_forward(ref, g['x'], g['t'])
    torch.nn.functional.mse_loss(g['target'], y).backward()
    u = _small_unet(sd)
    _grads(u, g['x'], g['t'], g['target'], 1)
    errs = sorted((rel(p.grad, ref[n].grad), n) for n, p in u.named_parameters())
    os.makedirs('gpurun_out', exist_ok=True)
    with open('gpurun_out/grad_errors_tc.txt', 'w') as f:
        f.write('median %.3e  p90 %.3e  max %.3e\n' % (errs[len(errs) // 2][0], errs[int(len(errs) * 0.9)][0], errs[-1][0]))
        for e, n in errs[-10:]:
            f.write('%.3e %s\n' % (e, n))
    # the TF32 operand rounding (2^-11 relative per operand, what cuDNN's default path does too) accumulated over the ~70 convolutions between the
    # loss and the first block; the fp32 CUDA-core path of the same schedule is at 2e-6 (test above)
    assert errs[len(errs) // 2][0] < 1.1e-3 and errs[-1][0] < 1.5e-3, errs[-3:]


def test_gradient_accumulation_and_flat_buffer():
    """two backward passes accumulate (Trainer's gradient_accumulate_every=2, DB:1190-1196) and every
    parameter's .grad is a view of the engine's flat buffer (what the all-reduce and Adam consume)."""
    import cold_diffusion_models_b200 as cdm
    from cold_diffusion_models_b200.deblurring import _LossFn
    g = load('unet_small')
    sd = {k[3:]: v for k, v in g.items() if k.startswith('sd:')}
    with contextlib.redirect_stdout(io.StringIO()):
        u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
    u.load_state_dict(sd)
    u = u.cuda()
    for _ in range(2):
        y = u(g['x'].cuda(), g['t'].cuda())
        (_LossFn.apply(g['target'].cuda(), y, 0) / 2).backward()
    torch.cuda.synchronize()
    eng = u.engine
    lo, hi = eng.flat_grad.data_ptr(), eng.flat_grad.data_ptr() + 4 * eng.flat_grad.numel()
    for n, p in u.named_parameters():
        assert lo <= p.grad.data_ptr() < hi, n
    w = 'downs.1.0.net.1.weight'
    assert rel(dict(u.named_parameters())[w].grad.reshape(-1)[::(dict(u.named_parameters())[w].numel() // 2048)],
               g['gsub:' + w]) < 1e-2
