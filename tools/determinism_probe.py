"""Run the same Unet forward repeatedly and report run-to-run differences under a few kernel switches."""
import sys, os, io, contextlib
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
import numpy as np, torch
import cold_diffusion_models_b200 as cdm
from cold_diffusion_models_b200._lib import lib
from cold_diffusion_models_b200.ops import CONV_SIMT, CONV_TC

z = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'unet_small.npz'))
sd = {k[3:]: torch.from_numpy(np.asarray(z[k])) for k in z.files if k.startswith('sd:')}
with contextlib.redirect_stdout(io.StringIO()):
    u = cdm.Unet(dim=32, dim_mults=(1, 2), channels=3)
u.load_state_dict(sd); u = u.cuda()
x = torch.from_numpy(np.asarray(z['x'])).cuda()
t = torch.tensor([3, 1]).cuda()


def probe(tag, n=40):
    with torch.no_grad():
        ref = u(x, t).clone()
        bad, worst = 0, 0.0
        for _ in range(n):
            y = u(x * 1.0, t)
            if not torch.equal(y, ref):
                bad += 1; worst = max(worst, (y - ref).abs().max().item())
    print("%-28s mismatching runs %2d/%d  max abs diff %.3e" % (tag, bad, n, worst))


probe('default')
lib.cd_dwconv7_set_pipe(0); probe('dwconv pipe off'); lib.cd_dwconv7_set_pipe(1)
u.engine.conv_impl = CONV_SIMT; probe('conv SIMT'); u.engine.conv_impl = CONV_TC
# per-stage check: which engine buffers differ between two runs
with torch.no_grad():
    u(x, t); torch.cuda.synchronize()
    snap = {k: v.clone() for k, v in u.engine._bufs.items()} if hasattr(u.engine, '_bufs') else {}
    for rep in range(10):
        u(x, t); torch.cuda.synchronize()
        diff = [k for k, v in u.engine._bufs.items() if k in snap and not torch.equal(v, snap[k])] if snap else []
        if diff:
            print('differing buffers:', diff[:12]); break
    else:
        print('no differing buffers in 10 reruns (or engine has no _bufs)')
