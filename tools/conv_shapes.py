"""Per-launch time of every tensor-core convolution of one Unet forward (config 3 network), grouped by GEMM shape, under the
library's kernel-selection switches side by side."""
import sys, io, contextlib, os, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import cold_diffusion_models_b200 as cdm
from cold_diffusion_models_b200._lib import lib

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
# name: (SM-pair mode, SM-pair N-tile mask, halo-kernel mask, two-CTAs-per-SM mask) -- cd_conv_tc_set_2cta / _2cta_bn / _halo /
# _two_ctas
CONFIGS = collections.OrderedDict([
    ('per-tap', (0, 0, 0, 0)),
    ('pair256', (1, 0, 0, 0)),
    ('pair+128', (1, 128, 0, 0)),
    ('halo16x8', (0, 0, 1, 0)),
    ('halo16x16', (0, 0, 2, 0)),
    ('2ctas', (0, 0, 0, 192)),
])
DEFAULT = (0, 0, 0, 0)


def apply(cfg):
    lib.cd_conv_tc_set_2cta(cfg[0]); lib.cd_conv_tc_set_2cta_bn(cfg[1]); lib.cd_conv_tc_set_halo(cfg[2]); lib.cd_conv_tc_set_two_ctas(cfg[3])


with contextlib.redirect_stdout(io.StringIO()):
    u = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
x = torch.rand(B, 3, 128, 128, device='cuda') * 2 - 1
t = torch.randint(0, 200, (B,), device='cuda')
res = {}
with torch.no_grad():
    for name, cfg in CONFIGS.items():
        apply(cfg)
        for _ in range(2):
            u(x, t)
        acc = collections.OrderedDict()
        for rep in range(5):
            u.engine.profile_convs, u.engine.profile_shapes = [], []
            u(x, t)
            torch.cuda.synchronize()
            for (a, b, f), shp in zip(u.engine.profile_convs, u.engine.profile_shapes):
                e = acc.setdefault(shp, [0, 0.0, f])
                e[0] += 1; e[1] += a.elapsed_time(b)
        u.engine.profile_convs = u.engine.profile_shapes = None
        res[name] = acc
apply(DEFAULT)
names = list(CONFIGS)
print("%-42s %3s" % ("(B,Hg,Wg,Cout,K,nsrc,per_batch)", "n") + ''.join(' %12s' % n for n in names) + '   | TFLOP/s: ' + ' '.join(names))
tot = {n: 0.0 for n in names}
for shp, (n, ms, f) in res[names[0]].items():
    n //= 5
    us = [res[m][shp][1] / 5 / n * 1e3 for m in names]
    for m in names:
        tot[m] += res[m][shp][1] / 5
    print("%-42s %3d" % (str(shp), n) + ''.join(' %12.1f' % v for v in us) + '   | ' + ' '.join('%6.0f' % (f / v / 1e6) for v in us))
print("total conv ms per forward: " + '   '.join('%s %.3f' % (m, tot[m]) for m in names))
