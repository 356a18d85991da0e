"""Per-launch time of every tensor-core weight-gradient GEMM of one Unet backward (config 3 network), grouped by shape, under
the kernel choices and K-split policies of csrc/wgrad_tc.cu (cd_wgrad_tc_set_mode / cd_wgrad_tc_set_split):

  wgmma      mode 1 (default): the wgmma kernel for the stride-1 3x3 shapes it takes, the mma.sync kernels for the rest
  mma.sync   mode 8: the mma.sync halo kernel everywhere (the weight gradient before the wgmma kernel)
  2waves-up / 1wave / 2waves / model-12k: K-split policies 0 / 1 / 2 / 3 of the default kernel choice

    python tools/wgrad_shapes.py [B] [config,config,...]      (default: B = 32, wgmma,mma.sync)

The configurations are taken in turns, so that clock drift under the power cap hits them all alike.  Per shape it prints
microseconds per launch and achieved TFLOP/s of each configuration, and for the 3x3 shapes the modelled shared-memory bytes per
FLOP of each kernel (the mainloop's shared-memory traffic: operand loads, TMA writes, the dY transposition; bank conflicts
counted as extra wavefronts), then the totals per backward: all shapes, the 3x3 shapes alone and the rest.  The per-batch
attention product dweff is listed with stride 'batch'."""
import sys, io, contextlib, os, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import cold_diffusion_models_b200 as cdm
from cold_diffusion_models_b200._lib import lib

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
# name: (cd_wgrad_tc_set_mode, split policy, per-CTA overhead in SM clocks)
ALL = collections.OrderedDict([('wgmma', (1, 3, 12000)), ('mma.sync', (8, 3, 12000)), ('2waves-up', (1, 0, 0)),
                               ('1wave', (1, 1, 0)), ('2waves', (1, 2, 0)), ('model-12k', (1, 3, 12000))])
names = sys.argv[2].split(',') if len(sys.argv) > 2 else ['wgmma', 'mma.sync']
ROUNDS = 3

with contextlib.redirect_stdout(io.StringIO()):
    u = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
x = torch.rand(B, 3, 128, 128, device='cuda') * 2 - 1
t = torch.randint(0, 200, (B,), device='cuda')
target = torch.rand(B, 3, 128, 128, device='cuda')


def step():
    y = u(x, t)
    ((y - target) ** 2).mean().backward()


def apply(name):
    mode, pol, over = ALL[name]
    lib.cd_wgrad_tc_set_mode(mode)
    lib.cd_wgrad_tc_set_split(pol, over)


def cdiv(a, b):
    return -(-a // b)


def smem_bytes_per_flop(shp, kernel):
    """modelled shared-memory bytes per FLOP of one chunk of one CTA (stride-1 3x3 shapes; None for the rest)"""
    _, H, W, Cout, Cin, nt, stride = shp
    if nt != 9 or stride != 1:
        return None
    if kernel == 'wgmma':
        if Cin % 64 or Cout % 64:
            return None
        bn = 128 if Cout % 128 == 0 else 64
        taps = 4 if bn == 128 else 8              # taps of a full tap group
        cw = 16 if W >= 16 else 8
        r = 64 // cw
        flop = taps * 64 * bn * 64 * 2
        a = taps * 64 * 64 * 4                    # A fragments: conflict-free LDS
        b = taps * bn * 64 * 4                    # wgmma reads of the transposed dY tile
        tma = 2 * (cw + 8) * (r + 2) * 128 + bn * 64 * 4
        transpose = 2 * bn * 64 * 4
        return (a + b + tma + transpose) / flop
    # mma.sync halo kernel: 128 co x 64 ci x 3 taps per CTA, 64-pixel chunks; per warp and k8 step 8 A + 3 x 4 x 2 B scalar LDS,
    # each 2-way bank-conflicted (256 bytes of wavefronts)
    cw = min(W, 64)
    r = 64 // cw
    flop_k8 = 3 * 128 * 64 * 8 * 2
    lds_k8 = 8 * 32 * 256
    tma = (128 * 64 * 4 + (cw + 2) * r * 64 * 4) / 8
    return (lds_k8 + tma) / flop_k8


for nm in names:                     # warm every configuration once
    apply(nm)
    for _ in range(2):
        step()
res = {nm: collections.OrderedDict() for nm in names}
for rnd in range(ROUNDS):
    for nm in names:
        apply(nm)
        step()
        u.engine.profile_wgrads = []
        step()
        torch.cuda.synchronize()
        for a, b, shp in u.engine.profile_wgrads:
            e = res[nm].setdefault(shp, [0, 0.0])
            e[0] += 1; e[1] += a.elapsed_time(b)
        u.engine.profile_wgrads = None
apply('wgmma')

print("%-34s %3s " % ("(B,H,W,Cout,Cin,taps,stride)", "n") + " ".join("%10s" % n for n in names) + "  " +
      " ".join("%9s" % ('TF/s ' + n[:4]) for n in names) + "   B/FLOP wgmma mma.sync")
tot = {n: 0.0 for n in names}
tot3 = {n: 0.0 for n in names}
for shp in res[names[0]]:
    n = res[names[0]][shp][0] // ROUNDS
    fl = 2.0 * shp[0] * shp[1] * shp[2] * shp[3] * shp[4] * shp[5]
    us, tf = [], []
    for nm in names:
        ms = res[nm][shp][1] / ROUNDS
        tot[nm] += ms
        if shp[5] == 9 and shp[6] == 1:
            tot3[nm] += ms
        us.append(ms / n * 1e3)
        tf.append(fl / (ms / n * 1e-3) / 1e12)
    mw, ms_ = smem_bytes_per_flop(shp, 'wgmma'), smem_bytes_per_flop(shp, 'mma.sync')
    model = ("%12.3f" % mw if mw else "%12s" % '-') + ("%9.3f" % ms_ if ms_ else "%9s" % '-')
    print("%-34s %3d " % (str(shp), n) + " ".join("%10.1f" % v for v in us) + "  " + " ".join("%9.1f" % v for v in tf) + model)
print("%-34s     " % "total ms per backward" + " ".join("%10.3f" % tot[n] for n in names))
print("%-34s     " % "other shapes ms per backward" + " ".join("%10.3f" % (tot[n] - tot3[n]) for n in names))
print("%-34s     " % "3x3 (stride 1) ms per backward" + " ".join("%10.3f" % tot3[n] for n in names))
if len(names) > 1 and tot3[names[0]] > 0:
    print("3x3 total, %s / %s: %.2fx" % (names[1], names[0], tot3[names[1]] / tot3[names[0]]))
