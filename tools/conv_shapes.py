"""Per-launch time of every tensor-core convolution of one Unet forward and of the data-gradient launches of its backward
(config 3 network; `fwd` / `dgrad` rows), grouped by GEMM shape, under the library's kernel-selection switches side by side,
with a traffic model of each launch:

  L2 MB   modelled L2 -> SM bytes of one launch: (A + B bytes per k-iteration) x k-iterations x output tiles, for the per-tap
          kernel (one 128-pixel x 32-channel A box per tap), for the shared-row kernel with 16 x 8 pixel tiles (one 16 x (8 + 2)
          box per distinct tap column dx, read by every tap of that column) and for the one with 16 x 16 pixel tiles (one
          16 x (16 + 2) box per tap column and one weight tile per tap for 256 pixels); '-' where the problem is not eligible;
  HBM MB  modelled DRAM bytes: every source and weight read once, plus out / out2 / resid / aux;
  then per configuration: microseconds per launch, achieved TFLOP/s, and the L2 -> SM and HBM byte rates (GB/s) implied by that
  time (the L2 rate uses the model of the kernel that configuration runs; none for 'default', which chooses by shape).

    python tools/conv_shapes.py [batch [config,config,...]]     # default: batch 32, every configuration"""
import sys, io, contextlib, os, collections, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import cold_diffusion_models_b200 as cdm
from cold_diffusion_models_b200 import ops
from cold_diffusion_models_b200._lib import lib

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
# name: ((SM-pair mode, SM-pair N-tile mask, shared-row mode, two-CTAs-per-SM mask), kernel the traffic model follows) --
# cd_conv_tc_set_2cta / _2cta_bn / _halo / _two_ctas.  Shared-row mode: 0 = shape-based choice, 1 = 16 x 8 tiles wherever
# eligible, 4 = 16 x 16 tiles wherever eligible, 8 = per-tap kernel everywhere
PER_TAP = 8
CONFIGS = collections.OrderedDict([
    ('per-tap', ((0, 0, PER_TAP, 0), 'tap')),
    ('pair256', ((1, 0, PER_TAP, 0), 'tap')),
    ('pair+128', ((1, 128, PER_TAP, 0), 'tap')),
    ('2ctas', ((0, 0, PER_TAP, 192), 'tap')),
    ('rows', ((0, 0, 1, 0), 'rows')),
    ('rows2ctas', ((0, 0, 1, 192), 'rows')),
    ('rows256', ((0, 0, 4, 192), 'rows256')),
    ('default', ((0, 0, 0, 192), None)),
])
if len(sys.argv) > 2:
    CONFIGS = collections.OrderedDict((n, CONFIGS[n]) for n in sys.argv[2].split(','))
DEFAULT = (0, 0, 0, 192)
SMS = torch.cuda.get_device_properties(0).multi_processor_count


def apply(cfg):
    lib.cd_conv_tc_set_2cta(cfg[0]); lib.cd_conv_tc_set_2cta_bn(cfg[1]); lib.cd_conv_tc_set_halo(cfg[2]); lib.cd_conv_tc_set_two_ctas(cfg[3])


def cdiv(a, b):
    return -(-a // b)


def tap_tile_cost(m_tiles, cout, bn):      # conv_tc.cu: tc_cost (N-tile choice of the per-tap kernel)
    rate = {256: 0.92, 128: 0.75, 64: 0.40}[bn]
    return cdiv(m_tiles * cdiv(cout, bn), SMS) * bn / rate


def rows_eligible(d):
    if d.sy != 1 or d.sx != 1 or d.s[0].ntaps < 3 * len({d.s[0].dx[t] for t in range(d.s[0].ntaps)}):
        return False
    for s in range(d.nsrc):
        cs = d.s[s]
        if cs.w_per_batch or cs.C % 32 or cs.W != d.Wg or cs.H != d.Hg:
            return False
        if any(not (-1 <= cs.dy[t] <= 1 and -1 <= cs.dx[t] <= 1) for t in range(cs.ntaps)):
            return False
    return True


def traffic(d):
    """modelled bytes of one launch: {'tap': L2 bytes of the per-tap kernel, 'rows' / 'rows256': of the shared-row kernel with
    16 x 8 / 16 x 16 pixel tiles (None when not eligible), 'hbm': DRAM bytes}"""
    res = {}
    if d.Wg >= 128:
        tw, th, tn = 128, 1, 1
    else:
        tw = d.Wg; th = min(128 // tw, d.Hg); tn = 128 // (tw * th)
    mt = (d.Wg // tw) * (d.Hg // th) * cdiv(d.B, tn)
    bn = 256 if d.Cout % 256 == 0 else (128 if d.Cout > 64 else 64)
    if bn == 256 and tap_tile_cost(mt, d.Cout, 128) < tap_tile_cost(mt, d.Cout, 256):
        bn = 128
    kiters = sum(d.s[s].ntaps * (d.s[s].C // 32) for s in range(d.nsrc))
    res['tap'] = mt * cdiv(d.Cout, bn) * kiters * (128 * 128 + bn * 128)
    for kind, tw, th in (('rows', 16, 8), ('rows256', 16, 16)):
        res[kind] = None
        if rows_eligible(d):
            mt = cdiv(d.Wg, tw) * cdiv(d.Hg, th) * d.B
            bn = 128 if d.Cout > 64 else 64
            per_tile = 0
            for s in range(d.nsrc):
                cs = d.s[s]
                ndx = len({cs.dx[t] for t in range(cs.ntaps)})
                per_tile += (cs.C // 32) * (ndx * tw * (th + 2) * 128 + cs.ntaps * bn * 128)
            res[kind] = mt * cdiv(d.Cout, bn) * per_tile
    hbm = 0
    for s in range(d.nsrc):
        cs = d.s[s]
        hbm += d.B * cs.H * cs.W * cs.C * 4 + cs.ntaps * d.Cout * cs.C * 4 * (d.B if cs.w_per_batch else 1)
    outs = 1 + sum(1 for p in (d.out2, d.resid, d.aux) if p)
    res['hbm'] = hbm + outs * d.B * d.Hg * d.Wg * d.Cout * 4
    return res


def shape_key(d):     # engine.profile_shapes
    return (d.B, d.Hg, d.Wg, d.Cout, sum(d.s[i].ntaps * d.s[i].C for i in range(d.nsrc)), d.nsrc, d.s[0].w_per_batch)


model = {}
_conv_fwd = ops.conv_fwd
phase = ['fwd']          # which pass the launches being recorded belong to: 'fwd' or 'dgrad'


def conv_fwd_recording(desc, impl=ops.CONV_TC):
    if impl == ops.CONV_TC:
        model.setdefault((phase[0],) + shape_key(desc), traffic(desc))
    return _conv_fwd(desc, impl)


ops.conv_fwd = conv_fwd_recording

with contextlib.redirect_stdout(io.StringIO()):
    u = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
x = torch.rand(B, 3, 128, 128, device='cuda') * 2 - 1
t = torch.randint(0, 200, (B,), device='cuda')
gy = torch.randn(B, 3, 128, 128, device='cuda')
res = {name: collections.OrderedDict() for name in CONFIGS}


def collect(name, tag):
    torch.cuda.synchronize()
    for (a, b, f), shp in zip(u.engine.profile_convs, u.engine.profile_shapes):
        e = res[name].setdefault((tag,) + shp, [0, 0.0, f])
        e[0] += 1; e[1] += a.elapsed_time(b)
    u.engine.profile_convs = u.engine.profile_shapes = None


for rep in range(-1, 5):          # the configurations take turns, so that clock drift over the run affects all alike
    for name, (cfg, _) in CONFIGS.items():
        apply(cfg)
        phase[0] = 'fwd'
        with torch.no_grad():
            u(x, t)                    # warm-up of this configuration's forward kernels
            if rep >= 0:
                u.engine.profile_convs, u.engine.profile_shapes = [], []
                u(x, t)
                collect(name, 'fwd')
        y = u(x, t)                    # training forward; the data gradients of its backward are recorded
        phase[0] = 'dgrad'
        if rep >= 0:
            u.engine.profile_convs, u.engine.profile_shapes = [], []
        y.backward(gy)
        if rep >= 0:
            collect(name, 'dgrad')
apply(DEFAULT)
ops.conv_fwd = _conv_fwd
try:
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=10).stdout.strip()
except Exception as e:  # noqa
    gpu = 'nvidia-smi unavailable: %r' % e
print('GPU: %s (%d SMs), batch %d' % (gpu, SMS, B))
names = list(CONFIGS)
print("%-46s %3s %8s %8s %8s %8s" % ("(pass,B,Hg,Wg,Cout,K,nsrc,per_batch)", "n", "L2tap_MB", "L2rowsMB", "L2r256MB", "HBM_MB")
      + ''.join(' | %-27s' % (n + ' us/TF/L2/HBM') for n in names))
tot = {n: 0.0 for n in names}
tot_pass = {(n, k): 0.0 for n in names for k in ('fwd', 'dgrad')}
for shp, (n, ms, f) in res[names[0]].items():
    n //= 5
    m = model.get(shp, {})
    mb = lambda v: ('%8.1f' % (v / 1e6)) if v else '%8s' % '-'
    row = "%-46s %3d %s %s %s %s" % (str(shp), n, mb(m.get('tap')), mb(m.get('rows')), mb(m.get('rows256')), mb(m.get('hbm')))
    for name in names:
        us = res[name][shp][1] / 5 / n * 1e3
        tot[name] += res[name][shp][1] / 5
        tot_pass[(name, shp[0])] += res[name][shp][1] / 5
        kind = CONFIGS[name][1]
        l2 = (m.get(kind) or m.get('tap')) if kind else None
        row += ' | %7.1f %4.0f %6.0f %5.0f' % (us, f / us / 1e6, l2 / us / 1e3 if l2 else 0, m.get('hbm', 0) / us / 1e3)
    print(row)
print("conv ms per forward + data gradients of one backward: " +
      '   '.join('%s %.3f (%.3f + %.3f)' % (m, tot[m], tot_pass[(m, 'fwd')], tot_pass[(m, 'dgrad')]) for m in names))
