"""How much of the 16 x 16 shared-row convolution's time its epilogue operands cost: for every launch of one Unet config 3 training
micro-batch (128^2, batch 32: forward and backward data gradients) that goes to conv_rows256_kernel and reads resid or a GELU'
aux, the launch as the engine issues it against the same GEMM with that operand dropped (no resid; act none instead of GELU',
no aux).  The two variants take turns, launch by launch, so that clock drift affects both alike.  The summed difference bounds
what hiding the operand loads can save.

Measured on an H100 80GB HBM3 at a 700 W power limit (SM clock 1965-1980 MHz), two runs: the 26 such launches of a micro-batch
take 8.95-8.97 ms as issued and 4.68-4.69 ms without their operands, so hiding the loads can save at most 4.27 ms per
micro-batch, 8.5 ms per step.  Most of it is in the GELU' data gradients at 64^2 and 128^2, whose launches take 2.5-3.6 times
as long with aux as without.  These were measured with the operands read from global memory in the epilogue.  With the operands
now staged in shared memory by TMA during the mainloop, the same launches take about 6.5 ms per micro-batch.

The timed launches run in the middle of the step and overwrite their outputs: only the times are meaningful.

    python tools/conv_epilogue_bound.py [batch [rounds [launches per round]]]     # default: 32 5 10"""
import sys, io, contextlib, os, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import cold_diffusion_models_b200 as cdm
from cold_diffusion_models_b200 import ops
from cold_diffusion_models_b200._lib import ConvDesc, CONV_TC, ACT_NONE, ACT_GELU_BWD

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
N = int(sys.argv[3]) if len(sys.argv) > 3 else 10
MICRO_BATCHES = 2                      # config 3: two micro-batches of 32 per optimizer step
SMS = torch.cuda.get_device_properties(0).multi_processor_count


def cdiv(a, b):
    return -(-a // b)


def goes_to_rows256(d):
    """conv_tc.cu, conv_fwd_rows in its default (shape-based) mode"""
    if d.sy != 1 or d.sx != 1:
        return False
    for s in range(d.nsrc):
        cs = d.s[s]
        if cs.w_per_batch or cs.C % 32 or cs.W != d.Wg or cs.H != d.Hg:
            return False
        if any(not (-1 <= cs.dy[t] <= 1 and -1 <= cs.dx[t] <= 1) for t in range(cs.ntaps)):
            return False
    if d.s[0].ntaps < 3 * len({d.s[0].dx[t] for t in range(d.s[0].ntaps)}):
        return False
    bn = 128 if d.Cout > 64 else 64
    tiles = cdiv(d.Wg, 16) * cdiv(d.Hg, 8) * d.B * cdiv(d.Cout, bn)
    tiles256 = cdiv(d.Wg, 16) * cdiv(d.Hg, 16) * d.B * cdiv(d.Cout, bn)
    return (tiles > SMS and 4 * tiles256 >= 3 * SMS and (d.oys, d.oxs, d.oy0, d.ox0) == (1, 1, 0, 0) and d.Ho == d.Hg
            and d.Wo == d.Wg)


def dropped(d):
    e = ConvDesc.from_buffer_copy(d)
    e.resid, e.resid_ld = None, 0
    if e.act == ACT_GELU_BWD:
        e.act, e.aux, e.aux_ld = ACT_NONE, None, 0
    return e


def ms_per_launch(d):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(N):
        _conv_fwd(d, CONV_TC)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / N


rows = []                # (pass, shape, operand, engine us, dropped us)
other_rows256 = [0]      # rows256 launches without resid / aux (nothing to drop)
timing = [False]
phase = ['fwd']
_conv_fwd = ops.conv_fwd


def conv_fwd_timed(d, impl=CONV_TC):
    if timing[0] and impl == CONV_TC and goes_to_rows256(d):
        if d.resid or d.act == ACT_GELU_BWD:
            dd = dropped(d)
            ms_per_launch(d); ms_per_launch(dd)                        # warm-up of both
            t = {'engine': [], 'dropped': []}
            for _ in range(ROUNDS):
                t['engine'].append(ms_per_launch(d))
                t['dropped'].append(ms_per_launch(dd))
            med = lambda v: sorted(v)[len(v) // 2] * 1e3
            k = sum(d.s[i].ntaps * d.s[i].C for i in range(d.nsrc))
            rows.append((phase[0], (d.Hg, d.Wg, k, d.Cout), 'resid' if d.resid else 'aux', med(t['engine']), med(t['dropped'])))
        else:
            other_rows256[0] += 1
    return _conv_fwd(d, impl)


ops.conv_fwd = conv_fwd_timed
with contextlib.redirect_stdout(io.StringIO()):
    u = cdm.Unet(dim=64, dim_mults=(1, 2, 4, 8), channels=3).cuda()
x = torch.rand(B, 3, 128, 128, device='cuda') * 2 - 1
t = torch.randint(0, 200, (B,), device='cuda')
gy = torch.randn(B, 3, 128, 128, device='cuda')
for timed in (False, True):              # the first micro-batch warms every kernel up
    timing[0] = timed
    phase[0] = 'fwd'
    y = u(x, t)
    phase[0] = 'dgrad'
    y.backward(gy)
    torch.cuda.synchronize()
ops.conv_fwd = _conv_fwd

try:
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=10).stdout.strip()
except Exception as e:  # noqa
    gpu = 'nvidia-smi unavailable: %r' % e
print('GPU: %s (%d SMs), batch %d, median of %d rounds of %d launches' % (gpu, SMS, B, ROUNDS, N))
print('%-6s %-24s %-6s %10s %10s %9s' % ('pass', '(Hg, Wg, K, Cout)', 'opnd', 'engine_us', 'dropped_us', 'diff_us'))
te = td = 0.0
for ph, shp, op, ue, ud in rows:
    te += ue; td += ud
    print('%-6s %-24s %-6s %10.1f %10.1f %9.1f' % (ph, str(shp), op, ue, ud, ue - ud))
print('%d launches with an operand: %.3f ms as issued, %.3f ms without the operand, difference %.3f ms per micro-batch, '
      '%.3f ms per step of %d micro-batches (%d rows256 launches without an operand not timed)'
      % (len(rows), te / 1e3, td / 1e3, (te - td) / 1e3, MICRO_BATCHES * (te - td) / 1e3, MICRO_BATCHES, other_rows256[0]))
