"""Operand-format probe (FP16 operands instead of TF32): the tensor-core tap-list convolution on FP16 sources and
FP16 packed weights (cd_conv_fwd_f16_probe: wgmma on FP16, fp32 accumulate, fp32 epilogue) next to today's TF32 kernel on the SAME
values, for the convolution shapes of the config-3 network.  Inputs are rounded to FP16 first, which is also exactly representable
in TF32 (both have a 10-bit mantissa), so the two kernels multiply identical numbers: outputs must agree to fp32 summation order.
Prints per shape: TF32 us, FP16 us, TFLOP/s of both, max relative difference.
Usage: python tools/conv_f16_probe.py [batch]      (check only: python tools/conv_f16_probe.py --check)"""
import ctypes as C
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from cold_diffusion_models_b200 import ops
from cold_diffusion_models_b200._lib import lib, _check, stream

# (H, Cin, Cout, k) of the stride-1 convolutions of Unet(dim 64, mults (1,2,4,8)) with Cin % 64 == 0
SHAPES = [(128, 128, 64, 3), (128, 64, 128, 3), (128, 64, 384, 1), (64, 128, 256, 3), (64, 256, 128, 3), (64, 128, 384, 1),
          (64, 64, 64, 3), (32, 256, 512, 3), (32, 512, 256, 3), (32, 256, 384, 1), (16, 512, 1024, 3), (16, 1024, 512, 3),
          (16, 256, 256, 3)]


def run(B, H, Ci, Co, k, reps=5):
    g = torch.Generator().manual_seed(H + Ci + Co)
    x = torch.randn(B, H, H, Ci, generator=g).half().cuda()
    w = (torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5).half().cuda()
    bias = torch.randn(Co, generator=g).cuda()
    taps = ops.taps_conv(k, k // 2)
    wp16 = w.permute(2, 3, 0, 1).reshape(k * k, Co, Ci).contiguous()             # packed [tap][Cout][Cin], FP16
    x32, wp32 = x.float().contiguous(), wp16.float().contiguous()
    out32, out16 = torch.empty(B, H, H, Co, device='cuda'), torch.empty(B, H, H, Co, device='cuda')
    d32 = ops.make_conv_desc([(ops.View(x32), taps, wp32, False)], ops.View(out32), (B, H, H), Cout=Co, bias=bias, act=ops.ACT_GELU)
    d16 = ops.make_conv_desc([(ops.View(x), taps, wp16, False)], ops.View(out16), (B, H, H), Cout=Co, bias=bias, act=ops.ACT_GELU)
    t = []
    for fn in (lambda: ops.conv_fwd(d32, ops.CONV_TC), lambda: _check(lib.cd_conv_fwd_f16_probe(C.byref(d16), stream()), 'cd_conv_fwd_f16_probe')):
        fn(); fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1) / reps * 1e3)
    err = ((out16.double() - out32.double()).norm() / out32.double().norm()).item()
    flops = 2.0 * B * H * H * Co * Ci * k * k
    return t[0], t[1], flops, err


if __name__ == '__main__':
    if '--check' in sys.argv:
        for shp in ((32, 64, 128, 3), (16, 128, 64, 1), (16, 256, 256, 3)):
            t32, t16, fl, err = run(4, *shp, reps=1)
            assert err < 1e-5, (shp, err)
        print('F16_PROBE_OK')
        sys.exit(0)
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    print("%-28s %9s %9s %9s %9s %10s" % ("(H, Cin, Cout, k)", "tf32 us", "f16 us", "TF/s tf32", "TF/s f16", "rel diff"))
    for shp in SHAPES:
        t32, t16, fl, err = run(B, *shp)
        print("%-28s %9.1f %9.1f %9.1f %9.1f %10.2e" % (str(shp), t32, t16, fl / t32 / 1e6, fl / t16 / 1e6, err))
