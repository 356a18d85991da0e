"""ctypes binding of libcolddiff.so (the C ABI in include/colddiff.h).

The product path has NO fallback: if the shared library (built in-tree by
__graft_entry__.build() / `make -C cold_diffusion_models_b200/csrc`) is missing, importing
this module raises.  All pointers passed down are raw device pointers of torch tensors; the
stream is torch's current CUDA stream.
"""
import ctypes as C
import os
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'csrc', 'libcolddiff.so')
CD_MAX_TAPS = 16
CONV_SIMT, CONV_TC = 0, 1
ACT_NONE, ACT_GELU, ACT_GELU_BWD = 0, 1, 2


class ColdDiffError(RuntimeError):
    pass


if not os.path.exists(LIB_PATH):
    raise ImportError("libcolddiff.so not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'`"
                      % LIB_PATH)
lib = C.CDLL(LIB_PATH)


class ConvSrc(C.Structure):
    _fields_ = [('src', C.c_void_p), ('ld', C.c_int32), ('C', C.c_int32), ('H', C.c_int32), ('W', C.c_int32),
                ('ntaps', C.c_int32), ('dy', C.c_int32 * CD_MAX_TAPS), ('dx', C.c_int32 * CD_MAX_TAPS),
                ('w', C.c_void_p), ('w_per_batch', C.c_int32)]


class ConvDesc(C.Structure):
    _fields_ = [('B', C.c_int32), ('Hg', C.c_int32), ('Wg', C.c_int32), ('sy', C.c_int32), ('sx', C.c_int32),
                ('Cout', C.c_int32), ('nsrc', C.c_int32), ('s', ConvSrc * 2),
                ('out', C.c_void_p), ('out_ld', C.c_int32), ('Ho', C.c_int32), ('Wo', C.c_int32),
                ('oys', C.c_int32), ('oxs', C.c_int32), ('oy0', C.c_int32), ('ox0', C.c_int32),
                ('bias', C.c_void_p), ('resid', C.c_void_p), ('resid_ld', C.c_int32),
                ('act', C.c_int32), ('round_tf32', C.c_int32),
                ('out2', C.c_void_p), ('out2_ld', C.c_int32),
                ('aux', C.c_void_p), ('aux_ld', C.c_int32)]




class RepackJob(C.Structure):          # CdRepackJob (include/colddiff.h): one row of the device-resident table of the batched repacks
    _fields_ = [('src', C.c_void_p), ('dst', C.c_void_p), ('O', C.c_int32), ('I', C.c_int32), ('KH', C.c_int32), ('KW', C.c_int32),
                ('transposed_conv', C.c_int32), ('mode', C.c_int32), ('ntaps', C.c_int32), ('round_tf32', C.c_int32),
                ('ky', C.c_int32 * CD_MAX_TAPS), ('kx', C.c_int32 * CD_MAX_TAPS), ('block0', C.c_int32), ('nblocks', C.c_int32)]


lib.cd_version.restype = C.c_int
if os.environ.get('COLDDIFF_2CTA') in ('0', '1', '2'):   # SM-pair (two-CTA cluster) convolution kernel; library default 0
    lib.cd_conv_tc_set_2cta(int(os.environ['COLDDIFF_2CTA']))
lib.cd_last_error.argtypes = [C.c_char_p, C.c_size_t]
if os.environ.get('COLDDIFF_CONV_TWO_CTAS') in ('0', '64', '128', '192'):   # two CTAs per SM for the N <= 128 convolution tiles (bit mask)
    lib.cd_conv_tc_set_two_ctas(int(os.environ['COLDDIFF_CONV_TWO_CTAS']))
if os.environ.get('COLDDIFF_CONV_HALO') in ('0', '1', '2', '6', '8'):   # 3x3 convolution kernel: 0 shape-based (default), 1 / 2 / 6 shared-row kernel, 8 per-tap kernel
    lib.cd_conv_tc_set_halo(int(os.environ['COLDDIFF_CONV_HALO']))
if os.environ.get('COLDDIFF_WGRAD_MODE') in ('0', '1', '8'):   # tensor-core weight gradient: 1 wgmma kernel where eligible (default), 8 mma.sync halo kernel, 0 mma.sync one X tile per tap
    lib.cd_wgrad_tc_set_mode(int(os.environ['COLDDIFF_WGRAD_MODE']))
if os.environ.get('COLDDIFF_2CTA_BN') in ('0', '64', '128', '192'):   # N tiles below 256 on the SM-pair kernel (bit mask 128 | 64)
    lib.cd_conv_tc_set_2cta_bn(int(os.environ['COLDDIFF_2CTA_BN']))
if os.environ.get('COLDDIFF_CONV_STAGED_EPILOGUE') in ('0', '1', '2', '3'):   # line-coalesced conv epilogue (csrc/conv_epilogue.cuh); default 0
    lib.cd_conv_tc_set_staged_epilogue(int(os.environ['COLDDIFF_CONV_STAGED_EPILOGUE']))


def _check(rc, what):
    if rc != 0:
        buf = C.create_string_buffer(512)
        lib.cd_last_error(buf, 512)
        raise ColdDiffError("%s failed (%d): %s" % (what, rc, buf.value.decode()))


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    if t is None:
        return C.c_void_p(0)
    return C.c_void_p(t.data_ptr())


_LAUNCHES = {'cd_linattn_context_det': 2, 'cd_conv_wgrad': 2, 'cd_time_mlp_fwd': 2, 'cd_time_mlp2_fwd': 2, 'cd_version': 0, 'cd_last_error': 0}
_launch_count = 0


_PROF_SHAPE_ARGS = {'cd_dwconv7_fwd': (2, 3, 4, 5), 'cd_dwconv7_wgrad': (4, 5, 6, 7), 'cd_layernorm_bwd': (6, 7),
                    'cd_layernorm_fwd': (2, 3), 'cd_linattn_context_det': (2, 3), 'cd_linattn_bwd_kv': (2, 3)}
_prof = None          # tools/op_profile.py: list of (name, event0, event1) while profiling, else None


def call(name, *args):
    global _launch_count
    _launch_count += _LAUNCHES.get(name, 1)
    if _prof is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _check(getattr(lib, name)(*args), name)
        e1.record()
        idx = _PROF_SHAPE_ARGS.get(name)
        if idx:                  # per-shape rows for the HBM-bound kernels: (B, H, W, C) / (npix, C) / (B, n)
            name = name + str(tuple(int(getattr(args[i], 'value', args[i])) for i in idx))
        _prof.append((name, e0, e1))
        return
    _check(getattr(lib, name)(*args), name)


def profile_start():
    """time every C-ABI call with CUDA events on the current stream (in-situ, warm caches) until profile_stop()"""
    global _prof
    _prof = []


def profile_stop():
    """-> {name: (calls, total_ms)}"""
    global _prof
    torch.cuda.synchronize()
    out = {}
    for name, e0, e1 in _prof:
        c, t = out.get(name, (0, 0.0))
        out[name] = (c + 1, t + e0.elapsed_time(e1))
    _prof = None
    return out


def reset_launch_count():
    global _launch_count
    _launch_count = 0


def launch_count():
    """kernels launched through the C ABI since the last reset (each entry point launches >= 1 kernel)"""
    return _launch_count


EXPORTS = [
    'cd_version', 'cd_last_error', 'cd_conv_fwd', 'cd_conv_wgrad', 'cd_pack_weight', 'cd_unpack_wgrad',
]
