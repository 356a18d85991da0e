"""Thin Python wrappers over the C ABI (include/colddiff.h): descriptor builders for the tap-list
convolution contract and one function per entry point.  No arithmetic happens here -- torch is
used for device memory and streams only."""
import ctypes as C
import torch

from . import _lib
from ._lib import lib, ptr, stream, call, ConvDesc, ConvSrc, CONV_SIMT, CONV_TC, ACT_NONE, ACT_GELU, ACT_GELU_BWD


# --------------------------------------------------------------------------------------------
# tap lists
# --------------------------------------------------------------------------------------------
def taps_conv(k, pad):
    """forward taps of nn.Conv2d(k, padding=pad): (ky, kx, dy, dx)"""
    return [(ky, kx, ky - pad, kx - pad) for ky in range(k) for kx in range(k)]


def taps_conv_dgrad(k, pad):
    """data-gradient of a stride-1 conv: a conv of dY with the flipped kernel"""
    return [(ky, kx, pad - ky, pad - kx) for ky in range(k) for kx in range(k)]


def taps_convT4_parity(py, px):
    """nn.ConvTranspose2d(4, stride 2, padding 1) (and the dgrad of Conv2d(4, 2, 1)) for the output
    parity class (Y % 2, X % 2) == (py, px): out[2g+p] = sum_k in[g + d] * W[k]"""
    ys = [(1, 0), (3, -1)] if py == 0 else [(0, 1), (2, 0)]
    xs = [(1, 0), (3, -1)] if px == 0 else [(0, 1), (2, 0)]
    return [(ky, kx, dy, dx) for (ky, dy) in ys for (kx, dx) in xs]


def pack_weight(w, taps, mode=0, transposed_conv=False, round_tf32=True, out=None):
    """reference-layout conv weight (O,I,KH,KW) [or ConvTranspose2d (I,O,KH,KW)] -> packed
    [tap][N][K] fp32 (mode 0: N=out ch, K=in ch; mode 1 (data-gradient operand): N=in, K=out)."""
    if transposed_conv:
        I, O, KH, KW = w.shape
    else:
        O, I, KH, KW = w.shape
    n, k = (O, I) if mode == 0 else (I, O)
    nt = len(taps)
    if out is None:
        out = torch.empty((nt, n, k), device=w.device, dtype=torch.float32)
    ky = (C.c_int32 * nt)(*[t[0] for t in taps])
    kx = (C.c_int32 * nt)(*[t[1] for t in taps])
    call('cd_pack_weight', ptr(w), O, I, KH, KW, int(transposed_conv), mode, ky, kx, nt, int(round_tf32),
         ptr(out), stream())
    return out


def unpack_wgrad(packed, taps, w_grad, transposed_conv=False, accumulate=True):
    if transposed_conv:
        I, O, KH, KW = w_grad.shape
    else:
        O, I, KH, KW = w_grad.shape
    nt = len(taps)
    ky = (C.c_int32 * nt)(*[t[0] for t in taps])
    kx = (C.c_int32 * nt)(*[t[1] for t in taps])
    call('cd_unpack_wgrad', ptr(packed), O, I, KH, KW, int(transposed_conv), ky, kx, nt, ptr(w_grad),
         int(accumulate), stream())


class RepackBatch:
    """all weight repacks (kind 'pack') or all packed-gradient unpacks (kind 'unpack') of one pass in ONE launch
    (cd_pack_weight_batched / cd_unpack_wgrad_batched).  add() has the argument meaning of pack_weight() / unpack_wgrad();
    run() uploads the job table when the set of (source, destination) buffers changed (they are persistent buffers, so
    normally once) and launches.  The block split mirrors the single-weight entry points: one block per 256 (o, i) rows
    for Conv2d weights with KH*KW <= 16, an element-strided range otherwise."""

    MAX_STRIDED_BLOCKS = None       # cap on the blocks of an element-strided job; None: two per SM, as the single-weight entry points

    def __init__(self, kind):
        assert kind in ('pack', 'unpack')
        self.kind = kind
        self._jobs = []
        self._key = None
        self._table = None
        self._total = 0

    def __len__(self):
        return len(self._jobs)

    def add(self, src, taps, dst, *, shape, mode=0, transposed_conv=False, round_tf32=False):
        """shape = the reference-layout weight shape ((O,I,KH,KW), or (I,O,KH,KW) for nn.ConvTranspose2d)"""
        if transposed_conv:
            I, O, KH, KW = shape
        else:
            O, I, KH, KW = shape
        assert 1 <= len(taps) <= _lib.CD_MAX_TAPS
        self._jobs.append((src, dst, O, I, KH, KW, int(transposed_conv), int(mode), tuple((t[0], t[1]) for t in taps), int(round_tf32)))

    def clear(self):
        self._jobs = []

    def _build(self, device):
        n = len(self._jobs)
        arr = (_lib.RepackJob * n)()
        b0 = 0
        for j, (src, dst, O, I, KH, KW, tr, mode, taps, rnd) in enumerate(self._jobs):
            r = arr[j]
            r.src, r.dst = src.data_ptr(), dst.data_ptr()
            r.O, r.I, r.KH, r.KW, r.transposed_conv, r.mode, r.ntaps, r.round_tf32 = O, I, KH, KW, tr, mode, len(taps), rnd
            for t, (ky, kx) in enumerate(taps):
                r.ky[t], r.kx[t] = ky, kx
            tiled = (not tr) and KH * KW <= 16 and (self.kind == 'unpack' or mode == 0)
            if tiled:
                nb = (O * I + 255) // 256
            else:
                nb = min((len(taps) * O * I + 1023) // 1024, self.MAX_STRIDED_BLOCKS or 2 * sm_count(dst.device))
            r.block0, r.nblocks = b0, max(nb, 1)
            b0 += r.nblocks
        raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
        self._table = raw.to(device)
        self._total = b0

    def run(self, *, accumulate=True, clear_src=False):
        if not self._jobs:
            return
        key = tuple((j[0].data_ptr(), j[1].data_ptr()) + j[2:] for j in self._jobs)
        if key != self._key:
            self._build(self._jobs[0][0].device)
            self._key = key
        if self.kind == 'pack':
            call('cd_pack_weight_batched', ptr(self._table), len(self._jobs), self._total, stream())
        else:
            call('cd_unpack_wgrad_batched', ptr(self._table), len(self._jobs), self._total, int(accumulate), int(clear_src), stream())


class TapTransposeBatch:
    """data-gradient operands of many dense convolutions in ONE launch (cd_transpose_taps_batched), from forward operands that
    are already packed [KH*KW][O][I] -- the engine's master layout of dense conv weights.  add(src, O, I, KW, taps, dst):
    dst[t][i][o] = src[ky_t * KW + kx_t][o][i].  The job table is built once (all buffers are persistent)."""

    def __init__(self):
        self._jobs, self._key, self._table, self._total = [], None, None, 0

    def __len__(self):
        return len(self._jobs)

    def clear(self):
        self._jobs = []

    def add(self, src, O, I, KW, taps, dst):
        assert 1 <= len(taps) <= _lib.CD_MAX_TAPS and dst.numel() == len(taps) * O * I
        self._jobs.append((src, dst, int(O), int(I), int(KW), tuple((t[0], t[1]) for t in taps)))

    def run(self):
        if not self._jobs:
            return
        key = tuple((j[0].data_ptr(), j[1].data_ptr()) + j[2:] for j in self._jobs)
        if key != self._key:
            arr = (_lib.RepackJob * len(self._jobs))()
            b0 = 0
            for j, (src, dst, O, I, KW, taps) in enumerate(self._jobs):
                r = arr[j]
                r.src, r.dst, r.O, r.I, r.KH, r.KW, r.ntaps = src.data_ptr(), dst.data_ptr(), O, I, 1, KW, len(taps)
                for t, (ky, kx) in enumerate(taps):
                    r.ky[t], r.kx[t] = ky, kx
                r.block0, r.nblocks = b0, len(taps) * ((O + 31) // 32) * ((I + 31) // 32)
                b0 += r.nblocks
            self._table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(self._jobs[0][0].device)
            self._total, self._key = b0, key
        call('cd_transpose_taps_batched', ptr(self._table), len(self._jobs), self._total, stream())


# --------------------------------------------------------------------------------------------
# NHWC views: (tensor, channel offset, channels).  tensor is [B, H, W, ld] contiguous.
# --------------------------------------------------------------------------------------------
class View:
    __slots__ = ('t', 'c0', 'C')

    def __init__(self, t, c0=0, C=None):
        self.t, self.c0 = t, c0
        self.C = (t.shape[-1] - c0) if C is None else C

    @property
    def ld(self):
        return self.t.shape[-1]

    @property
    def B(self):
        return self.t.shape[0]

    @property
    def H(self):
        return self.t.shape[1]

    @property
    def W(self):
        return self.t.shape[2]

    def addr(self):
        return self.t.data_ptr() + 4 * self.c0


def make_conv_desc(srcs, out, grid, *, stride=1, Cout, bias=None, resid=None, act=ACT_NONE,
                   round_tf32=False, out_map=(1, 1, 0, 0), out2=None, aux=None):
    """srcs: list of (View, taps[(ky,kx,dy,dx)], packed_w, w_per_batch); out/resid/out2: View;
    grid: (B, Hg, Wg)."""
    d = ConvDesc()
    d.B, d.Hg, d.Wg = grid
    d.sy = d.sx = stride
    d.Cout = Cout
    d.nsrc = len(srcs)
    keep = []
    for i, (v, taps, w, wpb) in enumerate(srcs):
        s = d.s[i]
        s.src = v.addr(); s.ld = v.ld; s.C = v.C; s.H = v.H; s.W = v.W
        s.ntaps = len(taps)
        for j, tp in enumerate(taps):
            s.dy[j] = tp[2]; s.dx[j] = tp[3]
        s.w = w.data_ptr(); s.w_per_batch = int(wpb)
        keep.append(w)
    d.out = out.addr(); d.out_ld = out.ld; d.Ho = out.H; d.Wo = out.W
    d.oys, d.oxs, d.oy0, d.ox0 = out_map
    d.bias = bias.data_ptr() if bias is not None else None
    if resid is not None:
        d.resid = resid.addr(); d.resid_ld = resid.ld
    d.act = act
    d.round_tf32 = int(round_tf32)
    if out2 is not None:
        d.out2 = out2.addr(); d.out2_ld = out2.ld
    if aux is not None:
        d.aux = aux.addr(); d.aux_ld = aux.ld
    d._keep = keep
    return d


def conv_fwd(desc, impl=CONV_TC):
    call('cd_conv_fwd', C.byref(desc), impl, stream())


def conv_wgrad(desc, dout, dw_packed, db=None, impl=CONV_SIMT):
    call('cd_conv_wgrad', C.byref(desc), C.c_void_p(dout.addr()), dout.ld, ptr(dw_packed), ptr(db), impl, stream())


_SM_COUNT = {}


def sm_count(device=None):
    """SM count of a CUDA device (132, the H100 SXM's, for CPU tensors and when there is no device): sizes the launch splits
    that the host computes, like cd_num_sms() in the library"""
    key = str(device)
    sms = _SM_COUNT.get(key)
    if sms is None:
        sms = 132
        if device is not None and torch.device(device).type == 'cuda' and torch.cuda.is_available():
            sms = torch.cuda.get_device_properties(device).multi_processor_count
        _SM_COUNT[key] = sms
    return sms


def linattn_ctx_plan(B, n, device=None):
    """how cd_linattn_context_det cuts the pixel axis of one image: -> (nblk, ppb) with ppb a multiple of 32 and
    nblk = ceil(n / ppb) partials per image; about one wave of resident blocks (3 per SM) over the whole batch"""
    sms = sm_count(device)
    per_img = max(1, (3 * sms) // max(B, 1))
    ppb = max(64, -(-(-(-n // per_img)) // 32) * 32)
    return -(-n // ppb), ppb
