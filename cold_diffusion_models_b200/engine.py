"""UnetEngine -- host-side schedule of the sm_90a kernels that execute the reference `Unet.forward`
(DB:256-282) on NHWC fp32 activations.  Python here only sequences C-ABI calls (include/colddiff.h) on
torch's current stream and owns device buffers; it performs no arithmetic.

Data layout in HBM
  * activations: NHWC fp32, one buffer per tensor; skip connections are never copied -- the down-path
    attention writes its output straight into the second channel half of the up-path concat buffer and
    the Upsample transpose-conv writes into the first half (replaces torch.cat, DB:274);
  * dense conv weights: packed [tap][Cout][Cin] fp32 (K-major rows for TMA/UMMA), repacked from the
    reference OIHW parameters whenever they change; TF32 rounding happens in the TMA unit on load;
  * time conditioning of all 16 blocks is one [B][sumC] matrix produced by a single kernel.
"""
import ctypes as C
import torch

from . import ops
from .ops import View, CONV_TC, CONV_SIMT, ACT_NONE, ACT_GELU
from ._lib import call, ptr, stream
from .graphs import GraphedForward

T3 = ops.taps_conv(3, 1)
T1 = ops.taps_conv(1, 0)
T4 = ops.taps_conv(4, 1)
T3D = ops.taps_conv_dgrad(3, 1)
TPAR = {(py, px): ops.taps_convT4_parity(py, px) for py in (0, 1) for px in (0, 1)}


_BATCHED_REPACK = None


def batched_repack(enable=None):
    """switch of the one-launch weight repacks (ops.RepackBatch: cd_pack_weight_batched / cd_unpack_wgrad_batched).  Default
    from COLDDIFF_BATCHED_REPACK (off by default)."""
    global _BATCHED_REPACK
    if enable is not None:
        _BATCHED_REPACK = bool(enable)
    if _BATCHED_REPACK is None:
        import os
        _BATCHED_REPACK = os.environ.get('COLDDIFF_BATCHED_REPACK', '0') == '1'
    return _BATCHED_REPACK


def _tc_ok(*chans):
    return all(c % 32 == 0 for c in chans)


class _BackwardHolder:
    """placeholder base; engine_bwd.BackwardMixin's methods are grafted on at import time (avoids a cycle)"""


class BlockSpec:
    """one ConvNextBlock (DB:135-165)"""

    def __init__(self, name, mod, cond_off):
        self.name = name
        self.mod = mod
        self.din = mod.ds_conv.weight.shape[0]
        self.dmid = mod.net[1].weight.shape[0]
        self.dout = mod.net[3].weight.shape[0]
        self.has_norm = hasattr(mod.net[0], 'g')
        self.has_res = hasattr(mod.res_conv, 'weight')
        self.cond_off = cond_off if mod.mlp is not None else None


class AttnSpec:
    """Residual(PreNorm(LinearAttention)) (DB:83-89,123-131,167-187)"""

    def __init__(self, name, mod):
        self.name = name
        self.norm = mod.fn.norm
        self.attn = mod.fn.fn
        self.dim = self.norm.g.shape[1]


class UnetEngine(_BackwardHolder, GraphedForward):
    def __init__(self, unet):
        self.unet = unet
        self.dev = next(unet.parameters()).device
        self.channels = unet.channels
        self.dim = unet.dim
        self._bufs = {}
        self._packed = {}
        self._batches = {}
        self._dirty = True
        self._version = None
        self.conv_impl = CONV_TC
        # ---- static program ----
        off = 0
        self.blocks = {}

        def mk(name, mod):
            nonlocal off
            bs = BlockSpec(name, mod, off)
            if mod.mlp is not None:
                off += (bs.din + 3) // 4 * 4          # keep every block's slice 16-byte aligned
            self.blocks[name] = bs
            return bs

        self.levels_down = []
        for i, (b0, b1, at, dn) in enumerate(unet.downs):
            self.levels_down.append((mk('downs.%d.0' % i, b0), mk('downs.%d.1' % i, b1),
                                     AttnSpec('downs.%d.2' % i, at), dn if hasattr(dn, 'weight') else None))
        self.mid1 = mk('mid_block1', unet.mid_block1)
        self.mid_attn = AttnSpec('mid_attn', unet.mid_attn)
        self.mid2 = mk('mid_block2', unet.mid_block2)
        self.levels_up = []
        for i, (b0, b1, at, up) in enumerate(unet.ups):
            self.levels_up.append((mk('ups.%d.0' % i, b0), mk('ups.%d.1' % i, b1),
                                   AttnSpec('ups.%d.2' % i, at), up if hasattr(up, 'weight') else None))
        self.final_block = mk('final_conv.0', unet.final_conv[0])
        self.final_proj = unet.final_conv[1]
        self.sumC = off
        self.cond_blocks = [b for b in self.blocks.values() if b.cond_off is not None]
        # dense nn.Conv2d weights (3x3 of the blocks, 4x4 stride-2 Downsample, every 1x1): their master copy can live PACKED
        # [KH*KW][O][I] -- the forward operand of the tap-list convolution and the layout the tensor-core weight gradient writes --
        # with the nn.Parameter a permuted (O, I, KH, KW) view of it (flatten_params / _setup_grads in engine_bwd.py)
        self.dense_convs = {}
        for mn, mod in unet.named_modules():
            if isinstance(mod, torch.nn.Conv2d) and not isinstance(mod, torch.nn.ConvTranspose2d) and mod.groups == 1:
                self.dense_convs[mn + '.weight'] = tuple(mod.weight.shape)
        self._pname = {id(p): n for n, p in unet.named_parameters()}
        self._init_graphs(unet, self.forward, self.prepare_weights)        # CUDA-graph replay (enable_cuda_graph)

    # ------------------------------------------------------------------------------------------
    _epoch = 0            # bumped by every in-place parameter update that bypasses torch's version counters

    def mark_weights_dirty(self):
        """the parameters changed behind torch's back (fused Adam / EMA kernels write the flat buffer through raw pointers, so
        `p._version` stays put): every packed operand -- forward, data-gradient and graph-captured -- is stale."""
        self._dirty = True
        self._epoch += 1

    def _weights_key(self):
        return (self._epoch, self._params_version())

    def param_list(self):
        return [p for p in self.unet.parameters()]

    def buf(self, name, shape, zero=False):
        key = (name, tuple(shape))
        t = self._bufs.get(key)
        if t is None:
            t = (torch.zeros if zero else torch.empty)(shape, device=self.dev, dtype=torch.float32)
            self._bufs[key] = t
        return t

    def _params_version(self, params=None):
        return tuple(p._version for p in (self.unet.parameters() if params is None else params))

    @staticmethod
    def packed_view(w):
        """(KH*KW, O, I) view of a dense conv weight whose storage is the packed master layout (a permuted view created by
        flatten_params), or of any 1x1 weight (packed == OIHW); None for a contiguous OIHW weight with KH*KW > 1"""
        O, I, KH, KW = w.shape
        if KH * KW == 1 and w.is_contiguous():
            return w.detach().view(1, O, I)
        if w.stride() == (I, 1, KW * O * I, O * I):
            return torch.as_strided(w.detach(), (KH * KW, O, I), (O * I, I, 1))
        return None

    def _pack_padded(self, key, w):
        """[KH*KW][O][pad32(I)] copy of a dense conv weight with the extra input channels zero (a data-movement copy)"""
        O, I, KH, KW = w.shape
        out = self._packed.get(key)
        if out is None:
            out = self._packed[key] = torch.zeros((KH * KW, O, self._pad32(I)), device=w.device, dtype=torch.float32)
        out[:, :, :I].copy_(w.detach().permute(2, 3, 0, 1).reshape(KH * KW, O, I))

    def _pack_fwd(self, batch, key, w, taps):
        """forward operand of a dense Conv2d: the weight itself when it is stored packed (no launch), else a repack"""
        pv = self.packed_view(w)
        if pv is not None and len(taps) == pv.shape[0]:
            self._packed[key] = pv
            return
        if self._packed.get(key) is not None and self._packed[key].data_ptr() == w.data_ptr():
            self._packed[key] = None               # was an alias of a weight that has since been re-laid out
        self._pack(batch, key, w, taps)

    def _pack(self, batch, key, w, taps, mode=0, transposed_conv=False):
        """packed operand P[key] of weight `w`: launched at once, or queued on `batch` (ops.RepackBatch) when batching is on"""
        P = self._packed
        if batch is None:
            P[key] = ops.pack_weight(w, taps, mode=mode, transposed_conv=transposed_conv, round_tf32=False, out=P.get(key))
            return
        out = P.get(key)
        if out is None:
            if transposed_conv:
                I, O = w.shape[0], w.shape[1]
            else:
                O, I = w.shape[0], w.shape[1]
            n, k = (O, I) if mode == 0 else (I, O)
            out = P[key] = torch.empty((len(taps), n, k), device=w.device, dtype=torch.float32)
        batch.add(w, taps, out, shape=tuple(w.shape), mode=mode, transposed_conv=transposed_conv, round_tf32=False)

    def _repack_batch(self, name, kind):
        """the persistent ops.RepackBatch `name` (emptied), or None when COLDDIFF_BATCHED_REPACK is off"""
        if not batched_repack():
            return None
        b = self._batches.get(name)
        if b is None:
            b = self._batches[name] = ops.RepackBatch(kind)
        b.clear()
        return b

    def prepare_weights(self, params=None):
        """(re)pack reference-layout parameters into kernel layouts when they changed; `params`: the parameter list, when the
        caller has it cached"""
        ver = self._params_version(params)
        if not (self._dirty or ver != self._version):
            return
        P = self._packed
        batch = self._repack_batch('pack_fwd', 'pack')
        with torch.no_grad():
            for name, bs in self.blocks.items():
                m = bs.mod
                self._pack_fwd(batch, name + '.w1', m.net[1].weight, T3)
                self._pack_fwd(batch, name + '.w2', m.net[3].weight, T3)
                if bs.has_res:
                    self._pack_fwd(batch, name + '.wr', m.res_conv.weight, T1)
                    # bias of the fused [conv2 | res_conv] GEMM
                    b = P.get(name + '.b2r')
                    if b is None:
                        b = P[name + '.b2r'] = torch.empty_like(m.net[3].bias)
                    torch.add(m.net[3].bias, m.res_conv.bias, out=b)
                if bs.din % 32 != 0:          # image-edge block: forward operands with K zero-padded to 32 channels
                    self._pack_padded(name + '.w1p', m.net[1].weight)
                    if bs.has_res:
                        self._pack_padded(name + '.wrp', m.res_conv.weight)
            for spec in self._attn_specs():
                a = spec.attn
                self._pack_fwd(batch, spec.name + '.wqkv', a.to_qkv.weight, T1)
            for i, lv in enumerate(self.levels_down):
                if lv[3] is not None:
                    self._pack_fwd(batch, 'downs.%d.3' % i, lv[3].weight, T4)
            for i, lv in enumerate(self.levels_up):
                if lv[3] is not None:
                    for k, tp in TPAR.items():
                        key = 'ups.%d.3.%d%d' % (i, k[0], k[1])
                        self._pack(batch, key, lv[3].weight, tp, transposed_conv=True)
            if self.cond_blocks:
                wc = P.get('cond.w')
                if wc is None:
                    wc = P['cond.w'] = torch.zeros(self.sumC, self.dim, device=self.dev)
                    P['cond.b'] = torch.zeros(self.sumC, device=self.dev)
                for bs in self.cond_blocks:
                    wdst, bdst = wc[bs.cond_off:bs.cond_off + bs.din], P['cond.b'][bs.cond_off:bs.cond_off + bs.din]
                    if batch is None:
                        wdst.copy_(bs.mod.mlp[1].weight)
                        bdst.copy_(bs.mod.mlp[1].bias)
                    else:          # the same copies as 1x1 "repacks" inside the one batched launch (46 copy launches per optimizer step)
                        batch.add(bs.mod.mlp[1].weight, T1, wdst, shape=(bs.din, self.dim, 1, 1))
                        batch.add(bs.mod.mlp[1].bias, T1, bdst, shape=(bs.din, 1, 1, 1))
            if batch is not None:
                batch.run()
        self._dirty = False
        self._version = ver

    def _attn_specs(self):
        out = [lv[2] for lv in self.levels_down] + [self.mid_attn] + [lv[2] for lv in self.levels_up]
        return out

    # ------------------------------------------------------------------------------------------
    # forward pieces.  `save` is None for inference; a dict for training (tensors kept for backward)
    # ------------------------------------------------------------------------------------------
    profile_convs = None          # bench.py: list of (event0, event1, flops) per tensor-core conv launch
    profile_shapes = None         # tools/conv_shapes.py: (B, Hg, Wg, Cout, K, nsrc, per_batch) per entry of profile_convs

    @staticmethod
    def _tc_geometry_ok(desc):
        """the tensor-core kernels tile the pixel grid with power-of-two boxes; other image sizes use the fp32 CUDA-core kernel"""
        w, h = desc.Wg, desc.Hg
        pow2 = lambda v: v > 0 and (v & (v - 1)) == 0
        return (w % 128 == 0) if w >= 128 else (pow2(w) and pow2(h))

    def _conv(self, desc, tc):
        impl = self.conv_impl if (tc and self._tc_geometry_ok(desc)) else CONV_SIMT
        if self.profile_convs is not None and impl == CONV_TC:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ops.conv_fwd(desc, impl)
            e1.record()
            k = sum(desc.s[i].ntaps * desc.s[i].C for i in range(desc.nsrc))
            self.profile_convs.append((e0, e1, 2.0 * desc.B * desc.Hg * desc.Wg * desc.Cout * k))
            if self.profile_shapes is not None:
                self.profile_shapes.append((desc.B, desc.Hg, desc.Wg, desc.Cout, k, desc.nsrc, desc.s[0].w_per_batch))
            return
        ops.conv_fwd(desc, impl)

    @staticmethod
    def _pad32(c):
        return (c + 31) // 32 * 32

    def _block(self, bs, xv, outv, cond_all, save, tag, xpad=None):
        """xpad: the block input as a zero-padded 32-channel-multiple view (image-edge block: tensor-core K padded with zeros)"""
        B, H, W = xv.B, xv.H, xv.W
        m = bs.mod
        P = self._packed
        uniq = bs.name if save is not None else tag
        # image-edge block (din = 1 / 3 image channels): its two convolutions over `din` channels run on the tensor cores with K
        # padded to 32 zero-filled channels (activations and packed weights) instead of the register-tiled CUDA-core kernels,
        # which are far from their HBM bound at these channel counts
        edge = bs.din % 32 != 0 and xpad is not None
        ld_h = bs.din if bs.din % 4 == 0 else 4
        ld_in = self._pad32(bs.din) if edge else ld_h
        hn = self.buf('hn.' + uniq, (B, H, W, ld_in), zero=edge)
        stats = hpre = None
        if save is not None:
            if bs.has_norm:
                stats = self.buf('st.' + bs.name, (B, H, W, 2))
                hpre = self.buf('hp.' + bs.name, (B, H, W, ld_h))
        cond = None
        if bs.cond_off is not None:
            cond = C.c_void_p(cond_all.data_ptr() + 4 * bs.cond_off)
        g = m.net[0].g if bs.has_norm else None
        be = m.net[0].b if bs.has_norm else None
        condp = cond if cond is not None else C.c_void_p(0)
        if bs.din % 32 == 0:
            # tiled depthwise conv -> h ; channel LayerNorm as its own HBM pass (training keeps h for the backward anyway)
            h = hpre if (hpre is not None) else hn
            call('cd_dwconv7_fwd', C.c_void_p(xv.addr()), xv.ld, B, H, W, bs.din, ptr(m.ds_conv.weight), ptr(m.ds_conv.bias),
                 condp, self.sumC, ptr(h), ld_in, 0, C.c_void_p(0), 0, stream())
            if bs.has_norm:
                call('cd_layernorm_fwd', ptr(h), ld_in, C.c_int64(B * H * W), bs.din, ptr(g), ptr(be), C.c_float(1e-5),
                     ptr(hn), ld_in, ptr(stats), 0, stream())
        else:
            call('cd_dwconv7_ln_fwd', C.c_void_p(xv.addr()), xv.ld, B, H, W, bs.din, ptr(m.ds_conv.weight), ptr(m.ds_conv.bias),
                 condp, self.sumC, ptr(g), ptr(be), C.c_float(1e-5), ptr(hn), ld_in,
                 ptr(stats), ptr(hpre), ld_h, 0, 0, C.c_void_p(0), 0, stream())
        hv = View(hn, 0, ld_in if edge else bs.din)
        u = self.buf('u.' + uniq, (B, H, W, bs.dmid))
        pre = self.buf('pre.' + bs.name, (B, H, W, bs.dmid)) if save is not None else None
        w1 = P[bs.name + ('.w1p' if edge else '.w1')]
        d1 = ops.make_conv_desc([(hv, T3, w1, False)], View(u), (B, H, W), Cout=bs.dmid,
                                bias=m.net[1].bias, act=ACT_GELU, out2=View(pre) if pre is not None else None)
        self._conv(d1, edge or _tc_ok(bs.din))
        uv = View(u)
        if bs.has_res:
            if edge or _tc_ok(bs.din):
                xs, wr = (xpad, P[bs.name + '.wrp']) if edge else (xv, P[bs.name + '.wr'])
                d2 = ops.make_conv_desc([(uv, T3, P[bs.name + '.w2'], False), (xs, T1, wr, False)],
                                        outv, (B, H, W), Cout=bs.dout, bias=P[bs.name + '.b2r'])
                self._conv(d2, True)
            else:
                dr = ops.make_conv_desc([(xv, T1, P[bs.name + '.wr'], False)], outv, (B, H, W), Cout=bs.dout,
                                        bias=P[bs.name + '.b2r'])
                self._conv(dr, False)
                d2 = ops.make_conv_desc([(uv, T3, P[bs.name + '.w2'], False)], outv, (B, H, W), Cout=bs.dout, resid=outv)
                self._conv(d2, True)
        else:
            d2 = ops.make_conv_desc([(uv, T3, P[bs.name + '.w2'], False)], outv, (B, H, W), Cout=bs.dout,
                                    bias=m.net[3].bias, resid=xv)
            self._conv(d2, True)
        if save is not None:
            save[bs.name] = dict(x=xv, hn=hv, u=uv, pre=View(pre), stats=stats, hpre=hpre, out=outv, ld_h=ld_h,
                                 xpad=xpad if edge else None)

    def _attn(self, spec, xv, outv, save, tag):
        B, H, W = xv.B, xv.H, xv.W
        n = H * W
        dim = spec.dim
        uniq = spec.name if save is not None else tag
        xn = self.buf('xn.' + uniq, (B, H, W, dim))
        stats = self.buf('ast.' + spec.name, (B, H, W, 2)) if save is not None else None
        call('cd_layernorm_fwd', C.c_void_p(xv.addr()), xv.ld, C.c_int64(B * n), dim, ptr(spec.norm.g), ptr(spec.norm.b),
             C.c_float(1e-5), ptr(xn), dim, ptr(stats), 0, stream())
        qkv = self.buf('qkv.' + uniq, (B, H, W, 384))
        dq = ops.make_conv_desc([(View(xn), T1, self._packed[spec.name + '.wqkv'], False)], View(qkv), (B, H, W), Cout=384)
        self._conv(dq, True)
        kmax = self.buf('kmax.' + uniq, (B, 128))
        ksum = self.buf('ksum.' + uniq, (B, 128))
        ctx = self.buf('ctx.' + uniq, (B, 4, 32, 32))
        weff = self.buf('weff.' + uniq, (B, dim, 128))
        nblk, ppb = ops.linattn_ctx_plan(B, n, self.dev)
        ws = self.buf('ctxws.' + uniq, (B, nblk, 4352))
        call('cd_linattn_context_det', ptr(qkv), 384, B, n, nblk, ppb, ptr(ws), ptr(kmax), ptr(ksum), ptr(ctx), stream())
        call('cd_linattn_weff', ptr(ctx), ptr(ksum), ptr(spec.attn.to_out.weight), B, dim, C.c_float(spec.attn.scale), 0,
             ptr(weff), stream())
        do = ops.make_conv_desc([(View(qkv, 0, 128), T1, weff, True)], outv, (B, H, W), Cout=dim,
                                bias=spec.attn.to_out.bias, resid=xv)
        self._conv(do, n >= 128)
        if save is not None:
            save[spec.name] = dict(x=xv, xn=View(xn), qkv=qkv, kmax=kmax, ksum=ksum, ctx=ctx, weff=weff, stats=stats, out=outv)

    def forward(self, x, time, save=None, out=None):
        """x (B,C,H,W) NCHW fp32 cuda, time (B,) int64 -> (B,out_dim,H,W) NCHW."""
        unet = self.unet
        B, Cc, H, W = x.shape
        assert Cc == self.channels
        x = x.contiguous().float()
        time = time.to(device=x.device, dtype=torch.int64).contiguous()
        self.prepare_weights()
        # activations live in engine buffers keyed by (layer, shape): a later forward at the same shape overwrites what an
        # earlier training forward saved for its backward.  Stamp every forward; backward() refuses a stale `save`.
        self._fwd_gen = getattr(self, '_fwd_gen', 0) + 1
        if getattr(self, '_gen_by_shape', None) is None:
            self._gen_by_shape = {}
        self._gen_by_shape[tuple(x.shape)] = self._fwd_gen
        if save is not None:
            save['_gen'] = (tuple(x.shape), self._fwd_gen)
        P = self._packed
        ld0 = Cc if Cc % 4 == 0 else 4
        x0 = self.buf('x0', (B, H, W, ld0))
        call('cd_nchw_to_nhwc', ptr(x), B, Cc, H, W, ptr(x0), ld0, stream())
        x0p = None
        if Cc % 32 != 0:       # second copy with the image channels zero-padded to a tensor-core K chunk (res_conv of the first block;
            ldp = self._pad32(Cc)   # the depthwise 7x7 keeps reading the compact rows: 49 taps per pixel, 8x fewer cache lines)
            x0p = self.buf('x0p', (B, H, W, ldp))
            call('cd_nchw_to_nhwc', ptr(x), B, Cc, H, W, ptr(x0p), ldp, stream())
        cond_all = None
        if unet.time_mlp is not None:
            dim = self.dim
            cond_all = self.buf('cond_all', (B, max(self.sumC, 1)))
            temb = self.buf('temb', (B, dim))
            sinemb = self.buf('sinemb', (B, dim)) if save is not None else None
            hid = self.buf('hid_pre', (B, 4 * dim)) if save is not None else None
            l1, l2 = unet.time_mlp[1], unet.time_mlp[3]
            call('cd_time_mlp_fwd', ptr(time), B, dim, ptr(l1.weight), ptr(l1.bias), ptr(l2.weight), ptr(l2.bias),
                 ptr(P['cond.w']), ptr(P['cond.b']), self.sumC, ptr(sinemb), ptr(hid), ptr(temb), ptr(cond_all), stream())
            if save is not None:
                save['time'] = dict(sinemb=sinemb, hid=hid, temb=temb, cond_all=cond_all, t=time)
        nd = len(self.levels_down)
        nu = len(self.levels_up)
        # spatial size and channels per down level
        xv = View(x0, 0, Cc)
        skips = []
        h, w = H, W
        for i, (b0, b1, at, dn) in enumerate(self.levels_down):
            c = b0.dout
            a = self.buf('d%d.a' % i, (B, h, w, c))
            self._block(b0, xv, View(a), cond_all, save, 'L%d' % i, xpad=View(x0p) if (i == 0 and x0p is not None) else None)
            bb = self.buf('d%d.b' % i, (B, h, w, c))
            self._block(b1, View(a), View(bb), cond_all, save, 'L%d' % i)
            # attention output = skip connection: lives in the concat buffer of the consuming up level
            k = nd - 1 - i                       # up level that pops this skip
            if k < nu:
                cat = self.buf('cat%d' % k, (B, h, w, 2 * c))
                sv = View(cat, c, c)
            else:
                sv = View(self.buf('d%d.s' % i, (B, h, w, c)))
            self._attn(at, View(bb), sv, save, 'L%d' % i)
            skips.append(sv)
            if dn is not None:
                nxt = self.buf('d%d.dn' % i, (B, h // 2, w // 2, c))
                dd = ops.make_conv_desc([(sv, T4, P['downs.%d.3' % i], False)], View(nxt), (B, h // 2, w // 2), stride=2,
                                        Cout=c, bias=dn.bias)
                self._conv(dd, True)
                if save is not None:
                    save['downs.%d.3' % i] = dict(x=sv, out=View(nxt))
                xv = View(nxt)
                h, w = h // 2, w // 2
            else:
                xv = sv
        cm = self.mid1.dout
        m1 = self.buf('mid.a', (B, h, w, cm))
        self._block(self.mid1, xv, View(m1), cond_all, save, 'M')
        m2 = self.buf('mid.b', (B, h, w, cm))
        self._attn(self.mid_attn, View(m1), View(m2), save, 'M')
        # mid_block2 writes the first half of the first concat buffer
        if nu > 0:
            cat0 = self.buf('cat0', (B, h, w, 2 * cm))
            xo = View(cat0, 0, cm)
        else:
            xo = View(self.buf('mid.c', (B, h, w, cm)))
        self._block(self.mid2, View(m2), xo, cond_all, save, 'M')
        xv = xo
        for k, (b0, b1, at, up) in enumerate(self.levels_up):
            cat = self.buf('cat%d' % k, (B, h, w, b0.din))
            a = self.buf('u%d.a' % k, (B, h, w, b0.dout))
            self._block(b0, View(cat), View(a), cond_all, save, 'U%d' % k)
            bb = self.buf('u%d.b' % k, (B, h, w, b0.dout))
            self._block(b1, View(a), View(bb), cond_all, save, 'U%d' % k)
            cc = self.buf('u%d.c' % k, (B, h, w, b0.dout))
            self._attn(at, View(bb), View(cc), save, 'U%d' % k)
            xv = View(cc)
            if up is not None:
                c = b0.dout
                if k + 1 < nu:
                    nb = self.levels_up[k + 1][0]
                    tgt = View(self.buf('cat%d' % (k + 1), (B, 2 * h, 2 * w, nb.din)), 0, c)
                else:
                    tgt = View(self.buf('up_last', (B, 2 * h, 2 * w, c)))
                for (py, px), tp in TPAR.items():
                    du = ops.make_conv_desc([(xv, tp, P['ups.%d.3.%d%d' % (k, py, px)], False)], tgt, (B, h, w), Cout=c,
                                            bias=up.bias, out_map=(2, 2, py, px))
                    self._conv(du, True)
                if save is not None:
                    save['ups.%d.3' % k] = dict(x=xv, out=tgt)
                xv = tgt
                h, w = 2 * h, 2 * w
        fo = self.buf('final.a', (B, h, w, self.final_block.dout))
        self._block(self.final_block, xv, View(fo), None, save, 'F')
        od = self.final_proj.weight.shape[0]
        if out is None:
            out = torch.empty(B, od, h, w, device=x.device, dtype=torch.float32)
        call('cd_conv1x1_to_nchw', ptr(fo), fo.shape[-1], B, h, w, fo.shape[-1], ptr(self.final_proj.weight),
             ptr(self.final_proj.bias), od, ptr(x) if unet.residual else C.c_void_p(0), ptr(out), stream())
        if save is not None:
            save['final'] = dict(x=View(fo), x_in=x)
        return out


from .engine_bwd import BackwardMixin as _BM  # noqa: E402
for _k, _v in _BM.__dict__.items():
    if not _k.startswith('__'):
        setattr(_BackwardHolder, _k, _v)
