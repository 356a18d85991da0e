"""Backward schedule of UnetEngine (training step of GaussianDiffusion.p_losses, DB:963-975 + loss.backward()).

Every gradient the reference obtains from torch autograd through Unet.forward (DB:256-282) is produced here by
sm_90a kernels: data-gradients of the dense convolutions are tap-list convolutions with transposed/flipped
packed weights (cd_conv_fwd), weight-gradients are cd_conv_wgrad, and the HBM-bound pieces have dedicated
kernels (backward.cu).  Parameter gradients are ACCUMULATED into reference-layout views of one flat fp32
buffer (`engine.flat_grad`), which is what the optimizer / the NCCL all-reduce consume.
"""
import ctypes as C
import torch

from . import ops
from .ops import View, CONV_TC, CONV_SIMT, ACT_NONE, ACT_GELU_BWD
from ._lib import call, ptr, stream
from .engine import T1, T3, T4, T3D, TPAR, _tc_ok

NULL = C.c_void_p(0)


def flat_offsets(named_numels):
    """[(name, numel)] -> ({name: (offset, numel)}, total) with every slice 128-byte aligned (dense conv weights are TMA
    operands straight out of the flat parameter buffer: rows of 32 channels must not straddle two 128-byte lines): the layout
    shared by the flat parameter / gradient / Adam-moment / EMA buffers and by the single NCCL all-reduce."""
    table, off = {}, 0
    for n, k in named_numels:
        table[n] = (off, k)
        off += (k + 31) // 32 * 32
    return table, off


def allreduce_mean_(flat_grad, world):
    """the one collective of the training step: sum-all-reduce the flat gradient; returns the 1/world scale that the
    fused Adam kernel applies (DB:1192: the loss is a mean of equal-size per-replica means)."""
    if world > 1:
        torch.distributed.all_reduce(flat_grad)
    return 1.0 / world


class BackwardMixin:
    # ------------------------------------------------------------------------------------------
    # gradient storage
    # ------------------------------------------------------------------------------------------
    def _setup_grads(self):
        if getattr(self, 'flat_grad', None) is not None:
            return
        params = list(self.unet.named_parameters())
        # Flat layout = registration order, except that the parameters whose gradients are produced at the very END of the
        # backward (the time MLP and every block's conditioning projection `mlp.1.*`: _time_bwd) come first.  The rest closes
        # level by level while the backward walks final -> ups -> mid -> downs, so the gradient all-reduce of a finished suffix
        # of the buffer can run while the remaining levels are still being differentiated (`grad_ready_hook`).
        late = [(n, p) for n, p in params if n.startswith('time_mlp.') or '.mlp.1.' in n]
        late_names = {n for n, _ in late}
        order = late + [(n, p) for n, p in params if n not in late_names]
        self._offsets, total = flat_offsets([(n, p.numel()) for n, p in order])
        self.flat_grad = torch.zeros(total, device=self.dev, dtype=torch.float32)
        self._grad_total = total
        starts = {}
        for n, _ in order:
            if n in late_names:
                continue
            grp = '.'.join(n.split('.')[:2]) if n.startswith(('downs.', 'ups.')) else n.split('.')[0]
            starts.setdefault(grp, self._offsets[n][0])
        self._group_start = starts           # first element of every top-level group; groups are contiguous and in registration order
        self.G = {}
        self.Gp = {}                # data_ptr of G[n] -> packed (KH*KW, O, I) view: what the weight-gradient kernels accumulate into
        for n, p in params:
            off, k = self._offsets[n]
            sl = self.flat_grad[off:off + k]
            if n in self.dense_convs:
                # gradients of dense Conv2d weights are STORED packed [KH*KW][O][I] (the tensor-core weight gradient writes that
                # layout: no per-step unpack); .grad is the permuted reference-shaped view of the same memory
                O, I, KH, KW = p.shape
                self.G[n] = sl.view(KH, KW, O, I).permute(2, 3, 0, 1)
                self.Gp[self.G[n].data_ptr()] = sl.view(KH * KW, O, I)
            else:
                self.G[n] = sl.view_as(p)

    def flatten_params(self):
        """rebind every parameter's storage to a slice of ONE flat fp32 buffer (same offsets as flat_grad) so the
        optimizer / EMA / all-reduce are single launches.  state_dict() keys and shapes are unchanged."""
        self._setup_grads()
        if getattr(self, 'flat_param', None) is not None:
            return
        self.flat_param = torch.zeros_like(self.flat_grad)
        with torch.no_grad():
            for n, p in self.unet.named_parameters():
                off, k = self._offsets[n]
                sl = self.flat_param[off:off + k]
                if n in self.dense_convs:
                    # master copy packed [KH*KW][O][I] == the forward operand of the convolution kernels (no per-step repack);
                    # the parameter keeps its reference shape (O, I, KH, KW) as a permuted view, so state_dict() /
                    # load_state_dict() / checkpoints are unchanged.  Adam, EMA and the all-reduce are elementwise over the flat
                    # buffers, whose layouts (parameters, gradients, moments, EMA copy) are identical.
                    O, I, KH, KW = p.shape
                    v = sl.view(KH, KW, O, I).permute(2, 3, 0, 1)
                else:
                    v = sl.view_as(p)
                v.copy_(p.data)
                p.data = v
        self._packed = {}              # operands that aliased the old parameter storage
        if getattr(self, '_graphs', None):
            self._graphs = {}
        self.mark_weights_dirty()

    def attach_grads(self):
        """make every parameter's .grad a view of the flat buffer (zeroing slices that were detached)."""
        self._setup_grads()
        for n, p in self.unet.named_parameters():
            g = self.G[n]
            if p.grad is None or p.grad.data_ptr() != g.data_ptr():
                g.zero_()
                p.grad = g

    def _gname(self, prefix, leaf):
        return prefix + '.' + leaf

    def prepare_weights_bwd(self):
        """packed operands of the data-gradient convolutions (mode 1: N = in-channels, K = out-channels)."""
        ver = self._weights_key()
        if getattr(self, '_bwd_version', None) == ver:
            return
        batch = self._repack_batch('pack_bwd', 'pack')
        tb = getattr(self, '_tapT', None)
        if tb is None:
            tb = self._tapT = ops.TapTransposeBatch()
        tb.clear()

        def packT(key, w, taps):
            """data-gradient operand [tap][I][O]: one job of the single batched transpose when the weight is stored packed,
            else a repack from the reference layout"""
            pv = self.packed_view(w)
            if pv is None:
                self._pack(batch, key, w, taps, mode=1)
                return
            O, I, KH, KW = w.shape
            out = self._packed.get(key)
            if out is None or tuple(out.shape) != (len(taps), I, O):
                out = self._packed[key] = torch.empty((len(taps), I, O), device=w.device, dtype=torch.float32)
            tb.add(pv, O, I, KW, taps, out)

        with torch.no_grad():
            for name, bs in self.blocks.items():
                m = bs.mod
                packT(name + '.w1T', m.net[1].weight, T3D)
                packT(name + '.w2T', m.net[3].weight, T3D)
                if bs.has_res:
                    packT(name + '.wrT', m.res_conv.weight, T1)
            for spec in self._attn_specs():
                packT(spec.name + '.wqkvT', spec.attn.to_qkv.weight, T1)
            for i, lv in enumerate(self.levels_down):
                if lv[3] is not None:
                    for k, tp in TPAR.items():
                        packT('downs.%d.3T.%d%d' % (i, k[0], k[1]), lv[3].weight, tp)
            for i, lv in enumerate(self.levels_up):
                if lv[3] is not None:
                    self._pack(batch, 'ups.%d.3T' % i, lv[3].weight, T4, mode=1, transposed_conv=True)
            if batch is not None:
                batch.run()
            tb.run()
        self._bwd_version = ver

    # ------------------------------------------------------------------------------------------
    profile_wgrads = None
    _unpack_batch = None            # ops.RepackBatch of the running backward() when COLDDIFF_BATCHED_REPACK is on
    _dwp_clean = None

    def _wgrad(self, src, taps, Cout, grid, dout, wgrad_param, bias_param, *, stride=1, out_map=(1, 1, 0, 0),
               transposed_conv=False, key=None, real_c=None):
        """accumulate the weight (and bias) gradient of one tap-list convolution into reference-layout grads.
        real_c: `src` is a zero-padded view of an activation with only real_c channels (image-edge block): the tensor-core
        kernel writes the padded gradient into a scratch buffer whose first real_c columns are then added to the packed gradient."""
        nt = len(taps)
        if real_c is not None:
            pk = self.Gp[wgrad_param.data_ptr()]
            tmp = self.buf('dwp.pad.' + key, (nt, Cout, src.C))
            tmp.zero_()
            d = ops.make_conv_desc([(src, taps, tmp, False)], dout, grid, stride=stride, Cout=Cout, out_map=out_map)
            ops.conv_wgrad(d, dout, tmp, bias_param, impl=self.conv_impl)
            call('cd_add', ptr(pk), real_c, ptr(tmp), src.C, ptr(pk), real_c, C.c_int64(nt * Cout), real_c, stream())
            return
        pk = self.Gp.get(wgrad_param.data_ptr())            # gradients of dense Conv2d weights are stored packed [KH*KW][O][I]
        direct = (not transposed_conv) and ((pk is not None and pk.shape[0] == nt) or (nt == 1 and wgrad_param.is_contiguous()))
        ub = self._unpack_batch
        if direct:
            dwp = pk if pk is not None else wgrad_param
        else:
            dwp = self.buf('dwp.' + key, (nt, Cout, src.C))
            # batched mode: the one-launch unpack at the end of backward() clears what it read, so a buffer is zero-filled
            # here only when it is new or when the previous backward did not reach its unpack
            if ub is None or self._dwp_clean.get(key) != dwp.data_ptr():
                dwp.zero_()
                if ub is not None:
                    self._dwp_clean[key] = dwp.data_ptr()
            if ub is not None:
                assert key not in self._dwp_seen, "packed-gradient buffer %r used twice in one backward" % key
                self._dwp_seen.add(key)
        d = ops.make_conv_desc([(src, taps, dwp, False)], dout, grid, stride=stride, Cout=Cout, out_map=out_map)
        bias_ok = bias_param is not None and out_map == (1, 1, 0, 0)
        if self.profile_wgrads is not None:                 # tools/wgrad_shapes.py: time the weight-gradient GEMM alone
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ops.conv_wgrad(d, dout, dwp, None, impl=self.conv_impl)
            e1.record()
            self.profile_wgrads.append((e0, e1, (grid[0], grid[1], grid[2], Cout, src.C, nt, stride)))
            if bias_ok:
                call('cd_colsum', C.c_void_p(dout.addr()), dout.ld, C.c_int64(grid[0] * grid[1] * grid[2]), Cout, ptr(bias_param), stream())
        else:
            ops.conv_wgrad(d, dout, dwp, bias_param if bias_ok else None, impl=self.conv_impl)
        if not direct:
            if ub is None:
                ops.unpack_wgrad(dwp, taps, wgrad_param, transposed_conv=transposed_conv, accumulate=True)
            else:
                ub.add(dwp, taps, wgrad_param, shape=tuple(wgrad_param.shape), transposed_conv=transposed_conv)

    def _block_bwd(self, bs, save, dyv, need_dx=True):
        sv = save[bs.name]
        xv, hv, uv, prev, stats, hpre = sv['x'], sv['hn'], sv['u'], sv['pre'], sv['stats'], sv['hpre']
        B, H, W = xv.B, xv.H, xv.W
        m = bs.mod
        P, G = self._packed, self.G
        pn = bs.name
        grid = (B, H, W)
        # ---- conv2 (+ res_conv) ----
        xpad = sv.get('xpad')                      # image-edge block: zero-padded 32-channel views feed the tensor-core kernels
        edge_c = bs.din if xpad is not None else None
        if bs.has_res:
            # conv2 and res_conv add into the same output: one column sum of dy feeds both bias gradients
            tmp = self.buf('g.dbias', (max(b_.dout for b_ in self.blocks.values()),))
            tmp.zero_()
            self._wgrad(uv, T3, bs.dout, grid, dyv, G[pn + '.net.3.weight'], tmp, key=pn + '.w2')
            self._wgrad(xpad if xpad is not None else xv, T1, bs.dout, grid, dyv, G[pn + '.res_conv.weight'], None, key=pn + '.wr',
                        real_c=edge_c)
            for leaf in ('.net.3.bias', '.res_conv.bias'):
                call('cd_add', ptr(G[pn + leaf]), bs.dout, ptr(tmp), bs.dout, ptr(G[pn + leaf]), bs.dout, C.c_int64(1), bs.dout, stream())
        else:
            self._wgrad(uv, T3, bs.dout, grid, dyv, G[pn + '.net.3.weight'], G[pn + '.net.3.bias'], key=pn + '.w2')
        dpre = self.buf('g.pre.%dx%dx%d' % (H, W, bs.dmid), (B, H, W, bs.dmid))
        d = ops.make_conv_desc([(dyv, T3D, P[pn + '.w2T'], False)], View(dpre), grid, Cout=bs.dmid,
                               act=ACT_GELU_BWD, aux=prev)
        self._conv(d, _tc_ok(bs.dout))
        # ---- conv1 ----
        self._wgrad(hv, T3, bs.dmid, grid, View(dpre), G[pn + '.net.1.weight'], G[pn + '.net.1.bias'], key=pn + '.w1', real_c=edge_c)
        ld_in = sv.get('ld_h', hv.ld)
        dhn = self.buf('g.hn.%dx%dx%d' % (H, W, ld_in), (B, H, W, ld_in))
        d = ops.make_conv_desc([(View(dpre), T3D, P[pn + '.w1T'], False)], View(dhn, 0, bs.din), grid, Cout=bs.din)
        self._conv(d, True)
        # ---- LayerNorm ----
        if bs.has_norm:
            dh = self.buf('g.h.%dx%dx%d' % (H, W, ld_in), (B, H, W, ld_in))
            call('cd_layernorm_bwd', ptr(dhn), ld_in, ptr(hpre), ld_in, ptr(stats), ptr(m.net[0].g), C.c_int64(B * H * W),
                 bs.din, NULL, 0, ptr(dh), ld_in, ptr(G[pn + '.net.0.g']), ptr(G[pn + '.net.0.b']), stream())
        else:
            dh = dhn
        # ---- time conditioning + depthwise bias ----
        if bs.cond_off is not None:
            dslice = C.c_void_p(self._dcond.data_ptr() + 4 * bs.cond_off)
            call('cd_colsum_batched', ptr(dh), ld_in, B, C.c_int64(H * W), bs.din, dslice, self.sumC, stream())
            # d(ds_conv.bias) = sum_b dcond[b]  (same per-pixel gradient, already reduced over pixels)
            call('cd_colsum', dslice, self.sumC, C.c_int64(B), bs.din, ptr(G[pn + '.ds_conv.bias']), stream())
        else:
            call('cd_colsum', ptr(dh), ld_in, C.c_int64(B * H * W), bs.din, ptr(G[pn + '.ds_conv.bias']), stream())
        call('cd_dwconv7_wgrad', ptr(dh), ld_in, C.c_void_p(xv.addr()), xv.ld, B, H, W, bs.din,
             ptr(G[pn + '.ds_conv.weight']), stream())
        if not need_dx:
            return None
        # ---- dx = dwconv7^T(dh) + residual path ----
        if bs.has_res:
            r = self.buf('g.r.%dx%dx%d' % (H, W, ld_in), (B, H, W, ld_in))
            d = ops.make_conv_desc([(dyv, T1, P[pn + '.wrT'], False)], View(r, 0, bs.din), grid, Cout=bs.din)
            self._conv(d, _tc_ok(bs.dout))
            addv = View(r, 0, bs.din)
        else:
            addv = dyv
        dx = self.buf('g.x.' + pn, (B, H, W, ld_in))
        if bs.din % 32 == 0:
            call('cd_dwconv7_fwd', ptr(dh), ld_in, B, H, W, bs.din, ptr(m.ds_conv.weight), NULL, NULL, 0, ptr(dx), ld_in, 1,
                 C.c_void_p(addv.addr()), addv.ld, stream())
        else:
            call('cd_dwconv7_ln_fwd', ptr(dh), ld_in, B, H, W, bs.din, ptr(m.ds_conv.weight), NULL, NULL, 0, NULL, NULL,
                 C.c_float(0.0), ptr(dx), ld_in, NULL, NULL, 0, 0, 1, C.c_void_p(addv.addr()), addv.ld, stream())
        return View(dx, 0, bs.din)

    def _attn_bwd(self, spec, save, dyv):
        sv = save[spec.name]
        xv, xnv, qkv, kmax, ksum, ctx, weff, stats = sv['x'], sv['xn'], sv['qkv'], sv['kmax'], sv['ksum'], sv['ctx'], sv['weff'], sv['stats']
        B, H, W = xv.B, xv.H, xv.W
        n = H * W
        dim = spec.dim
        a = spec.attn
        P, G = self._packed, self.G
        pn = spec.name + '.fn'
        grid = (B, H, W)
        tc_pb = n >= 128
        call('cd_colsum', C.c_void_p(dyv.addr()), dyv.ld, C.c_int64(B * n), dim, ptr(G[pn + '.fn.to_out.bias']), stream())
        # dweff[b][co][hd] = sum_pix dy[pix][co] * q[pix][hd]
        dweff = self.buf('g.dweff', (B, dim, 128))
        dweff.zero_()
        qv = View(qkv, 0, 128)
        d = ops.make_conv_desc([(qv, T1, dweff, True)], dyv, grid, Cout=dim)
        ops.conv_wgrad(d, dyv, dweff, None, impl=self.conv_impl)
        dctxn = self.buf('g.dctxn', (B, 4, 32, 32))
        rowdot = self.buf('g.rowdot', (B, 128))
        call('cd_linattn_bwd_small', ptr(dweff), ptr(ctx), ptr(ksum), ptr(a.to_out.weight), B, dim, C.c_float(a.scale),
             ptr(G[pn + '.fn.to_out.weight']), ptr(dctxn), ptr(rowdot), stream())
        dqkv = self.buf('g.qkv.%dx%d' % (H, W), (B, H, W, 384))
        wt = self.buf('g.wefft', (B, 128, dim))
        call('cd_transpose_weff', ptr(weff), B, dim, ptr(wt), stream())
        d = ops.make_conv_desc([(dyv, T1, wt, True)], View(dqkv, 0, 128), grid, Cout=128)
        self._conv(d, tc_pb and _tc_ok(dim))
        call('cd_linattn_bwd_kv', ptr(qkv), 384, B, n, ptr(kmax), ptr(ksum), ptr(dctxn), ptr(rowdot), ptr(dqkv), 384, stream())
        # to_qkv
        self._wgrad(xnv, T1, 384, grid, View(dqkv), G[pn + '.fn.to_qkv.weight'], None, key=spec.name + '.wqkv')
        dxn = self.buf('g.xn.%dx%dx%d' % (H, W, dim), (B, H, W, dim))
        d = ops.make_conv_desc([(View(dqkv), T1, P[spec.name + '.wqkvT'], False)], View(dxn), grid, Cout=dim)
        self._conv(d, True)
        dx = self.buf('g.x.' + spec.name, (B, H, W, dim))
        call('cd_layernorm_bwd', ptr(dxn), dim, C.c_void_p(xv.addr()), xv.ld, ptr(stats), ptr(spec.norm.g), C.c_int64(B * n),
             dim, C.c_void_p(dyv.addr()), dyv.ld, ptr(dx), dim, ptr(G[pn + '.norm.g']), ptr(G[pn + '.norm.b']), stream())
        return View(dx)

    # ------------------------------------------------------------------------------------------
    def backward(self, save, dout):
        """dout: (B, out_dim, H, W) NCHW gradient of the network output.  Accumulates into self.G."""
        unet = self.unet
        shape, gen = save.get('_gen', (None, None))
        if shape is not None and self._gen_by_shape.get(shape) != gen:
            raise RuntimeError("Unet backward: another forward with input shape %r ran on this network after the forward being "
                               "differentiated; the engine keeps one set of saved activations per input shape -- call "
                               "backward() before the next forward (e.g. accumulate micro-batches one at a time)" % (shape,))
        self._setup_grads()
        self.prepare_weights_bwd()
        P, G = self._packed, self.G
        dout = dout.contiguous().float()
        B = dout.shape[0]
        # packed weight gradients: unpacked one by one right after each wgrad, or (COLDDIFF_BATCHED_REPACK) all at once below
        self._unpack_batch = self._repack_batch('unpack', 'unpack') if self.profile_wgrads is None else None
        if self._unpack_batch is None or self._dwp_clean is None or getattr(self, '_dwp_pending', False):
            self._dwp_clean = {}                    # a backward that raised half-way left partial sums behind: refill all
        self._dwp_pending = self._unpack_batch is not None
        self._dwp_seen = set()
        self._dcond = self.buf('g.dcond', (B, max(self.sumC, 1)))
        self._dcond.zero_()
        nd, nu = len(self.levels_down), len(self.levels_up)
        # ---- final projection + final block ----
        fx = save['final']['x']
        h, w = fx.H, fx.W
        dfo = self.buf('g.final', (B, h, w, fx.ld))
        od = self.final_proj.weight.shape[0]
        call('cd_conv1x1_to_nchw_bwd', ptr(dout), ptr(fx.t), fx.ld, B, h, w, fx.C, ptr(self.final_proj.weight), od,
             ptr(dfo), fx.ld, ptr(G['final_conv.1.weight']), ptr(G['final_conv.1.bias']), stream())
        d = self._block_bwd(self.final_block, save, View(dfo))
        # ---- up path ----
        dskip = {}
        for k in reversed(range(nu)):
            b0, b1, at, up = self.levels_up[k]
            if up is not None:
                sv = save['ups.%d.3' % k]
                xv = sv['x']
                c = xv.C
                hh, ww = xv.H, xv.W
                # bias
                call('cd_colsum', C.c_void_p(d.addr()), d.ld, C.c_int64(B * d.H * d.W), c, ptr(G['ups.%d.3.bias' % k]), stream())
                for (py, px), tp in TPAR.items():
                    self._wgrad(xv, tp, c, (B, hh, ww), d, G['ups.%d.3.weight' % k], None, out_map=(2, 2, py, px),
                                transposed_conv=True, key='ups.%d.3.%d%d' % (k, py, px))
                dxu = self.buf('g.up%d' % k, (B, hh, ww, c))
                dd = ops.make_conv_desc([(d, T4, P['ups.%d.3T' % k], False)], View(dxu), (B, hh, ww), stride=2, Cout=c)
                self._conv(dd, True)
                d = View(dxu)
            d = self._attn_bwd(at, save, d)
            d = self._block_bwd(b1, save, d)
            dcat = self._block_bwd(b0, save, d)             # gradient w.r.t. the concat buffer [x | skip]
            c = dcat.C // 2
            dskip[nd - 1 - k] = View(dcat.t, c, c)
            d = View(dcat.t, 0, c)
        # ---- mid ----
        d = self._block_bwd(self.mid2, save, d)
        d = self._attn_bwd(self.mid_attn, save, d)
        d = self._block_bwd(self.mid1, save, d)
        self._grads_ready_from('ups.0')                    # ups.*, mid_block1, mid_attn, mid_block2, final_conv: 57 % of the buffer
        # ---- down path ----
        for i in reversed(range(nd)):
            b0, b1, at, dn = self.levels_down[i]
            sk = dskip.get(i)
            if dn is not None:
                sv = save['downs.%d.3' % i]
                xv = sv['x']
                c = xv.C
                hh, ww = xv.H, xv.W
                self._wgrad(xv, T4, c, (B, hh // 2, ww // 2), d, G['downs.%d.3.weight' % i], G['downs.%d.3.bias' % i],
                            stride=2, key='downs.%d.3' % i)
                dsv = self.buf('g.dn%d' % i, (B, hh, ww, c))
                for (py, px), tp in TPAR.items():
                    dd = ops.make_conv_desc([(d, tp, P['downs.%d.3T.%d%d' % (i, py, px)], False)], View(dsv), (B, hh // 2, ww // 2),
                                            Cout=c, out_map=(2, 2, py, px), resid=sk)
                    self._conv(dd, True)
                d = View(dsv)
            elif sk is not None:
                # last level: output feeds mid_block1 directly AND the skip -> sum the two gradients
                dsum = self.buf('g.dsum%d' % i, (B, d.H, d.W, d.C))
                call('cd_add', C.c_void_p(d.addr()), d.ld, C.c_void_p(sk.addr()), sk.ld, ptr(dsum), d.C, C.c_int64(B * d.H * d.W), d.C, stream())
                d = View(dsum)
            d = self._attn_bwd(at, save, d)
            d = self._block_bwd(b1, save, d)
            d = self._block_bwd(b0, save, d, need_dx=(i > 0))
            if i >= 2:
                self._grads_ready_from('downs.%d' % i)     # the two coarsest levels carry 22 of the 24 M down-path parameters
        # ---- time MLP ----
        if unet.time_mlp is not None:
            self._time_bwd(save)
        if self._unpack_batch is not None:
            self._unpack_batch.run(accumulate=True, clear_src=True)
            self._dwp_pending = False

    def _grads_ready_from(self, group):
        """tell the trainer that flat_grad[start of `group` : previous mark) holds final values (multi-GPU: the all-reduce of
        that range is issued now and overlaps the rest of the backward).  Marks move from the end of the buffer to the front."""
        hook = getattr(self, 'grad_ready_hook', None)
        if hook is None or self._unpack_batch is not None:     # batched unpack writes the reference-layout gradients at the end
            return
        lo = self._group_start.get(group)
        hi = getattr(self, '_ready_mark', self._grad_total)
        if lo is None or lo >= hi:
            return
        self._ready_mark = lo
        hook(lo, hi)

    def _time_bwd(self, save):
        sv = save['time']
        unet = self.unet
        G, P = self.G, self._packed
        dim = self.dim
        B = sv['temb'].shape[0]
        dcond = self._dcond
        temb, hid_pre, sinemb = sv['temb'], sv['hid'], sv['sinemb']
        gt = self.buf('g.gt', (B, dim))
        call('cd_gelu_bwd', NULL, ptr(temb), C.c_int64(B * dim), NULL, ptr(gt), stream())
        for bs in self.cond_blocks:
            wname = bs.name + '.mlp.1.weight'
            # dW[c][k] += sum_b dcond[b][off+c] * gt[b][k]
            call('cd_small_gemm', C.c_void_p(dcond.data_ptr() + 4 * bs.cond_off), self.sumC, 1, ptr(gt), dim, 0,
                 ptr(G[wname]), dim, bs.din, dim, B, 1, stream())
            call('cd_colsum', C.c_void_p(dcond.data_ptr() + 4 * bs.cond_off), self.sumC, C.c_int64(B), bs.din,
                 ptr(G[bs.name + '.mlp.1.bias']), stream())
        dgt = self.buf('g.dgt', (B, dim))
        call('cd_small_gemm', ptr(dcond), self.sumC, 0, ptr(P['cond.w']), dim, 0, ptr(dgt), dim, B, dim, self.sumC, 0, stream())
        dtemb = self.buf('g.dtemb', (B, dim))
        call('cd_gelu_bwd', ptr(dgt), ptr(temb), C.c_int64(B * dim), ptr(dtemb), NULL, stream())
        l1, l2 = unet.time_mlp[1], unet.time_mlp[3]
        hact = self.buf('g.hact', (B, 4 * dim))
        call('cd_gelu_bwd', NULL, ptr(hid_pre), C.c_int64(B * 4 * dim), NULL, ptr(hact), stream())
        call('cd_small_gemm', ptr(dtemb), dim, 1, ptr(hact), 4 * dim, 0, ptr(G['time_mlp.3.weight']), 4 * dim, dim, 4 * dim, B, 1, stream())
        call('cd_colsum', ptr(dtemb), dim, C.c_int64(B), dim, ptr(G['time_mlp.3.bias']), stream())
        dh = self.buf('g.dhid', (B, 4 * dim))
        call('cd_small_gemm', ptr(dtemb), dim, 0, ptr(l2.weight), 4 * dim, 0, ptr(dh), 4 * dim, B, 4 * dim, dim, 0, stream())
        call('cd_gelu_bwd', ptr(dh), ptr(hid_pre), C.c_int64(B * 4 * dim), ptr(dh), NULL, stream())
        call('cd_small_gemm', ptr(dh), 4 * dim, 1, ptr(sinemb), dim, 0, ptr(G['time_mlp.1.weight']), dim, 4 * dim, dim, B, 1, stream())
        call('cd_colsum', ptr(dh), 4 * dim, C.c_int64(B), 4 * dim, ptr(G['time_mlp.1.bias']), stream())
