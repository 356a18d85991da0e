"""`Model` -- the DDPM-style ResNet UNet of the reference (deblurring-diffusion-pytorch/deblurring_diffusion_pytorch/Model2.py
:191-332, "M2"; used by the CIFAR-10 drivers, BASELINE config 2), with the reference's keyword-only constructor,
`forward(x, t)` and state_dict keys, executed on the sm_90a engine (inference / sampling path).

Forward schedule (NHWC fp32): GroupNorm(32)+swish kernels (the time-embedding projection is folded into norm2's load),
tensor-core tap-list convolutions for conv1/conv2/nin_shortcut/q/k/v/proj_out/Downsample (asymmetric zero pad = TMA
out-of-bounds fill) and for the two batched matmuls of AttnBlock (per-batch-weight 1x1 convolutions: k is already
the [n][C] weight slab, v is transposed once), a row-softmax kernel, and channel-sliced concat buffers instead of
torch.cat.  Training (backward of GroupNorm / softmax attention, dropout) lives in model2_train.py and is reachable only
with COLDDIFF_MODEL_TRAINING=1 ; otherwise calling the model with autograd enabled raises.
"""
import ctypes as C
import torch
import torch.nn as nn

from . import ops
from .ops import View, CONV_TC, CONV_SIMT, ACT_NONE
from ._lib import call, ptr, stream

T3 = ops.taps_conv(3, 1)
T1 = ops.taps_conv(1, 0)
TDOWN = [(ky, kx, ky, kx) for ky in range(3) for kx in range(3)]     # F.pad(0,1,0,1) + conv3x3 stride 2 padding 0 (M2:66-70)


def Normalize(in_channels):
    return torch.nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)


class _P(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter container: arithmetic runs in libcolddiff")


class Upsample(_P):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)


class Downsample(_P):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)


class ResnetBlock(_P):
    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout, temb_channels=512):
        super().__init__()
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut
        self.norm1 = Normalize(in_channels)
        self.conv1 = torch.nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.temb_proj = torch.nn.Linear(temb_channels, out_channels)
        self.norm2 = Normalize(out_channels)
        self.dropout = torch.nn.Dropout(dropout)
        self.conv2 = torch.nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            if self.use_conv_shortcut:
                self.conv_shortcut = torch.nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
            else:
                self.nin_shortcut = torch.nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)


class AttnBlock(_P):
    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1)
        self.k = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1)
        self.v = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1)
        self.proj_out = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1)


class Model(nn.Module):
    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution):
        super().__init__()
        self.ch = ch
        self.temb_ch = self.ch * 4
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.out_ch = out_ch
        self.temb = nn.Module()
        self.temb.dense = nn.ModuleList([torch.nn.Linear(self.ch, self.temb_ch), torch.nn.Linear(self.temb_ch, self.temb_ch)])
        self.conv_in = torch.nn.Conv2d(in_channels, self.ch, kernel_size=3, stride=1, padding=1)
        curr_res = resolution
        in_ch_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        for i_level in range(self.num_resolutions):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for i_block in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            down = nn.Module()
            down.block, down.attn = block, attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            skip_in = ch * ch_mult[i_level]
            for i_block in range(self.num_res_blocks + 1):
                if i_block == self.num_res_blocks:
                    skip_in = ch * in_ch_mult[i_level]
                block.append(ResnetBlock(in_channels=block_in + skip_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            up = nn.Module()
            up.block, up.attn = block, attn
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
                curr_res = curr_res * 2
            self.up.insert(0, up)
        self.norm_out = Normalize(block_in)
        self.conv_out = torch.nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)
        self._bufs, self._packed, self._version = {}, {}, None
        self.conv_impl = CONV_TC

    # ---------------------------------------------------------------------------------------------------------
    def _apply(self, fn, *a, **k):
        self._bufs, self._packed, self._version = {}, {}, None
        return super()._apply(fn, *a, **k)

    def __deepcopy__(self, memo):
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = ({} if k in ('_bufs', '_packed') else (None if k in ('_version', '_engine', '_bwd_version') else copy.deepcopy(v, memo)))
        return new

    @property
    def engine(self):
        """flat parameter / gradient buffers for Trainer + FusedAdamEMA (training path, model2_train.py)"""
        if getattr(self, '_engine', None) is None:
            from .model2_train import ModelEngine
            self._engine = ModelEngine(self)
        return self._engine

    def _plan(self, B, H):
        """concat-buffer plan of forward(): every skip tensor is written straight into the second channel slice of the concat
        buffer of the up block that pops it (first slice = the running h).  -> {'cat_bufs': [(buffer, hin, skip_ch)], 'skip_view'}"""
        up_blocks = [(lv, ib) for lv in reversed(range(self.num_resolutions)) for ib in range(self.num_res_blocks + 1)]
        skip_ch, skip_res = [self.ch], [H]
        res = H
        for i_level in range(self.num_resolutions):
            for b in self.down[i_level].block:
                skip_ch.append(b.out_channels); skip_res.append(res)
            if i_level != self.num_resolutions - 1:
                skip_ch.append(skip_ch[-1]); res //= 2; skip_res.append(res)
        nsk = len(skip_ch)
        cat_bufs = []
        for j, (lv, ib) in enumerate(up_blocks):
            blk = self.up[lv].block[ib]
            sk = nsk - 1 - j
            r = skip_res[sk]
            cat_bufs.append((self._buf('cat.%d' % j, (B, r, r, blk.in_channels)), blk.in_channels - skip_ch[sk], skip_ch[sk]))

        def skip_view(sk):
            buf, hin, sc = cat_bufs[nsk - 1 - sk]
            return View(buf, hin, sc)
        return dict(cat_bufs=cat_bufs, skip_view=skip_view)

    def _buf(self, name, shape):
        key = (name, tuple(shape))
        t = self._bufs.get(key)
        if t is None:
            t = self._bufs[key] = torch.empty(shape, device=self.conv_in.weight.device, dtype=torch.float32)
        return t

    def _resblocks(self):
        out = []
        for i, d in enumerate(self.down):
            out += [('down.%d.block.%d' % (i, j), b) for j, b in enumerate(d.block)]
        out += [('mid.block_1', self.mid.block_1), ('mid.block_2', self.mid.block_2)]
        for i, u in enumerate(self.up):
            out += [('up.%d.block.%d' % (i, j), b) for j, b in enumerate(u.block)]
        return out

    def _attns(self):
        out = []
        for i, d in enumerate(self.down):
            out += [('down.%d.attn.%d' % (i, j), a) for j, a in enumerate(d.attn)]
        out.append(('mid.attn_1', self.mid.attn_1))
        for i, u in enumerate(self.up):
            out += [('up.%d.attn.%d' % (i, j), a) for j, a in enumerate(u.attn)]
        return out

    def _prepare(self):
        ver = tuple(p._version for p in self.parameters())
        if ver == self._version:
            return
        P = self._packed
        pk = lambda key, w, taps: P.__setitem__(key, ops.pack_weight(w, taps, round_tf32=False, out=P.get(key)))
        with torch.no_grad():
            pk('conv_in', self.conv_in.weight, T3)
            pk('conv_out', self.conv_out.weight, T3)
            off = 0
            for name, b in self._resblocks():
                pk(name + '.c1', b.conv1.weight, T3)
                pk(name + '.c2', b.conv2.weight, T3)
                if hasattr(b, 'nin_shortcut'):
                    pk(name + '.sc', b.nin_shortcut.weight, T1)
                    P[name + '.b2s'] = (b.conv2.bias + b.nin_shortcut.bias).contiguous()
                elif hasattr(b, 'conv_shortcut'):
                    pk(name + '.sc', b.conv_shortcut.weight, T3)
                    P[name + '.b2s'] = (b.conv2.bias + b.conv_shortcut.bias).contiguous()
                b._cond_off = off
                off += b.out_channels
            self._sumC = off
            wc = torch.zeros(off, self.temb_ch, device=self.conv_in.weight.device)
            bc = torch.zeros(off, device=self.conv_in.weight.device)
            for name, b in self._resblocks():
                wc[b._cond_off:b._cond_off + b.out_channels].copy_(b.temb_proj.weight)
                bc[b._cond_off:b._cond_off + b.out_channels].copy_(b.temb_proj.bias)
            P['cond.w'], P['cond.b'] = wc, bc
            for name, a in self._attns():
                for leaf in ('q', 'k', 'v', 'proj_out'):
                    pk(name + '.' + leaf, getattr(a, leaf).weight, T1)
            for i, d in enumerate(self.down):
                if hasattr(d, 'downsample') and d.downsample.with_conv:
                    pk('down.%d.ds' % i, d.downsample.conv.weight, TDOWN)
            for i, u in enumerate(self.up):
                if hasattr(u, 'upsample') and u.upsample.with_conv:
                    pk('up.%d.us' % i, u.upsample.conv.weight, T3)
        self._version = ver

    # ---- kernels ---------------------------------------------------------------------------------------------
    def _conv(self, desc, tc=True):
        ops.conv_fwd(desc, self.conv_impl if tc else CONV_SIMT)

    def _gn(self, xv, norm, outv, swish, cond=None):
        B, H, W = xv.B, xv.H, xv.W
        condp = C.c_void_p(cond) if cond is not None else C.c_void_p(0)
        call('cd_groupnorm_fwd', C.c_void_p(xv.addr()), xv.ld, B, C.c_int64(H * W), xv.C, norm.num_groups, condp, self._sumC,
             ptr(norm.weight), ptr(norm.bias), C.c_float(norm.eps), int(swish), C.c_void_p(outv.addr()), outv.ld, stream())

    def _res(self, name, b, xv, outv, cond_all):
        """ResnetBlock.forward (M2:114-133), dropout in eval mode"""
        B, H, W = xv.B, xv.H, xv.W
        P = self._packed
        cin, cout = b.in_channels, b.out_channels
        n1 = self._buf('n1.%dx%dx%d' % (H, W, cin), (B, H, W, cin))
        self._gn(xv, b.norm1, View(n1), True)
        h1 = self._buf('h1.%dx%dx%d' % (H, W, cout), (B, H, W, cout))
        self._conv(ops.make_conv_desc([(View(n1), T3, P[name + '.c1'], False)], View(h1), (B, H, W), Cout=cout, bias=b.conv1.bias))
        n2 = self._buf('n2.%dx%dx%d' % (H, W, cout), (B, H, W, cout))
        self._gn(View(h1), b.norm2, View(n2), True, cond=cond_all.data_ptr() + 4 * b._cond_off)   # + temb_proj(swish(temb))[b, c]
        if cin != cout:
            taps_sc = T1 if hasattr(b, 'nin_shortcut') else T3
            d = ops.make_conv_desc([(View(n2), T3, P[name + '.c2'], False), (xv, taps_sc, P[name + '.sc'], False)], outv, (B, H, W),
                                   Cout=cout, bias=P[name + '.b2s'])
        else:
            d = ops.make_conv_desc([(View(n2), T3, P[name + '.c2'], False)], outv, (B, H, W), Cout=cout, bias=b.conv2.bias, resid=xv)
        self._conv(d)

    def _attn(self, name, a, xv, outv):
        """AttnBlock.forward (M2:164-188)"""
        B, H, W = xv.B, xv.H, xv.W
        n, c = H * W, a.in_channels
        P = self._packed
        hn = self._buf('an.%dx%dx%d' % (H, W, c), (B, H, W, c))
        self._gn(xv, a.norm, View(hn), False)
        q = self._buf('aq.%dx%d' % (n, c), (B, H, W, c)); k = self._buf('ak.%dx%d' % (n, c), (B, H, W, c)); v = self._buf('av.%dx%d' % (n, c), (B, H, W, c))
        for t, leaf in ((q, 'q'), (k, 'k'), (v, 'v')):
            self._conv(ops.make_conv_desc([(View(hn), T1, P[name + '.' + leaf], False)], View(t), (B, H, W), Cout=c, bias=getattr(a, leaf).bias))
        tc = n >= 128 and n % 32 == 0
        s = self._buf('as.%d' % n, (B, H, W, n))                       # scores[b, i, j] = sum_c q[b,i,c] k[b,j,c]: weights = k[b] ([n][c])
        # the scores feed exp(): keep them in fp32 CUDA cores (the reference's torch.bmm is fp32 too: matmul.allow_tf32=False)
        self._conv(ops.make_conv_desc([(View(q), T1, k, True)], View(s), (B, H, W), Cout=n), False)
        call('cd_softmax_rows', ptr(s), n, C.c_int64(B * n), n, C.c_float(int(c) ** (-0.5)), stream())
        vt = self._buf('avt.%dx%d' % (n, c), (B, c, n))                # v^T per image: the [Cout=c][Cin=n] weight slab of the second matmul
        call('cd_transpose_batched', ptr(v), c, B, n, c, ptr(vt), stream())
        ho = self._buf('ah.%dx%d' % (n, c), (B, H, W, c))
        self._conv(ops.make_conv_desc([(View(s), T1, vt, True)], View(ho), (B, H, W), Cout=c), tc)
        self._conv(ops.make_conv_desc([(View(ho), T1, P[name + '.proj_out'], False)], outv, (B, H, W), Cout=c, bias=a.proj_out.bias, resid=xv))

    # ---------------------------------------------------------------------------------------------------------
    def forward(self, x, t):
        if not x.is_cuda:
            raise RuntimeError("cold_diffusion_models_b200.Model runs on a CUDA device (H100) only; got %s" % x.device)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            from . import model2_train
            return model2_train.ModelFunction.apply(self, x, t, *self.engine.param_list())
        assert x.shape[2] == x.shape[3] == self.resolution
        self._prepare()
        P = self._packed
        B, Cin, H, W = x.shape
        x = x.contiguous().float()
        t = t.to(device=x.device, dtype=torch.int64).contiguous()
        cond_all = self._buf('cond', (B, self._sumC))
        d0, d1 = self.temb.dense[0], self.temb.dense[1]
        call('cd_time_mlp2_fwd', ptr(t), B, self.ch, self.temb_ch, self.temb_ch, 1, ptr(d0.weight), ptr(d0.bias), ptr(d1.weight), ptr(d1.bias),
             ptr(P['cond.w']), ptr(P['cond.b']), self._sumC, ptr(self._buf('temb', (B, self.temb_ch))), ptr(cond_all), stream())
        ld0 = Cin if Cin % 4 == 0 else 4
        x0 = self._buf('x0', (B, H, W, ld0))
        call('cd_nchw_to_nhwc', ptr(x), B, Cin, H, W, ptr(x0), ld0, stream())

        # ---- plan the skip stack: every hs entry is consumed by exactly one up block; it is written straight into the second
        # channel slice of that block's concat buffer (first slice = the running h)
        up_blocks = []          # consumption order
        for i_level in reversed(range(self.num_resolutions)):
            for i_block in range(self.num_res_blocks + 1):
                up_blocks.append((i_level, i_block))
        skip_ch, skip_res = [self.ch], [H]          # production order of hs
        res = H
        for i_level in range(self.num_resolutions):
            for b in self.down[i_level].block:
                skip_ch.append(b.out_channels); skip_res.append(res)
            if i_level != self.num_resolutions - 1:
                skip_ch.append(skip_ch[-1]); res //= 2; skip_res.append(res)
        nsk = len(skip_ch)
        cat_bufs = []
        for j, (lv, ib) in enumerate(up_blocks):     # up block j pops hs[nsk-1-j]
            blk = self.up[lv].block[ib]
            sk = nsk - 1 - j
            hin = blk.in_channels - skip_ch[sk]
            r = skip_res[sk]
            cat_bufs.append((self._buf('cat.%d' % j, (B, r, r, blk.in_channels)), hin, skip_ch[sk]))

        def skip_view(sk):
            buf, hin, sc = cat_bufs[nsk - 1 - sk]
            return View(buf, hin, sc)

        # ---- down path ----
        hv = skip_view(0)
        self._conv(ops.make_conv_desc([(View(x0, 0, Cin), T3, P['conv_in'], False)], hv, (B, H, W), Cout=self.ch, bias=self.conv_in.bias), False)
        sk, res = 0, H
        for i_level in range(self.num_resolutions):
            d = self.down[i_level]
            for i_block, b in enumerate(d.block):
                sk += 1
                tgt = skip_view(sk)
                if len(d.attn) > 0:
                    tmp = View(self._buf('dtmp.%d.%d' % (res, b.out_channels), (B, res, res, b.out_channels)))
                    self._res('down.%d.block.%d' % (i_level, i_block), b, hv, tmp, cond_all)
                    self._attn('down.%d.attn.%d' % (i_level, i_block), d.attn[i_block], tmp, tgt)
                else:
                    self._res('down.%d.block.%d' % (i_level, i_block), b, hv, tgt, cond_all)
                hv = tgt
            if i_level != self.num_resolutions - 1:
                sk += 1
                tgt = skip_view(sk)
                if d.downsample.with_conv:
                    self._conv(ops.make_conv_desc([(hv, TDOWN, P['down.%d.ds' % i_level], False)], tgt, (B, res // 2, res // 2), stride=2,
                                                  Cout=hv.C, bias=d.downsample.conv.bias))
                else:
                    raise NotImplementedError("resamp_with_conv=False (avg-pool resampling) is not used by any reference driver")
                res //= 2
                hv = tgt
        # ---- middle ----
        cm = hv.C
        m1 = View(self._buf('m1', (B, res, res, cm))); m2 = View(self._buf('m2', (B, res, res, cm)))
        self._res('mid.block_1', self.mid.block_1, hv, m1, cond_all)
        self._attn('mid.attn_1', self.mid.attn_1, m1, m2)
        first_buf, hin0, _ = cat_bufs[0]
        h_run = View(first_buf, 0, hin0)
        self._res('mid.block_2', self.mid.block_2, m2, h_run, cond_all)
        # ---- up path ----
        j = 0
        for i_level in reversed(range(self.num_resolutions)):
            u = self.up[i_level]
            for i_block in range(self.num_res_blocks + 1):
                buf, hin, sc = cat_bufs[j]
                blk = u.block[i_block]
                last_in_level = i_block == self.num_res_blocks
                # where does this block's output go?  into the next concat buffer's first slice, unless an upsample or the end follows
                if not last_in_level:
                    nbuf, nhin, _ = cat_bufs[j + 1]
                    tgt = View(nbuf, 0, nhin)
                else:
                    tgt = View(self._buf('uo.%d' % i_level, (B, res, res, blk.out_channels)))
                if len(u.attn) > 0:
                    tmp = View(self._buf('utmp.%d.%d' % (res, blk.out_channels), (B, res, res, blk.out_channels)))
                    self._res('up.%d.block.%d' % (i_level, i_block), blk, View(buf), tmp, cond_all)
                    self._attn('up.%d.attn.%d' % (i_level, i_block), u.attn[i_block], tmp, tgt)
                else:
                    self._res('up.%d.block.%d' % (i_level, i_block), blk, View(buf), tgt, cond_all)
                h_run = tgt
                j += 1
            if i_level != 0:
                c = h_run.C
                upb = self._buf('ups.%d' % i_level, (B, 2 * res, 2 * res, c))
                call('cd_upsample_nearest2x', C.c_void_p(h_run.addr()), h_run.ld, B, res, res, c, ptr(upb), c, stream())
                res *= 2
                nbuf, nhin, _ = cat_bufs[j]
                tgt = View(nbuf, 0, nhin)
                if u.upsample.with_conv:
                    self._conv(ops.make_conv_desc([(View(upb), T3, P['up.%d.us' % i_level], False)], tgt, (B, res, res), Cout=c,
                                                  bias=u.upsample.conv.bias))
                else:
                    raise NotImplementedError("resamp_with_conv=False is not used by any reference driver")
                h_run = tgt
        # ---- end ----
        c = h_run.C
        no = self._buf('no', (B, res, res, c))
        self._gn(h_run, self.norm_out, View(no), True)
        oc = self.out_ch
        old = oc if oc % 4 == 0 else (oc + 3) // 4 * 4
        ob = self._buf('ob', (B, res, res, old))
        self._conv(ops.make_conv_desc([(View(no), T3, P['conv_out'], False)], View(ob, 0, oc), (B, res, res), Cout=oc, bias=self.conv_out.bias))
        out = torch.empty(B, oc, res, res, device=x.device, dtype=torch.float32)
        call('cd_nhwc_to_nchw', ptr(ob), old, B, res, res, oc, ptr(out), stream())
        return out
