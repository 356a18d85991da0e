"""Training path of the DDPM-style `Model` (Model2.py:191-332, "M2"): forward that keeps what the backward needs, and the
backward schedule, on the same sm_90a kernels as the ConvNeXt Unet (tap-list convolutions for every dense conv and for the
four batched matmuls of the AttnBlock backward; model2_bwd.cu for GroupNorm / softmax / upsample / dropout).

STATUS: tests/test_model2_train_gpu.py compares every parameter
gradient with the reference (tests/golden/model2_grads_small.npz) on the fp32 and the tensor-core path, checks the dropout mask
consistency and one Trainer step.

Gradient routing: every activation that the forward writes into a (slice of a) buffer has a gradient buffer of the same shape;
consumers ADD into it (dense data-gradient convolutions accumulate through their `resid` input, the rest through cd_add) and the
producer reads it once all consumers ran -- the reverse of the forward order guarantees that.

Only parameters with requires_grad get a gradient (the weight-gradient launches of frozen ones are skipped); the gradient of the
input x is formed on request, through the data gradient of conv_in.
"""
import ctypes as C
import os
import torch

from . import ops
from .ops import View, CONV_TC, CONV_SIMT
from ._lib import call, ptr, stream
from .engine_bwd import flat_offsets
from .autograd import check_first_order, trainable_names, once_differentiable
from .model2 import T1, T3, TDOWN
from .graphs import GraphedForward

NULL = C.c_void_p(0)
T3D = ops.taps_conv_dgrad(3, 1)


def enabled():
    return True


def taps_down_dgrad(py, px):
    """data gradient of F.pad(0,1,0,1) + Conv2d(3, stride 2, padding 0) (M2:66-70) for the input parity class (iy%2, ix%2) ==
    (py, px): din[2g+p] = sum_k dout[g + d] W[k] with d = (p - k)/2 for the kernel positions k of the same parity as p."""
    ys = [(0, 0), (2, -1)] if py == 0 else [(1, 0)]
    xs = [(0, 0), (2, -1)] if px == 0 else [(1, 0)]
    return [(ky, kx, dy, dx) for (ky, dy) in ys for (kx, dx) in xs]


class ModelEngine(GraphedForward):
    """what Trainer / FusedAdamEMA need from a network: flat parameter and gradient buffers with 16-byte aligned slices; and the
    CUDA-graph replay of the inference forward."""

    def __init__(self, model):
        self.model = model
        self.flat_grad = self.flat_param = None
        self.G = {}
        self._init_graphs(model, model._forward, model._prepare)

    @property
    def dev(self):
        return self.model.conv_in.weight.device

    def _setup_grads(self):
        if self.flat_grad is not None:
            return
        params = list(self.model.named_parameters())
        self._offsets, total = flat_offsets([(n, p.numel()) for n, p in params])
        self.flat_grad = torch.zeros(total, device=self.dev, dtype=torch.float32)
        for n, p in params:
            off, k = self._offsets[n]
            self.G[n] = self.flat_grad[off:off + k].view_as(p)

    def flatten_params(self):
        self._setup_grads()
        if self.flat_param is not None:
            return
        self.flat_param = torch.zeros_like(self.flat_grad)
        with torch.no_grad():
            for n, p in self.model.named_parameters():
                off, k = self._offsets[n]
                v = self.flat_param[off:off + k].view_as(p)
                v.copy_(p.data)
                p.data = v
        self.drop_graphs()                      # they address the old parameter storage
        self.mark_weights_dirty()

    def attach_grads(self):
        """.grad of every trainable parameter = its view of the flat buffer; frozen parameters keep theirs (None)"""
        self._setup_grads()
        for n, p in self.model.named_parameters():
            if not p.requires_grad:
                continue
            g = self.G[n]
            if p.grad is None or p.grad.data_ptr() != g.data_ptr():
                g.zero_()
                p.grad = g

    def mark_weights_dirty(self):
        # the fused Adam / EMA kernels write through raw pointers (p._version does not move): drop both pack generations
        self.model._version = None
        self.model._bwd_version = None

    def param_list(self):
        return list(self.model.parameters())

    def prepare_training_weights(self):
        """refill the packed operands of the training forward and backward when a parameter changed (before each replay of a
        captured training step, whose launches read them)"""
        prepare_bwd(self.model)


class ModelFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, x, t, *params):
        save = {}
        out = forward_train(model, x, t, save)
        ctx.model, ctx.save, ctx.nparams = model, save, len(params)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        check_first_order(dout, "Model backward")
        eng = ctx.model.engine
        eng.attach_grads()
        need_dx = ctx.needs_input_grad[1]
        dx = backward(ctx.model, ctx.save, dout, need_dx=need_dx,
                      trainable=trainable_names(ctx.model.named_parameters(), ctx.needs_input_grad))
        ctx.save = None
        return (None, dx if need_dx else None, None) + (None,) * ctx.nparams


# ---------------------------------------------------------------------------------------------------------------------
# packed data-gradient operands
# ---------------------------------------------------------------------------------------------------------------------
def prepare_bwd(m):
    m._prepare()
    ver = m._version
    if getattr(m, '_bwd_version', None) == ver:
        return
    P = m._packed
    pk = lambda key, w, taps: P.__setitem__(key, ops.pack_weight(w, taps, mode=1, round_tf32=False, out=P.get(key)))
    with torch.no_grad():
        pk('conv_out.T', m.conv_out.weight, T3D)
        for name, b in m._resblocks():
            pk(name + '.c1T', b.conv1.weight, T3D)
            pk(name + '.c2T', b.conv2.weight, T3D)
            if hasattr(b, 'nin_shortcut'):
                pk(name + '.scT', b.nin_shortcut.weight, T1)
            elif hasattr(b, 'conv_shortcut'):
                pk(name + '.scT', b.conv_shortcut.weight, T3D)
        for name, a in m._attns():
            for leaf in ('q', 'k', 'v', 'proj_out'):
                pk(name + '.' + leaf + 'T', getattr(a, leaf).weight, T1)
        for i, d in enumerate(m.down):
            if hasattr(d, 'downsample') and d.downsample.with_conv:
                for py in (0, 1):
                    for px in (0, 1):
                        pk('down.%d.dsT.%d%d' % (i, py, px), d.downsample.conv.weight, taps_down_dgrad(py, px))
        for i, u in enumerate(m.up):
            if hasattr(u, 'upsample') and u.upsample.with_conv:
                pk('up.%d.usT' % i, u.upsample.conv.weight, T3D)
    m._bwd_version = ver


# ---------------------------------------------------------------------------------------------------------------------
# small helpers
# ---------------------------------------------------------------------------------------------------------------------
def _zeros_like_view(m, key, v):
    t = m._buf(key, (v.B, v.H, v.W, v.C))
    t.zero_()
    return View(t)


def _add_into(tgt, src):
    """tgt += src (NHWC views of equal shape)"""
    call('cd_add', C.c_void_p(tgt.addr()), tgt.ld, C.c_void_p(src.addr()), src.ld, C.c_void_p(tgt.addr()), tgt.ld,
         C.c_int64(tgt.B * tgt.H * tgt.W), tgt.C, stream())


def _colsum(v, out):
    call('cd_colsum', C.c_void_p(v.addr()), v.ld, C.c_int64(v.B * v.H * v.W), v.C, ptr(out), stream())


def _wgrad(m, key, src, taps, Cout, grid, dout, wgrad_param, bias_param, *, stride=1):
    """accumulate the weight (and bias) gradient of one tap-list convolution into reference-layout (OIHW) gradients; a None
    gradient is a frozen parameter"""
    if wgrad_param is None:
        if bias_param is not None:
            _colsum(dout, bias_param)
        return
    nt = len(taps)
    if nt == 1:
        dwp = wgrad_param                                   # 1x1: packed layout == OIHW layout
    else:
        dwp = m._buf('dwp.' + key, (nt, Cout, src.C))
        dwp.zero_()
    d = ops.make_conv_desc([(src, taps, dwp, False)], dout, grid, stride=stride, Cout=Cout)
    ops.conv_wgrad(d, dout, dwp, bias_param, impl=m.conv_impl)
    if nt != 1:
        ops.unpack_wgrad(dwp, taps, wgrad_param, accumulate=True)


def _dgrad_into(m, dyv, taps, packedT, tgt, grid, Cin, accumulate):
    """tgt (+)= data gradient of a stride-1 convolution: a tap-list convolution of dY with flipped taps / transposed weights"""
    d = ops.make_conv_desc([(dyv, taps, packedT, False)], tgt, grid, Cout=Cin, resid=tgt if accumulate else None)
    impl_tc = dyv.C % 32 == 0
    ops.conv_fwd(d, m.conv_impl if impl_tc else CONV_SIMT)


def _gn_bwd(m, xv, norm, swish, dyv, dxv, G, gname, cond=None, dcond=None):
    B, H, W = xv.B, xv.H, xv.W
    condp = C.c_void_p(cond) if cond is not None else NULL
    dcondp = C.c_void_p(dcond) if dcond is not None else NULL
    dg, db = G.get(gname + '.weight'), G.get(gname + '.bias')
    if (dg is None) != (db is None):            # half-frozen pair: a scratch stand-in for the frozen one
        scratch = m._buf('g.scratch.gn', (xv.C,))
        dg, db = (scratch if dg is None else dg), (scratch if db is None else db)
    call('cd_groupnorm_bwd', C.c_void_p(xv.addr()), xv.ld, B, C.c_int64(H * W), xv.C, norm.num_groups, condp, m._sumC,
         ptr(norm.weight), ptr(norm.bias), C.c_float(norm.eps), int(swish), C.c_void_p(dyv.addr()), dyv.ld,
         C.c_void_p(dxv.addr()), dxv.ld, ptr(dg), ptr(db), dcondp, m._sumC, stream())


# ---------------------------------------------------------------------------------------------------------------------
# forward (training mode): same schedule as Model.forward, every block keeps its own buffers
# ---------------------------------------------------------------------------------------------------------------------
def _res_fwd(m, name, b, xv, outv, cond_all, save):
    B, H, W = xv.B, xv.H, xv.W
    P = m._packed
    cin, cout = b.in_channels, b.out_channels
    n1 = View(m._buf('t.n1.' + name, (B, H, W, cin)))
    m._gn(xv, b.norm1, n1, True)
    h1 = View(m._buf('t.h1.' + name, (B, H, W, cout)))
    m._conv(ops.make_conv_desc([(n1, T3, P[name + '.c1'], False)], h1, (B, H, W), Cout=cout, bias=b.conv1.bias))
    n2 = View(m._buf('t.n2.' + name, (B, H, W, cout)))
    m._gn(h1, b.norm2, n2, True, cond=cond_all.data_ptr() + 4 * b._cond_off)
    seed = None
    p = float(b.dropout.p)
    if m.training and p > 0.0:
        from .train_graph import recording
        draws = recording()
        if draws is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())       # host RNG (torch.manual_seed controls it); mask = f(seed, element index)
            call('cd_dropout', C.c_void_p(n2.addr()), n2.ld, C.c_int64(B * H * W), cout, C.c_float(p), C.c_uint64(seed),
                 C.c_void_p(n2.addr()), n2.ld, stream())
        else:
            # captured training step: the same host draw is made before every replay and staged in this device slot
            seed = draws.dropout_seed()
            call('cd_dropout_seed_dev', C.c_void_p(n2.addr()), n2.ld, C.c_int64(B * H * W), cout, C.c_float(p), ptr(seed),
                 C.c_void_p(n2.addr()), n2.ld, stream())
    if cin != cout:
        taps_sc = T1 if hasattr(b, 'nin_shortcut') else T3
        d = ops.make_conv_desc([(n2, T3, P[name + '.c2'], False), (xv, taps_sc, P[name + '.sc'], False)], outv, (B, H, W),
                               Cout=cout, bias=P[name + '.b2s'])
    else:
        d = ops.make_conv_desc([(n2, T3, P[name + '.c2'], False)], outv, (B, H, W), Cout=cout, bias=b.conv2.bias, resid=xv)
    m._conv(d)
    save[name] = dict(x=xv, n1=n1, h1=h1, n2=n2, seed=seed, p=p)


def _res_bwd(m, name, b, save, dyv, dx_acc, dcond_all, cond_all, G):
    """dyv: gradient of the block output (read only); dx_acc: gradient buffer of the block input (accumulated into);
    G: gradient views of the trainable parameters"""
    sv = save[name]
    xv, n1, h1, n2 = sv['x'], sv['n1'], sv['h1'], sv['n2']
    B, H, W = xv.B, xv.H, xv.W
    grid = (B, H, W)
    P = m._packed
    cin, cout = b.in_channels, b.out_channels
    # ---- conv2 (+ shortcut): weights, biases
    sc = 'nin_shortcut' if hasattr(b, 'nin_shortcut') else ('conv_shortcut' if hasattr(b, 'conv_shortcut') else None)
    _wgrad(m, name + '.c2', n2, T3, cout, grid, dyv, G.get(name + '.conv2.weight'), G.get(name + '.conv2.bias'))
    if cin != cout:
        taps_sc = T1 if sc == 'nin_shortcut' else T3
        _wgrad(m, name + '.sc', xv, taps_sc, cout, grid, dyv, G.get(name + '.%s.weight' % sc), G.get(name + '.%s.bias' % sc))
    # ---- through conv2 -> dropout -> swish(GroupNorm2(h1 + cond))
    dn2 = View(m._buf('g.n2.%dx%dx%d' % (H, W, cout), (B, H, W, cout)))
    _dgrad_into(m, dyv, T3D, P[name + '.c2T'], dn2, grid, cout, False)
    if torch.is_tensor(sv['seed']):
        call('cd_dropout_seed_dev', C.c_void_p(dn2.addr()), dn2.ld, C.c_int64(B * H * W), cout, C.c_float(sv['p']), ptr(sv['seed']),
             C.c_void_p(dn2.addr()), dn2.ld, stream())
    elif sv['seed'] is not None:
        call('cd_dropout', C.c_void_p(dn2.addr()), dn2.ld, C.c_int64(B * H * W), cout, C.c_float(sv['p']), C.c_uint64(sv['seed']),
             C.c_void_p(dn2.addr()), dn2.ld, stream())
    dh1 = View(m._buf('g.h1.%dx%dx%d' % (H, W, cout), (B, H, W, cout)))
    _gn_bwd(m, h1, b.norm2, True, dn2, dh1, G, name + '.norm2', cond=cond_all.data_ptr() + 4 * b._cond_off,
            dcond=dcond_all.data_ptr() + 4 * b._cond_off if dcond_all is not None else None)
    # ---- conv1
    _wgrad(m, name + '.c1', n1, T3, cout, grid, dh1, G.get(name + '.conv1.weight'), G.get(name + '.conv1.bias'))
    dn1 = View(m._buf('g.n1.%dx%dx%d' % (H, W, cin), (B, H, W, cin)))
    _dgrad_into(m, dh1, T3D, P[name + '.c1T'], dn1, grid, cin, False)
    dxg = View(m._buf('g.xg.%dx%dx%d' % (H, W, cin), (B, H, W, cin)))
    _gn_bwd(m, xv, b.norm1, True, dn1, dxg, G, name + '.norm1')
    _add_into(dx_acc, dxg)
    # ---- skip path: identity or shortcut convolution
    if cin != cout:
        _dgrad_into(m, dyv, T1 if sc == 'nin_shortcut' else T3D, P[name + '.scT'], dx_acc, grid, cin, True)
    else:
        _add_into(dx_acc, dyv)


def _attn_fwd(m, name, a, xv, outv, save):
    B, H, W = xv.B, xv.H, xv.W
    n, c = H * W, a.in_channels
    P = m._packed
    hn = View(m._buf('t.an.' + name, (B, H, W, c)))
    m._gn(xv, a.norm, hn, False)
    q = View(m._buf('t.aq.' + name, (B, H, W, c))); k = View(m._buf('t.ak.' + name, (B, H, W, c))); v = View(m._buf('t.av.' + name, (B, H, W, c)))
    for t, leaf in ((q, 'q'), (k, 'k'), (v, 'v')):
        m._conv(ops.make_conv_desc([(hn, T1, P[name + '.' + leaf], False)], t, (B, H, W), Cout=c, bias=getattr(a, leaf).bias))
    tc = n >= 128 and n % 32 == 0
    s = View(m._buf('t.as.' + name, (B, H, W, n)))
    m._conv(ops.make_conv_desc([(q, T1, k.t, True)], s, (B, H, W), Cout=n), False)
    call('cd_softmax_rows', C.c_void_p(s.addr()), n, C.c_int64(B * n), n, C.c_float(int(c) ** (-0.5)), stream())
    vt = m._buf('avt.%dx%d' % (n, c), (B, c, n))
    call('cd_transpose_batched', C.c_void_p(v.addr()), c, B, n, c, ptr(vt), stream())
    ho = View(m._buf('t.ah.' + name, (B, H, W, c)))
    m._conv(ops.make_conv_desc([(s, T1, vt, True)], ho, (B, H, W), Cout=c), tc)
    m._conv(ops.make_conv_desc([(ho, T1, P[name + '.proj_out'], False)], outv, (B, H, W), Cout=c, bias=a.proj_out.bias, resid=xv))
    save[name] = dict(x=xv, hn=hn, q=q, k=k, v=v, s=s, ho=ho)


def _attn_bwd(m, name, a, save, dyv, dx_acc, G):
    sv = save[name]
    xv, hn, q, k, v, s, ho = sv['x'], sv['hn'], sv['q'], sv['k'], sv['v'], sv['s'], sv['ho']
    B, H, W = xv.B, xv.H, xv.W
    n, c = H * W, a.in_channels
    grid = (B, H, W)
    P = m._packed
    scale = int(c) ** (-0.5)
    # proj_out
    _wgrad(m, name + '.po', ho, T1, c, grid, dyv, G.get(name + '.proj_out.weight'), G.get(name + '.proj_out.bias'))
    dho = View(m._buf('g.ah.%dx%d' % (n, c), (B, H, W, c)))
    _dgrad_into(m, dyv, T1, P[name + '.proj_outT'], dho, grid, c, False)
    # h_ = w_ v  (w_ = softmax weights s[b,i,j], M2:176-181)
    #   dv[b,j,c] = sum_i s[b,i,j] dho[b,i,c]: a per-batch weight gradient with "dY" = s and "X" = dho
    dv = m._buf('g.av.%dx%d' % (n, c), (B, 1, n, c)); dv.zero_()
    d = ops.make_conv_desc([(dho, T1, dv, True)], s, grid, Cout=n)
    ops.conv_wgrad(d, s, dv, None, impl=m.conv_impl)
    #   ds[b,i,j] = sum_c dho[b,i,c] v[b,j,c]: per-batch 1x1 convolution whose weight slab is v itself ([n][c])
    ds = View(m._buf('g.as.%d' % n, (B, H, W, n)))
    ops.conv_fwd(ops.make_conv_desc([(dho, T1, v.t, True)], ds, grid, Cout=n), CONV_SIMT)
    call('cd_softmax_bwd_rows', C.c_void_p(s.addr()), C.c_void_p(ds.addr()), n, C.c_int64(B * n), n, C.c_float(scale), stream())
    # w_ = q k^T (M2:169-172): dq[b,i,c] = sum_j ds[b,i,j] k[b,j,c];  dk[b,j,c] = sum_i ds[b,i,j] q[b,i,c]
    kt = m._buf('akt.%dx%d' % (n, c), (B, c, n))
    call('cd_transpose_batched', C.c_void_p(k.addr()), c, B, n, c, ptr(kt), stream())
    dq = View(m._buf('g.aq.%dx%d' % (n, c), (B, H, W, c)))
    ops.conv_fwd(ops.make_conv_desc([(ds, T1, kt, True)], dq, grid, Cout=c), CONV_SIMT)
    dk = m._buf('g.ak.%dx%d' % (n, c), (B, 1, n, c)); dk.zero_()
    d = ops.make_conv_desc([(q, T1, dk, True)], ds, grid, Cout=n)
    ops.conv_wgrad(d, ds, dk, None, impl=CONV_SIMT)
    dkv = View(dk.view(B, H, W, c)); dvv = View(dv.view(B, H, W, c))
    # q / k / v projections
    dhn = View(m._buf('g.an.%dx%d' % (n, c), (B, H, W, c)))
    first = True
    for leaf, g in (('q', dq), ('k', dkv), ('v', dvv)):
        _wgrad(m, name + '.' + leaf, hn, T1, c, grid, g, G.get(name + '.%s.weight' % leaf), G.get(name + '.%s.bias' % leaf))
        _dgrad_into(m, g, T1, P[name + '.' + leaf + 'T'], dhn, grid, c, not first)
        first = False
    dxg = View(m._buf('g.axg.%dx%d' % (n, c), (B, H, W, c)))
    _gn_bwd(m, xv, a.norm, False, dhn, dxg, G, name + '.norm')
    _add_into(dx_acc, dxg)
    _add_into(dx_acc, dyv)                                   # residual x + h_


def forward_train(m, x, t, save):
    assert x.is_cuda and x.shape[2] == x.shape[3] == m.resolution
    prepare_bwd(m)
    P = m._packed
    B, Cin, H, W = x.shape
    x = x.contiguous().float()
    t = t.to(device=x.device, dtype=torch.int64).contiguous()
    d0, d1 = m.temb.dense[0], m.temb.dense[1]
    # ---- time embedding, every stage kept (M2:293-299): emb -> dense0 -> swish -> dense1 -> swish -> per-block temb_proj rows
    emb = m._buf('t.emb', (B, m.ch)); h0 = m._buf('t.h0', (B, m.temb_ch)); a0 = m._buf('t.a0', (B, m.temb_ch))
    temb = m._buf('t.temb', (B, m.temb_ch)); st = m._buf('t.st', (B, m.temb_ch))
    cond_all = m._buf('cond', (B, m._sumC))
    call('cd_timestep_embedding', ptr(t), B, m.ch, ptr(emb), stream())
    call('cd_linear_fwd', ptr(emb), m.ch, ptr(d0.weight), ptr(d0.bias), B, m.temb_ch, ptr(h0), stream())
    call('cd_swish', NULL, ptr(h0), C.c_int64(B * m.temb_ch), NULL, ptr(a0), stream())
    call('cd_linear_fwd', ptr(a0), m.temb_ch, ptr(d1.weight), ptr(d1.bias), B, m.temb_ch, ptr(temb), stream())
    call('cd_swish', NULL, ptr(temb), C.c_int64(B * m.temb_ch), NULL, ptr(st), stream())
    call('cd_linear_fwd', ptr(st), m.temb_ch, ptr(P['cond.w']), ptr(P['cond.b']), B, m._sumC, ptr(cond_all), stream())
    ld0 = Cin if Cin % 4 == 0 else 4
    x0 = m._buf('x0', (B, H, W, ld0))
    call('cd_nchw_to_nhwc', ptr(x), B, Cin, H, W, ptr(x0), ld0, stream())

    plan = m._plan(B, H)
    cat_bufs, skip_view = plan['cat_bufs'], plan['skip_view']
    ops_log = []                                             # forward order of (kind, args) for the backward walk
    hv = skip_view(0)
    m._conv(ops.make_conv_desc([(View(x0, 0, Cin), T3, P['conv_in'], False)], hv, (B, H, W), Cout=m.ch, bias=m.conv_in.bias), False)
    ops_log.append(('conv_in', View(x0, 0, Cin), hv))
    sk, res = 0, H
    for i_level in range(m.num_resolutions):
        d = m.down[i_level]
        for i_block, b in enumerate(d.block):
            sk += 1
            tgt = skip_view(sk)
            rname = 'down.%d.block.%d' % (i_level, i_block)
            if len(d.attn) > 0:
                tmp = View(m._buf('t.dtmp.' + rname, (B, res, res, b.out_channels)))
                _res_fwd(m, rname, b, hv, tmp, cond_all, save)
                ops_log.append(('res', rname, b, hv, tmp))
                aname = 'down.%d.attn.%d' % (i_level, i_block)
                _attn_fwd(m, aname, d.attn[i_block], tmp, tgt, save)
                ops_log.append(('attn', aname, d.attn[i_block], tmp, tgt))
            else:
                _res_fwd(m, rname, b, hv, tgt, cond_all, save)
                ops_log.append(('res', rname, b, hv, tgt))
            hv = tgt
        if i_level != m.num_resolutions - 1:
            sk += 1
            tgt = skip_view(sk)
            m._conv(ops.make_conv_desc([(hv, TDOWN, P['down.%d.ds' % i_level], False)], tgt, (B, res // 2, res // 2), stride=2,
                                       Cout=hv.C, bias=d.downsample.conv.bias))
            ops_log.append(('down', i_level, hv, tgt))
            res //= 2
            hv = tgt
    cm = hv.C
    m1 = View(m._buf('t.m1', (B, res, res, cm))); m2 = View(m._buf('t.m2', (B, res, res, cm)))
    _res_fwd(m, 'mid.block_1', m.mid.block_1, hv, m1, cond_all, save); ops_log.append(('res', 'mid.block_1', m.mid.block_1, hv, m1))
    _attn_fwd(m, 'mid.attn_1', m.mid.attn_1, m1, m2, save); ops_log.append(('attn', 'mid.attn_1', m.mid.attn_1, m1, m2))
    first_buf, hin0, _ = cat_bufs[0]
    h_run = View(first_buf, 0, hin0)
    _res_fwd(m, 'mid.block_2', m.mid.block_2, m2, h_run, cond_all, save); ops_log.append(('res', 'mid.block_2', m.mid.block_2, m2, h_run))
    j = 0
    for i_level in reversed(range(m.num_resolutions)):
        u = m.up[i_level]
        for i_block in range(m.num_res_blocks + 1):
            buf, hin, sc = cat_bufs[j]
            blk = u.block[i_block]
            last_in_level = i_block == m.num_res_blocks
            if not last_in_level:
                nbuf, nhin, _ = cat_bufs[j + 1]
                tgt = View(nbuf, 0, nhin)
            else:
                tgt = View(m._buf('t.uo.%d' % i_level, (B, res, res, blk.out_channels)))
            rname = 'up.%d.block.%d' % (i_level, i_block)
            if len(u.attn) > 0:
                tmp = View(m._buf('t.utmp.' + rname, (B, res, res, blk.out_channels)))
                _res_fwd(m, rname, blk, View(buf), tmp, cond_all, save); ops_log.append(('res', rname, blk, View(buf), tmp))
                aname = 'up.%d.attn.%d' % (i_level, i_block)
                _attn_fwd(m, aname, u.attn[i_block], tmp, tgt, save); ops_log.append(('attn', aname, u.attn[i_block], tmp, tgt))
            else:
                _res_fwd(m, rname, blk, View(buf), tgt, cond_all, save); ops_log.append(('res', rname, blk, View(buf), tgt))
            h_run = tgt
            j += 1
        if i_level != 0:
            c = h_run.C
            upb = View(m._buf('t.ups.%d' % i_level, (B, 2 * res, 2 * res, c)))
            call('cd_upsample_nearest2x', C.c_void_p(h_run.addr()), h_run.ld, B, res, res, c, C.c_void_p(upb.addr()), c, stream())
            res *= 2
            nbuf, nhin, _ = cat_bufs[j]
            tgt = View(nbuf, 0, nhin)
            m._conv(ops.make_conv_desc([(upb, T3, P['up.%d.us' % i_level], False)], tgt, (B, res, res), Cout=c, bias=u.upsample.conv.bias))
            ops_log.append(('up', i_level, h_run, upb, tgt))
            h_run = tgt
    c = h_run.C
    no = View(m._buf('t.no', (B, res, res, c)))
    m._gn(h_run, m.norm_out, no, True)
    oc = m.out_ch
    old = oc if oc % 4 == 0 else (oc + 3) // 4 * 4
    ob = m._buf('ob', (B, res, res, old))
    m._conv(ops.make_conv_desc([(no, T3, P['conv_out'], False)], View(ob, 0, oc), (B, res, res), Cout=oc, bias=m.conv_out.bias))
    out = torch.empty(B, oc, res, res, device=x.device, dtype=torch.float32)
    call('cd_nhwc_to_nchw', ptr(ob), old, B, res, res, oc, ptr(out), stream())
    save['__'] = dict(ops=ops_log, emb=emb, h0=h0, a0=a0, temb=temb, st=st, cond_all=cond_all, last=h_run, no=no, B=B, H=H)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------
def backward(m, save, dout, need_dx=False, trainable=None):
    """dout: NCHW gradient of the output.  Accumulates the gradients of the parameters named in `trainable` (None: all) into the
    flat buffer; need_dx: returns the NCHW gradient of the input x, else None."""
    top = save['__']
    B, H = top['B'], top['H']
    P = m._packed
    G = m.engine.G
    if trainable is not None:
        trainable = set(trainable)
        G = {n: g for n, g in G.items() if n in trainable}
    time_train = any(n.startswith('temb.') or '.temb_proj.' in n for n in G)
    dout = dout.contiguous().float()
    oc = m.out_ch
    old = oc if oc % 4 == 0 else (oc + 3) // 4 * 4
    dob = m._buf('g.ob', (B, H, H, old))
    call('cd_nchw_to_nhwc', ptr(dout), B, oc, H, H, ptr(dob), old, stream())       # zero-fills the padding channel
    dyv = View(dob, 0, oc)
    grads = {}                                               # id of the forward buffer slice -> gradient View

    def gview(v):
        """gradient buffer of the tensor behind the forward view v (same base tensor -> same gradient tensor, same slice)"""
        key = v.t.data_ptr()
        if key not in grads:
            t = m._buf('g@%d' % len(grads) + 'x'.join(str(s) for s in v.t.shape), tuple(v.t.shape))
            t.zero_()
            grads[key] = t
        return View(grads[key], v.c0, v.C)

    # ---- conv_out and norm_out
    last, no = top['last'], top['no']
    res = last.H
    _wgrad(m, 'conv_out', no, T3, oc, (B, res, res), dyv, G.get('conv_out.weight'), G.get('conv_out.bias'))
    dno = View(m._buf('g.no', (B, res, res, no.C)))
    ops.conv_fwd(ops.make_conv_desc([(dyv, T3D, P['conv_out.T'], False)], dno, (B, res, res), Cout=no.C), CONV_SIMT)
    _gn_bwd(m, last, m.norm_out, True, dno, gview(last), G, 'norm_out')          # first and only writer of d(last)

    dcond_all = None
    if time_train:                                           # conditioning gradient: only the time path consumes it
        dcond_all = m._buf('g.cond', (B, m._sumC)); dcond_all.zero_()
    cond_all = top['cond_all']
    for op in reversed(top['ops']):
        kind = op[0]
        if kind == 'res':
            _, name, b, xin, xout = op
            _res_bwd(m, name, b, save, gview(xout), gview(xin), dcond_all, cond_all, G)
        elif kind == 'attn':
            _, name, a, xin, xout = op
            _attn_bwd(m, name, a, save, gview(xout), gview(xin), G)
        elif kind == 'up':
            _, i_level, hin, upb, tgt = op
            u = m.up[i_level]
            c, r2 = hin.C, upb.H
            dy = gview(tgt)
            _wgrad(m, 'up.%d.us' % i_level, upb, T3, c, (B, r2, r2), dy, G.get('up.%d.upsample.conv.weight' % i_level),
                   G.get('up.%d.upsample.conv.bias' % i_level))
            dup = View(m._buf('g.ups.%d' % i_level, (B, r2, r2, c)))
            _dgrad_into(m, dy, T3D, P['up.%d.usT' % i_level], dup, (B, r2, r2), c, False)
            dsm = View(m._buf('g.upsm.%d' % i_level, (B, r2 // 2, r2 // 2, c)))
            call('cd_upsample_nearest2x_bwd', C.c_void_p(dup.addr()), dup.ld, B, r2 // 2, r2 // 2, c, C.c_void_p(dsm.addr()), dsm.ld, stream())
            _add_into(gview(hin), dsm)
        elif kind == 'down':
            _, i_level, hin, tgt = op
            c, r = hin.C, hin.H
            dy = gview(tgt)
            _wgrad(m, 'down.%d.ds' % i_level, hin, TDOWN, c, (B, r // 2, r // 2), dy, G.get('down.%d.downsample.conv.weight' % i_level),
                   G.get('down.%d.downsample.conv.bias' % i_level), stride=2)
            dx = gview(hin)
            for py in (0, 1):
                for px in (0, 1):
                    d = ops.make_conv_desc([(dy, taps_down_dgrad(py, px), P['down.%d.dsT.%d%d' % (i_level, py, px)], False)], dx,
                                           (B, r // 2, r // 2), Cout=c, out_map=(2, 2, py, px), resid=dx)
                    ops.conv_fwd(d, m.conv_impl if c % 32 == 0 else CONV_SIMT)
        elif kind == 'conv_in':
            _, xin, hv = op
            _wgrad(m, 'conv_in', xin, T3, m.ch, (B, H, H), gview(hv), G.get('conv_in.weight'), G.get('conv_in.bias'))
            if need_dx:
                # data gradient of conv_in: ch -> in_channels (rows padded to 4 floats), then NCHW.  Its operand is packed
                # here, only by the backwards that need it, so the training step keeps its launches
                with torch.no_grad():
                    P['conv_in.T'] = ops.pack_weight(m.conv_in.weight, T3D, mode=1, round_tf32=False, out=P.get('conv_in.T'))
                dxb = View(m._buf('g.x0', (B, H, H, xin.ld)), 0, xin.C)
                _dgrad_into(m, gview(hv), T3D, P['conv_in.T'], dxb, (B, H, H), xin.C, False)

    if time_train:
        _time_bwd(m, top, G, dcond_all)
    if not need_dx:
        return None
    dx = torch.empty((B, dxb.C, H, H), device=dout.device, dtype=torch.float32)
    call('cd_nhwc_to_nchw_add', C.c_void_p(dxb.addr()), dxb.ld, B, H, H, dxb.C, NULL, ptr(dx), stream())
    return dx


def _time_bwd(m, top, G, dcond_all):
    """time embedding (M2:293-299) and the per-block temb_proj rows (M2:121); frozen parameters are skipped"""
    B = top['B']
    P = m._packed
    d0, d1 = m.temb.dense[0], m.temb.dense[1]
    st, temb, a0, h0, emb = top['st'], top['temb'], top['a0'], top['h0'], top['emb']
    tch = m.temb_ch
    for name, b in m._resblocks():
        off, co = b._cond_off, b.out_channels
        gw, gb = G.get(name + '.temb_proj.weight'), G.get(name + '.temb_proj.bias')
        # dW[c][k] += sum_b dcond[b][off+c] * st[b][k]
        if gw is not None:
            call('cd_small_gemm', C.c_void_p(dcond_all.data_ptr() + 4 * off), m._sumC, 1, ptr(st), tch, 0,
                 ptr(gw), tch, co, tch, B, 1, stream())
        if gb is not None:
            call('cd_colsum', C.c_void_p(dcond_all.data_ptr() + 4 * off), m._sumC, C.c_int64(B), co, ptr(gb), stream())
    g0w, g0b, g1w, g1b = (G.get('temb.dense.%s' % n) for n in ('0.weight', '0.bias', '1.weight', '1.bias'))
    if g0w is None and g0b is None and g1w is None and g1b is None:
        return
    dst = m._buf('g.dst', (B, tch))
    call('cd_small_gemm', ptr(dcond_all), m._sumC, 0, ptr(P['cond.w']), tch, 0, ptr(dst), tch, B, tch, m._sumC, 0, stream())
    dtemb = m._buf('g.dtemb', (B, tch))
    call('cd_swish', ptr(dst), ptr(temb), C.c_int64(B * tch), ptr(dtemb), NULL, stream())
    if g1w is not None:
        call('cd_small_gemm', ptr(dtemb), tch, 1, ptr(a0), tch, 0, ptr(g1w), tch, tch, tch, B, 1, stream())
    if g1b is not None:
        call('cd_colsum', ptr(dtemb), tch, C.c_int64(B), tch, ptr(g1b), stream())
    if g0w is None and g0b is None:
        return
    da0 = m._buf('g.da0', (B, tch))
    call('cd_small_gemm', ptr(dtemb), tch, 0, ptr(d1.weight), tch, 0, ptr(da0), tch, B, tch, tch, 0, stream())
    dh0 = m._buf('g.dh0', (B, tch))
    call('cd_swish', ptr(da0), ptr(h0), C.c_int64(B * tch), ptr(dh0), NULL, stream())
    if g0w is not None:
        call('cd_small_gemm', ptr(dh0), tch, 1, ptr(emb), m.ch, 0, ptr(g0w), m.ch, tch, m.ch, B, 1, stream())
    if g0b is not None:
        call('cd_colsum', ptr(dh0), tch, C.c_int64(B), tch, ptr(g0b), stream())
