"""torch.autograd.Function wrappers that put the hand-written sm_90a kernels on the autograd tape.

Activations are NHWC bf16 tensors (N,H,W,C); parameters stay fp32 masters in the reference's layouts
(conv weight OIHW, so checkpoints / optimizers see the reference's tensors) and are re-packed to the
kernels' bf16 OHWI layouts once per parameter version.  Forward AND backward run on libc3d.so:
  conv fwd  -> c3d_conv2d_fwd          dgrad -> c3d_conv2d_fwd with flipped/transposed weights
  wgrad     -> c3d_conv2d_wgrad        BN    -> c3d_bn_finalize / c3d_bn_apply / c3d_bn_bwd
"""
import weakref

import torch

from . import _lib
from . import conv as K
from . import kernels as Kx

# bf16 kernel-layout packs of the fp32 masters, per nn.Parameter: {id: ((version key), weak reference, packs)}
_pack_cache = {}        # conv weights: (fwd, dgrad, stride-2 phase packs or None)
_lin_cache = {}         # linear weights: (chw, fwd, transposed)
_epoch = 0


def invalidate_packed():
    """Call after parameters were updated outside autograd's view (the fused SGD kernel writes through raw
    pointers, so tensor._version does not move)."""
    global _epoch
    _epoch += 1
    _pack_cache.clear()
    _lin_cache.clear()


def _cache_key(w):
    """Only nn.Parameter objects are cached, keyed on the OBJECT (weak reference) + storage + version + optimizer epoch.
    Derived temporaries (the zero-padded stem weight, the fused RPN predictor weight) are leaf tensors under no_grad
    whose storage the caching allocator hands back on the next forward: a data_ptr key would alias them across
    load_state_dict / a second model, so they are packed on every call instead."""
    if not isinstance(w, torch.nn.Parameter):
        return None, None
    return id(w), (w.data_ptr(), w._version, _epoch, tuple(w.shape), tuple(w.stride()))


def _cache_get(cache, w):
    """the packs cached for parameter w, or None when there are none or they are stale"""
    key, ver = _cache_key(w)
    hit = cache.get(key) if key is not None else None
    return hit[2] if hit is not None and hit[0] == ver and hit[1]() is w else None


def _cache_put(cache, w, packs):
    key, ver = _cache_key(w)
    if key is not None:
        cache[key] = (ver, weakref.ref(w), packs)
    return packs


def _packed(w, phases=False):
    """(fwd, dgrad, phase packs) of an fp32 OIHW / channels_last conv master (conv.pack_desc) — the phase sub-kernels of a
    3x3 stride-2 data gradient only when asked for (else None) — produced by ONE pack launch and cached per parameter."""
    hit = _cache_get(_pack_cache, w)
    if hit is None or (phases and hit[2] is None):
        hit = _cache_put(_pack_cache, w, K.pack_conv_weight(w, phases=_phase_layout(w) if phases else None))
    return hit


# ---- all conv weights of a model packed by ONE launch per step (c3d_pack_conv_weights_batched) ----------------------------
_plans = {}


def prepack_model(model):
    """Pack every directly-used conv weight of `model` (forward OHWI pack, rotated data-gradient pack, and the four phase
    sub-kernels of 3x3 / stride-2 layers) with one kernel launch and seed the per-parameter cache, so the layer-by-layer
    `_packed` look-ups of this step are hits.  Output buffers and the descriptor table are built once per model (stable
    addresses: CUDA-graph safe); call at the start of every training step, after the optimizer update."""
    convs = [m for m in model.modules() if isinstance(m, torch.nn.Conv2d) and isinstance(m.weight, torch.nn.Parameter)
             and m.weight.is_cuda and m.weight.shape[1] % 16 == 0 and m.weight.shape[0] % 16 == 0]
    if not convs:
        return 0
    key = tuple((id(m.weight), m.weight.data_ptr(), tuple(m.weight.stride())) for m in convs)
    plan = _plans.get(id(model))
    if plan is None or plan["key"] != key:
        arr = (_lib.PackDesc * len(convs))()
        bufs, start = [], 0
        for i, m in enumerate(convs):
            w = m.weight
            O, I, KH, KW = w.shape
            phases = m.stride[0] == 2 and KH == 3 and KW == 3 and m.padding[0] == 1
            arr[i], packs = K.pack_desc(w, phases=_phase_layout(w) if phases else None)
            arr[i].start = start
            start += w.numel()
            bufs.append((w, packs))
        table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(convs[0].weight.device)
        plan = _plans[id(model)] = {"key": key, "table": table, "bufs": bufs, "total": start, "n": len(convs)}
    _lib.check(_lib.lib().c3d_pack_conv_weights_batched(plan["table"].data_ptr(), plan["n"], plan["total"], _lib.stream()))
    for w, packs in plan["bufs"]:
        _cache_put(_pack_cache, w, packs)
    return plan["n"]


_MERGE_MAX_O = 256


def _merge_phases(I, O):
    """stride-2 3x3 data gradient as ONE 2x2 convolution of dy with 4*I output channels — (row parity, column parity, ci), the
    conv epilogue places the two row halves one dx row apart (c3d.h y_split_*) — instead of four phase convs: 1.78x the
    FLOPs (7 of the 16 taps are zero) but one pass over dy, one launch, full-width tiles."""
    return O <= _MERGE_MAX_O and (2 * I) % 16 == 0 and O % 16 == 0


def _phase_layout(w):
    return "merged" if _merge_phases(w.shape[1], w.shape[0]) else "separate"


def _dgrad(dy, w, stride, pad, in_hw, into=None):
    """dx for y = conv(x, w, stride, pad).  stride 1: conv of dy with the 180-degree-rotated, transposed weights.
    3x3/s2/p1: four phase convs (one per output parity) written straight into the strided positions of dx —
    exactly the algorithmic FLOPs, no zero-stuffed intermediate.  into: an existing gradient buffer of x (dense or a
    channel slice) that the result is ADDED to in the conv epilogue (returned)."""
    KH = w.shape[2]
    acc = into is not None
    if stride == 2 and KH == 3 and pad == 1 and in_hw[0] == 2 * dy.shape[1] and in_hw[1] == 2 * dy.shape[2]:
        N, Ho, Wo, _ = dy.shape
        H, W = in_hw
        dx = into if acc else torch.empty((N, H, W, w.shape[1]), device=dy.device, dtype=dy.dtype)
        packs = _packed(w, phases=True)[2]
        I = w.shape[1]
        if "merged" in packs and dx.stride(2) == I:
            # channel j = (a, b, ci) of dy-pixel (h, w) is dx[2h + a, 2w + b, ci]: in a DENSE dx (b, ci) are 2*I contiguous
            # elements, the a = 1 half sits one dx row (W pixels) further
            K.conv2d_fwd(dy, packs["merged"], stride=1, pad=0, out=dx, out_place=(H * W, 2 * W, 2, 0), out_hw_override=(Ho, Wo),
                         accumulate=acc, split=(2 * I, W * I - 2 * I))
            return dx
        # exact-FLOP phases (wide layers), or the row blocks of the merged weight used one by one (2x2 taps, unused ones zero)
        # when dx is a channel slice of a wider gradient buffer (adjacent pixels are not adjacent in memory there)
        for key, wp in packs.items():
            if key == "merged":
                continue
            a, b = key
            K.conv2d_fwd(dy, wp, stride=1, pad=0, out=dx, out_place=(H * W, 2 * W, 2, a * W + b), out_hw_override=(Ho, Wo),
                         accumulate=acc)
        return dx
    wp = _packed(w)[1]
    if stride == 1:
        return K.conv2d_fwd(dy, wp, stride=1, pad=KH - 1 - pad, out=into, accumulate=acc)
    assert stride == 2
    H, W = in_hw
    z = Kx.zero_stuff2(dy, H, W)
    if KH == 1:                      # 1x1 stride 2: pure scatter + 1x1 conv
        return K.conv2d_fwd(z, wp, stride=1, pad=0, out=into, accumulate=acc)
    return K.conv2d_fwd(z, wp, stride=1, pad=KH - 1 - pad, out=into, accumulate=acc)


def _dgrad_chained(sink, dy, w, stride, pad, in_hw):
    """data gradient of a conv whose input may share its gradient buffer with the input's other consumers"""
    if sink is not None and sink.buf is not None and sink.buf.dtype == dy.dtype:
        _dgrad(dy, w, stride, pad, in_hw, into=sink.buf)
        return None
    return _deliver(sink, _dgrad(dy, w, stride, pad, in_hw))


def _own_grad(p):
    """p's own fp32 .grad (the trainer's flat arena), which a kernel can accumulate into in place, or None"""
    g = p.grad if p.is_leaf else None
    return g if g is not None and g.dtype == torch.float32 and g.shape == p.shape else None


def _wgrad_to_master(x, dy, w, stride, pad):
    """weight gradient in the master (Cout,Cin,KH,KW) layout.  When the parameter already owns a contiguous
    fp32 .grad (the trainer's flat arena) the kernel accumulates straight into it and autograd gets None."""
    g = _own_grad(w)
    if g is not None:
        if g.is_contiguous():
            K.conv2d_wgrad(x, dy, w.shape[2], w.shape[3], stride, pad, dw=g, oihw=True)
            return None
        if g.permute(0, 2, 3, 1).is_contiguous():      # channels_last arena: the kernel's native (O,H,W,I) layout
            K.conv2d_wgrad(x, dy, w.shape[2], w.shape[3], stride, pad, dw=g, oihw=False)
            return None
    return K.conv2d_wgrad(x, dy, w.shape[2], w.shape[3], stride, pad, oihw=True)


def _linear_wgrad_to_master(x, dz, w, chw, blocks=None):
    """linear weight gradient in the master layout, accumulated straight into w's own .grad when it has one (-> None)"""
    g = _own_grad(w)
    if g is not None and g.is_contiguous():
        K.linear_wgrad(x, dz, dw=g, chw=chw, blocks=blocks)
        return None
    return K.linear_wgrad(x, dz, chw=chw, blocks=blocks)


def _grad_slot(p):
    """(.grad to accumulate into in place, or a fresh zero buffer; True if autograd must be given the buffer)"""
    g = _own_grad(p)
    if g is not None and g.is_contiguous():
        return g, False
    return torch.zeros_like(p, dtype=torch.float32), True


# ---- gradient chaining -------------------------------------------------------------------------------------------------
# A tensor with several consumers (DLA: block input -> conv1 + residual; tree1 output -> tree2 + Root; Tree input ->
# pool + strided conv; FPN top-down map -> output conv + the next lateral's addend ...) makes autograd run one add pass
# per extra consumer over the whole gradient.
# `fork(t, n)` hands every consumer its own alias of t; the aliases share a _GradSink.  The first consumer to produce
# its gradient parks the buffer in the sink and returns it; every later consumer ADDS INTO that buffer inside the kernel
# that produces its contribution (conv epilogue add_mode 3, c3d_bn_bwd's accumulating dres, c3d_maxpool2_bwd's accumulate)
# and returns None.  _Fork.backward — which autograd runs after all consumers — folds in whatever reached it as a plain
# tensor (consumers that know nothing of sinks) and hands the buffer to the producer.  Same sums as autograd's, with
# the adds done in fp32 before the single bf16 rounding.
GRAD_CHAIN = True      # False: plain autograd sums (the reference the gradient-chaining tests compare against)


class _GradSink:
    __slots__ = ("buf",)

    def __init__(self):
        self.buf = None


def _same_buffer(a, b):
    return a is b or (a.data_ptr() == b.data_ptr() and a.shape == b.shape and a.stride() == b.stride())


class _Fork(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, n, sink, outermost):
        ctx.sink, ctx.outermost = sink, outermost
        ctx.set_materialize_grads(False)
        return tuple(x.view(x.shape) for _ in range(n))

    @staticmethod
    def backward(ctx, *gs):
        sink = ctx.sink
        carried, extra = False, None
        for g in gs:
            if g is None:
                continue
            if sink.buf is not None and _same_buffer(g, sink.buf):
                carried = True                         # the parked buffer itself, travelling up its own path
            elif sink.buf is not None:
                sink.buf.add_(g.to(sink.buf.dtype))    # plain gradient of a consumer outside the protocol
            else:
                extra = g if extra is None else extra + g     # nobody parked a buffer yet: plain autograd sums
        if ctx.outermost:
            total = sink.buf
            sink.buf = None
            if total is None:
                total = extra
            elif extra is not None:
                total.add_(extra.to(total.dtype))
            return total, None, None, None
        # inner fork: never park a foreign tensor (it may be shared with other autograd edges); pass it up instead
        if extra is not None:
            if sink.buf is None or not carried:
                return extra, None, None, None         # the outer fork adds it to / adopts it as the total
            sink.buf.add_(extra.to(sink.buf.dtype))
        return (sink.buf if carried else None), None, None, None


def fork(t, n):
    """n aliases of t, one per consumer (see above).  Nested forks of an alias share the outer sink."""
    if n <= 1 or not GRAD_CHAIN or not torch.is_grad_enabled() or not t.requires_grad:
        return (t,) * n
    outer = getattr(t, "_c3d_sink", None)
    sink = outer if outer is not None else _GradSink()
    outs = _Fork.apply(t, n, sink, outer is None)
    for o in outs:
        o._c3d_sink = sink
    return outs


def _sink_of(t):
    return getattr(t, "_c3d_sink", None) if GRAD_CHAIN else None


def _deliver(sink, g):
    """first arrival: park g and return it to autograd; later arrivals were added in place by the caller -> None"""
    if sink is None:
        return g
    if sink.buf is None:
        sink.buf = g
        return g
    if not _same_buffer(g, sink.buf):
        sink.buf.add_(g)                               # a contribution without an accumulating kernel variant
    return None


class CatChannels(torch.autograd.Function):
    """torch.cat(xs, dim=-1) of NHWC maps (dla.py:168 Root input); backward hands every input its channel slice of the
    gradient in place (no copies) and parks the slices in the inputs' gradient sinks."""

    @staticmethod
    def forward(ctx, *xs):
        ctx.sinks = [_sink_of(x) for x in xs]
        ctx.widths = [x.shape[-1] for x in xs]
        return torch.cat(xs, dim=-1)

    @staticmethod
    def backward(ctx, dout):
        outs, off = [], 0
        for sink, c in zip(ctx.sinks, ctx.widths):
            outs.append(_deliver(sink, dout[..., off:off + c]))
            off += c
        return tuple(outs)


class ConvBNAct(torch.autograd.Function):
    """out = [relu]( BN_train|eval( conv(x, w) ) [+ residual] ) — dla.py:40-68 BasicBlock halves, Root, project."""

    @staticmethod
    def forward(ctx, x, w, gamma, beta, running_mean, running_var, residual, stride, pad, relu, training, eps,
                momentum):
        x = x.contiguous()
        wp = _packed(w)[0]
        if training:
            y, stats = K.conv2d_fwd(x, wp, stride=stride, pad=pad, want_stats=True)
            count = y.numel() // y.shape[-1]
            mean, rstd = Kx.bn_finalize(stats, count, eps, momentum, running_mean, running_var)
        else:
            y = K.conv2d_fwd(x, wp, stride=stride, pad=pad)
            mean, rstd = running_mean, torch.rsqrt(running_var + eps)
        res = residual.contiguous() if residual is not None else None
        out = Kx.bn_apply(y, mean, rstd, gamma, beta, res, relu)
        ctx.save_for_backward(x, w, gamma, y, mean, rstd, out, beta)
        ctx.cfg = (stride, pad, relu, training, residual is not None)
        ctx.sinks = (_sink_of(x), _sink_of(residual) if residual is not None else None)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, w, gamma, y, mean, rstd, out, beta = ctx.saved_tensors
        stride, pad, relu, training, has_res = ctx.cfg
        dgamma, ret_g = _grad_slot(gamma)
        dbeta, ret_b = _grad_slot(beta)
        # a ReLU layer without residual: its mask is recomputed from y inside the kernels (no read of `out`)
        remask = relu and not has_res
        sx, sr = ctx.sinks
        want_res = has_res and ctx.needs_input_grad[6]
        into = sr.buf if (want_res and sr is not None and sr.buf is not None and sr.buf.dtype == y.dtype) else None
        dy, dres = Kx.bn_bwd(dout, None if remask else out, y, mean, rstd, gamma, relu, dgamma, dbeta,
                              want_res, frozen=not training, beta=beta if remask else None, dres_into=into)
        if want_res:
            dres = None if into is not None else _deliver(sr, dres)
        dx = _dgrad_chained(sx, dy, w, stride, pad, x.shape[1:3]) if ctx.needs_input_grad[0] else None
        dw = _wgrad_to_master(x, dy, w, stride, pad) if ctx.needs_input_grad[1] else None
        return (dx, dw, dgamma if ret_g else None, dbeta if ret_b else None, None, None, dres, None, None, None, None,
                None, None)


class ConvBias(torch.autograd.Function):
    """out = [relu]( conv(x, w) + b [+ up2(addend)] ) — FPN lateral/output convs and the RPN head conv."""

    @staticmethod
    def forward(ctx, x, w, bias, addend, stride, pad, relu, out_fp32):
        x = x.contiguous()
        add = addend.contiguous() if addend is not None else None
        out = K.conv2d_fwd(x, _packed(w)[0], bias, stride, pad, relu=relu, addend=add, up2=add is not None,
                           out_fp32=out_fp32)
        ctx.save_for_backward(x, w, out if relu else None, bias)
        ctx.cfg = (stride, pad, relu, addend is not None, bias is not None)
        ctx.sinks = (_sink_of(x), _sink_of(addend) if addend is not None else None)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, w, out, bias = ctx.saved_tensors
        stride, pad, relu, has_add, has_bias = ctx.cfg
        dbias, ret_b = _grad_slot(bias) if has_bias else (None, False)
        dzb = Kx.bias_act_bwd(dout, out, relu, dbias)
        sx, sa = ctx.sinks
        dadd = _deliver(sa, Kx.sumpool2(dzb)) if has_add and ctx.needs_input_grad[3] else None
        dx = _dgrad_chained(sx, dzb, w, stride, pad, x.shape[1:3]) if ctx.needs_input_grad[0] else None
        dw = _wgrad_to_master(x, dzb, w, stride, pad) if ctx.needs_input_grad[1] else None
        return dx, dw, dbias if ret_b else None, dadd, None, None, None, None


def _packed_linear(w, chw):
    """bf16 (N,K') forward operand and its (K',N) transpose for the data gradient, cached like the conv packs."""
    hit = _cache_get(_lin_cache, w)
    if hit is None or hit[0] != chw:
        hit = _cache_put(_lin_cache, w, (chw,) + K.pack_linear_weight(w, chw))
    return hit[1], hit[2]


class LinearAct(torch.autograd.Function):
    """y = [relu](x W^T + b) on the wgmma GEMM (c3d_linear_fwd / _dgrad / _wgrad) — the FC layers of
    FastRCNNConvFCHead / FastRCNNOutputLayers / CubeHead (Base.yaml:67-70, cube_head.py:63-73,108-144).
    x (rows, K) bf16; W fp32 master (N, K) in the reference's layout; chw = (C, PP) when the master's input features are
    ordered (c, p) while x is the NHWC-flattened RoI (p, c)."""

    @staticmethod
    def forward(ctx, x, w, bias, relu, out_fp32, chw):
        x = x.contiguous()
        wp, wt = _packed_linear(w, chw)
        b = bias.detach().float().contiguous() if bias is not None else None
        y = K.linear_fwd(x, wp, b, relu, out_fp32)
        ctx.save_for_backward(x, w, bias, y if relu else None, wt)
        ctx.cfg = (relu, chw)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, bias, y, wt = ctx.saved_tensors
        relu, chw = ctx.cfg
        dbias, ret_b = _grad_slot(bias) if bias is not None and ctx.needs_input_grad[2] else (None, False)
        dz = Kx.bias_act_bwd(dy, y, relu, dbias)                       # bf16 (rows, N); dbias += column sums
        dx = K.linear_dgrad(dz, wt) if ctx.needs_input_grad[0] else None
        dw = _linear_wgrad_to_master(x, dz, w, chw) if ctx.needs_input_grad[1] else None
        return dx, dw, dbias if ret_b else None, None, None, None


class TwoHeadFC1(torch.autograd.Function):
    """First FC layer of the box head over all B*S pooled RoIs and of the cube head over the first Fc RoIs of every image
    (Base.yaml:66-68,78-80: same pooler => the cube head's RoIs are a prefix of the box head's sampled RoIs), sharing ONE
    pooled tensor: the cube GEMM reads its rows in place (c3d_linear_fwd over row blocks) and its data gradient is accumulated
    into the box head's (c3d_linear_dgrad, in-place epilogue) — no gather copy forward, no zero-padded scatter + add
    backward (~1 GB of HBM traffic per step at batch 32)."""

    @staticmethod
    def forward(ctx, x, wb, bb, wc, bc, B, S, Fc, chw):
        x = x.contiguous()
        wpb, wtb = _packed_linear(wb, chw)
        wpc, wtc = _packed_linear(wc, chw)
        hb = K.linear_fwd(x, wpb, bb.detach().float().contiguous(), relu=True)
        hc = K.linear_fwd(x, wpc, bc.detach().float().contiguous(), relu=True, blocks=(B, Fc, S))
        ctx.save_for_backward(x, wb, bb, wc, bc, hb, hc, wtb, wtc)
        ctx.cfg = (B, S, Fc, chw)
        return hb, hc

    @staticmethod
    def backward(ctx, dhb, dhc):
        x, wb, bb, wc, bc, hb, hc, wtb, wtc = ctx.saved_tensors
        B, S, Fc, chw = ctx.cfg
        if dhb is None:
            dhb = torch.zeros_like(hb)
        if dhc is None:
            dhc = torch.zeros_like(hc)
        gbb, rb = _grad_slot(bb)
        gbc, rc = _grad_slot(bc)
        dzb = Kx.bias_act_bwd(dhb, hb, True, gbb)
        dzc = Kx.bias_act_bwd(dhc, hc, True, gbc)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = K.linear_dgrad(dzb, wtb)
            K.linear_dgrad(dzc, wtc, blocks=(B, Fc, S), dx=dx, accumulate=True)
        dwb = _linear_wgrad_to_master(x, dzb, wb, chw)
        dwc = _linear_wgrad_to_master(x, dzc, wc, chw, blocks=(B, Fc, S))
        return dx, dwb, gbb if rb else None, dwc, gbc if rc else None, None, None, None, None


class MaxPool2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.sink = _sink_of(x)
        x = x.contiguous()
        ctx.save_for_backward(x)
        return Kx.maxpool2_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        sink = ctx.sink
        if sink is not None and sink.buf is not None and sink.buf.dtype == x.dtype:
            Kx.maxpool2_bwd(x, dy, into=sink.buf)
            return None
        return _deliver(sink, Kx.maxpool2_bwd(x, dy))


class MaxPool3s2(torch.autograd.Function):
    """3x3 / stride 2 / pad 1 max pool of the torchvision ResNet stem (resnet.py:45-50) on NHWC bf16."""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        ctx.save_for_backward(x)
        return Kx.maxpool3s2_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return Kx.maxpool3s2_bwd(x, dy)


class ROIAlign(torch.autograd.Function):
    """feats (tuple of NHWC bf16 maps), rois (R,6) [batch, level, x1,y1,x2,y2] -> (R,7,7,C) bf16."""

    @staticmethod
    def forward(ctx, rois, strides, pooled, *feats):
        ctx.sinks = [_sink_of(f) for f in feats]
        feats = [f.contiguous() for f in feats]
        ctx.save_for_backward(rois, *feats)
        ctx.cfg = (strides, pooled)
        return Kx.roi_align_fwd(feats, strides, rois, pooled)

    @staticmethod
    def backward(ctx, dout):
        rois, *feats = ctx.saved_tensors
        strides, pooled = ctx.cfg
        grads = Kx.roi_align_bwd(feats, strides, rois, dout.contiguous(), pooled)
        return (None, None, None) + tuple(_deliver(s, g.to(torch.bfloat16)) for s, g in zip(ctx.sinks, grads))


class CubeLossRows(torch.autograd.Function):
    """raw (n,13) head outputs + aux (n,28) constants -> (n,10): [u, l_dims, l_xy, l_z, l_pose, l_joint (each x
    sqrt2*exp(-u)), |z-gz|, dims err, xy err, conf] — roi_heads.py:409-740 in one kernel each way."""

    @staticmethod
    def forward(ctx, raw, aux):
        raw, aux = raw.contiguous().float(), aux.contiguous().float()
        ctx.save_for_backward(raw, aux)
        out = Kx.cube_loss_fwd(raw, aux)
        ctx.mark_non_differentiable()
        return out

    @staticmethod
    def backward(ctx, dout):
        raw, aux = ctx.saved_tensors
        return Kx.cube_loss_bwd(raw, aux, dout[:, :6].contiguous().float()), None


class RPNLossSums(torch.autograd.Function):
    """logits (B,A), deltas (B,A,4) fp32 + labels / matches -> (6,) [sum cls, sum loc, #pos, #neg, sum sig(pos),
    sum sig(rest)]; gradients flow from the first two entries only (c3d_rpn_loss_fwd / _bwd, one launch each)."""

    @staticmethod
    def forward(ctx, logits, deltas, labels, matched_idx, gt_boxes, anchors, weights):
        logits, deltas = logits.contiguous().float(), deltas.contiguous().float()
        labels, matched_idx = labels.to(torch.int8).contiguous(), matched_idx.contiguous()
        gt_boxes, anchors = gt_boxes.contiguous().float(), anchors.contiguous().float()
        ctx.save_for_backward(logits, deltas, labels, matched_idx, gt_boxes, anchors)
        ctx.weights = tuple(weights)
        return Kx.rpn_loss_fwd(logits, deltas, labels, matched_idx, gt_boxes, anchors, weights)

    @staticmethod
    def backward(ctx, dacc):
        logits, deltas, labels, matched_idx, gt_boxes, anchors = ctx.saved_tensors
        dacc = dacc.contiguous().float()
        dl, dd = Kx.rpn_loss_bwd(logits, deltas, labels, matched_idx, gt_boxes, anchors, ctx.weights, dacc[0:1], dacc[1:2])
        return dl, dd, None, None, None, None, None


class BoxLoss(torch.autograd.Function):
    """FastRCNNOutputs.losses (fast_rcnn.py:145-194) on the fused predictor output rows [K+1 scores | 4K deltas | pad]:
    -> (7,) [loss_cls, loss_box_reg, cls_accuracy, fg_cls_accuracy, false_negative, #valid, #fg]; gradients flow from the
    first two entries (c3d_box_loss_fwd / _bwd, one launch each way)."""

    @staticmethod
    def forward(ctx, pred, classes, valid, boxes, gt_boxes, K, weights):
        pred = pred.contiguous().float()
        classes, valid = classes.contiguous().to(torch.int64), valid.contiguous().to(torch.uint8)
        boxes, gt_boxes = boxes.contiguous().float(), gt_boxes.contiguous().float()
        acc = Kx.box_loss_fwd(pred, classes, valid, boxes, gt_boxes, K, weights)
        ctx.save_for_backward(pred, classes, valid, boxes, gt_boxes, acc)
        ctx.cfg = (K, tuple(weights))
        nv, nfg = acc[2].clamp(min=1.0), acc[3].clamp(min=1.0)
        den = torch.stack([nv, nv, nv, nfg, nfg])
        # (no python-list indexing: that would be a host->device copy of the index, illegal inside a CUDA-graph capture)
        return torch.cat([torch.cat([acc[0:2], acc[4:7]]) / den, acc[2:4]])

    @staticmethod
    def backward(ctx, g):
        pred, classes, valid, boxes, gt_boxes, acc = ctx.saved_tensors
        K, weights = ctx.cfg
        dpred = Kx.box_loss_bwd(pred, classes, valid, boxes, gt_boxes, K, weights, acc, g[:2].contiguous().float())
        return dpred, None, None, None, None, None, None


class CubeHeadLoss(torch.autograd.Function):
    """fused cube-predictor output (n, ld) -> (11,) [Cube/uncert, loss_dims, loss_xy, loss_z, loss_pose, loss_joint (finite
    means over valid RoIs, unweighted), z_error, dims_error, xy_error, z_close, conf]: gather of the predicted class's 13
    outputs + the per-RoI constants (c3d_cube_gather), decode + disentangled losses (c3d_cube_loss_fwd), masked finite
    means (c3d_cube_reduce_fwd); backward = the three adjoint kernels + scatter into the class's columns."""

    @staticmethod
    def forward(ctx, pred, classes, valid, boxes, meta, priors, gt3, gtR, per_image, K, virtual_focal):
        pred = pred.contiguous().float()
        classes, valid8 = classes.contiguous().to(torch.int64), valid.contiguous().to(torch.uint8)
        raw, aux = Kx.cube_gather(pred, classes, boxes.contiguous().float(), meta.contiguous().float(), priors.contiguous().float(),
                                  gt3.contiguous().float(), gtR.contiguous().float(), per_image, K, virtual_focal)
        rows = Kx.cube_loss_fwd(raw, aux)
        sums, cnts = Kx.cube_reduce_fwd(rows, valid8)
        ctx.save_for_backward(raw, aux, rows, valid8, cnts, classes)
        ctx.cfg = (K, pred.shape[1])
        den = torch.cat([cnts[:6], cnts[6:7].expand(5)]).clamp(min=1.0)
        return sums[:11] / den

    @staticmethod
    def backward(ctx, g):
        raw, aux, rows, valid8, cnts, classes = ctx.saved_tensors
        K, ld = ctx.cfg
        drows = Kx.cube_reduce_bwd(rows, valid8, cnts, g[:6].contiguous().float())
        draw = Kx.cube_loss_bwd(raw, aux, drows)
        return Kx.cube_scatter(draw, classes, K, ld), None, None, None, None, None, None, None, None, None, None
