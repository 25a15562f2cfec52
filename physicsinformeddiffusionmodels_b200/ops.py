"""torch.autograd.Function wrappers around the libpidm C ABI (include/pidm.h).

Activations are NHWC tensors [B, H, W, C] in the activation dtype (bf16 by default, fp32 in the
exact mode used for parity debugging).  Every forward AND backward below is a libpidm kernel launch;
PyTorch only allocates the buffers and records the graph.

Parameter gradients: every wgrad-type kernel ACCUMULATES into the buffer it is given.  In the default
mode that buffer is a fresh zero tensor returned to autograd; when a parameter carries a
`_pidm_grad` view (flat-buffer engine, engine.py) the kernel accumulates straight into it and autograd
sees None, so one flat fp32 buffer is ready for the NCCL all-reduce / fused Adam with no per-tensor
copies."""
import torch

from . import _lib
from ._lib import call, stream

_STATE = {'act_dtype': torch.bfloat16, 'use_tc': True}


def set_precision(name):
    """'bf16' (default: bf16 activations / GEMM operands, fp32 accumulate) or 'fp32' (exact mode)."""
    _STATE['act_dtype'] = {'bf16': torch.bfloat16, 'fp32': torch.float32}[name]


def set_tensor_core_conv(flag):
    _STATE['use_tc'] = bool(flag)


def act_dtype():
    return _STATE['act_dtype']


def _code(t):
    return _lib.DTYPE_CODE[t.dtype]


def _grad_buffer(p):
    """(buffer to accumulate into, value to hand back to autograd)."""
    g = getattr(p, '_pidm_grad', None)
    if g is not None:
        return g, None
    z = torch.zeros_like(p)
    return z, z


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError('physicsinformeddiffusionmodels_b200 runs on CUDA (H100) only: got a CPU tensor. '
                               'There is no CPU fallback on the product path.')


def _need_f32(**named):
    """Raw device pointers cross the C ABI: a table / field of the wrong dtype or with strides would be read as garbage,
    so the public wrappers check what they hand over (fp32, contiguous, CUDA)."""
    for k, t in named.items():
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(f'{k}: expected a CUDA tensor (no CPU fallback on the product path)')
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError(f'{k}: expected a contiguous float32 tensor, got {t.dtype}, strides {t.stride()}')


# ----------------------------------------------------------------------------------------------
# layout
# ----------------------------------------------------------------------------------------------
def nchw_to_nhwc(x, cpad, dtype=None):
    """[B,C,H,W] fp32 -> [B,H,W,cpad] activations (zero-padded channels).  Input is data: no gradient."""
    _need_cuda(x)
    B, C, H, W = x.shape
    dtype = dtype or act_dtype()
    y = torch.empty(B, H, W, cpad, device=x.device, dtype=dtype)
    call('pidm_nchw_to_nhwc', x.contiguous().float(), y, B, C, H * W, cpad, _lib.DTYPE_CODE[dtype], stream())
    return y


class _CondEmbed(torch.autograd.Function):
    """GELU(emb_conv[0](cond)) of the residual-gradient guidance branch (reference unet_model.py:520-524,585-603) as NHWC
    activations, from cond [B, HW, 2] fp32 (data: no gradient) with the samples in null_mask [B] (bool) taking cond = 0.
    Backward only produces the weight and bias gradients, on the weight-gradient stream."""

    @staticmethod
    def forward(ctx, cond, null_mask, weight, bias, dtype):
        B, HW, _ = cond.shape
        C = weight.shape[0]
        out = torch.empty(B, HW, C, device=cond.device, dtype=dtype)
        call('pidm_cond_embed_fwd', cond, null_mask, weight, bias, out, B, HW, C, _lib.DTYPE_CODE[dtype], stream())
        ctx.save_for_backward(cond, null_mask, weight, bias)
        return out

    @staticmethod
    def backward(ctx, dg):
        cond, null_mask, weight, bias = ctx.saved_tensors
        B, HW, _ = cond.shape
        C = weight.shape[0]
        dg = dg.contiguous()
        gw_buf, gw_ret = _grad_buffer(weight)
        gb_buf, gb_ret = _grad_buffer(bias)
        call('pidm_cond_embed_wgrad', cond, null_mask, weight, bias, dg, gw_buf, gb_buf, B, HW, C, _code(dg),
             _wgrad_stream(cond, null_mask, dg))
        return None, None, gw_ret, gb_ret, None


def cond_embed(cond, null_mask, weight, bias, P, dtype=None):
    """[B, P*P, 2] fp32 cond, [B] bool null mask -> [B, P, P, C] activations GELU(W0 cond + b0)"""
    _need_cuda(cond, null_mask)
    if cond.shape[-1] != 2 or weight.shape[1] != 2:
        raise NotImplementedError('the guidance embedding is built for the 2-channel Darcy residual gradient')
    B = cond.shape[0]
    out = _CondEmbed.apply(cond.detach().contiguous().float(), null_mask.contiguous(), weight, bias,
                           dtype or act_dtype())
    return out.view(B, P, P, -1)


class _Stash(torch.autograd.Function):
    """Identity whose backward parks the incoming gradient in `link['skip']` instead of returning it.  Used for the
    skip branch of y = f(x) + x: the backward of the FIRST op of f (a convolution dgrad or the LayerNorm backward, both
    take a residual) adds the parked gradient in its epilogue, so autograd has a single contribution for x and no
    separate accumulation kernel runs.  Ordering: this node is created after every node of f, so the autograd engine
    (highest sequence number first among ready nodes) runs it before any node of f can become ready."""

    @staticmethod
    def forward(ctx, x, link):
        ctx.link = link
        link['expect_skip'] = True
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        ctx.link['skip'] = g.contiguous()
        return None, None


def stash_grad(x, link):
    return _Stash.apply(x, link)


def _take_skip(link):
    """gradient parked by _Stash / a stashing convolution for the op that owns `link` (None if there is no link)"""
    if link is None or not link.get('expect_skip'):
        return None
    if 'skip' not in link:
        raise RuntimeError('skip-connection gradient was expected but has not been produced yet (autograd order)')
    return link.pop('skip')


class _Concat(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        B, H, W, Ca = a.shape
        Cb = b.shape[-1]
        o = torch.empty(B, H, W, Ca + Cb, device=a.device, dtype=a.dtype)
        call('pidm_concat_channels', a, b, o, B * H * W, Ca, Cb, _code(a), stream())
        ctx.shapes = (a.shape, b.shape)
        return o

    @staticmethod
    def backward(ctx, g):
        sa, sb = ctx.shapes
        g = g.contiguous()
        ga = torch.empty(sa, device=g.device, dtype=g.dtype)
        gb = torch.empty(sb, device=g.device, dtype=g.dtype)
        call('pidm_split_channels', g, ga, gb, sa[0] * sa[1] * sa[2], sa[3], sb[3], _code(g), stream())
        return ga, gb


def concat(a, b):
    return _Concat.apply(a.contiguous(), b.contiguous())


# ----------------------------------------------------------------------------------------------
# convolution (implicit GEMM).  `spec` is a ConvSpec created by the owning module (packing.py).
# ----------------------------------------------------------------------------------------------
# Pool of pre-zeroed fp32 scratch (fused GroupNorm statistics): one fill per network forward instead of one memset
# node per convolution.  Slices stay alive through the tensors that view them (saved for backward).
_ZERO_POOL = {'buf': None, 'cur': 0}


def zero_pool_begin(nfloats, device):
    _ZERO_POOL['buf'] = torch.zeros(int(nfloats), device=device, dtype=torch.float32)
    _ZERO_POOL['cur'] = 0


def zero_pool_end():
    _ZERO_POOL['buf'] = None


def _zero_take(*shape):
    buf = _ZERO_POOL['buf']
    n = 1
    for d in shape:
        n *= int(d)
    n_al = (n + 31) // 32 * 32                     # keep slices 128-byte aligned
    if buf is None or _ZERO_POOL['cur'] + n_al > buf.numel():
        return None
    out = buf[_ZERO_POOL['cur']:_ZERO_POOL['cur'] + n].view(*shape)
    _ZERO_POOL['cur'] += n_al
    return out


def _conv_launch(x, wp, bias, residual, y, g, transposed, gn_sums=None, gn_groups=0, gn_zeroed=False):
    """g = (B,H,W,Cin,Ho,Wo,Cout,KH,KW,stride,pad).  Returns True if the fused GroupNorm statistics were produced."""
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad = g
    tr = 1 if transposed else 0
    if (_STATE['use_tc'] and x.dtype == torch.bfloat16
            and call('pidm_conv2d_tc_general_supported', B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, tr)):
        cpg = Cout // gn_groups if gn_groups else 0
        fuse = gn_sums is not None and (cpg in (4, 8, 16) or (cpg > 0 and cpg % 32 == 0))
        call('pidm_conv2d_tc_general', x, wp, bias, residual, y, B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, tr,
             gn_sums if fuse else None, gn_groups if fuse else 0, 1 if gn_zeroed else 0, stream())
        return fuse
    else:
        call('pidm_conv2d_simt', x, wp, bias, residual, y, B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad,
             1 if transposed else 0, _code(x), stream())
        return False


def wrap_pad(x, halo):
    """[B,H,W,C] -> [B,H+2h,W+2h,C] with the halo wrapped around both spatial axes (circular padding)."""
    B, H, W, C = x.shape
    y = torch.empty(B, H + 2 * halo, W + 2 * halo, C, device=x.device, dtype=x.dtype)
    call('pidm_wrap_pad_nhwc', x, y, B, H, W, C, halo, _code(x), stream())
    return y


def _halo_geometry(g, halo, transposed):
    """geometry g = (B,H,W,Cin,Ho,Wo,Cout,KH,KW,stride,pad) of a circular layer restated over its input with a wrapped
    halo: a valid (pad 0) convolution, or for the transposed gather (halo 1) every tap one pixel further in (pad + 2)"""
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad = g
    return (B, H + 2 * halo, W + 2 * halo, Cin, Ho, Wo, Cout, KH, KW, stride, pad + 2 if transposed else 0)


def _convT_wgrad_tc(dtype, g):
    """does the weight gradient of a transposed layer with forward geometry g run on the tensor cores?"""
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad = g
    return (_STATE['use_tc'] and dtype == torch.bfloat16
            and call('pidm_conv2d_wgrad_tc_supported', B, H, W, Cout, Cin, KH, KW, stride) == 1)


class _Conv2d(torch.autograd.Function):
    """`link` (optional dict) couples this convolution to the GroupNorm that consumes its output: forward leaves the
    fused statistics in link['sums']; the GroupNorm backward leaves this conv's bias gradient in link['dbias']."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, spec, link, skip):
        """skip (optional) = (mode, dict): mode 'take' -> this conv's dgrad adds the gradient parked in the dict;
        mode 'park' -> this conv parks its own input gradient there instead of returning it."""
        B, H, W, Cin = x.shape
        Ho, Wo = spec.out_hw(H, W)
        y = torch.empty(B, Ho, Wo, spec.cout, device=x.device, dtype=x.dtype)
        g = (B, H, W, Cin, Ho, Wo, spec.cout, spec.kh, spec.kw, spec.stride, spec.pad)
        xin, gin = x, g
        if spec.circular:
            xin, gin = wrap_pad(x, spec.halo), _halo_geometry(g, spec.halo, spec.transposed)
        sums, zeroed = None, False
        if link is not None:
            sums = _zero_take(B, link['groups'], 2)
            zeroed = sums is not None
            if sums is None:
                sums = torch.empty(B, link['groups'], 2, device=x.device, dtype=torch.float32)
        fused = _conv_launch(xin, spec.wp_fwd, bias, residual, y, gin, spec.transposed, sums,
                             link['groups'] if link else 0, zeroed)
        if link is not None:
            link['sums'] = sums if fused else None
            link['bias'] = bias
        # a circular conv keeps the halo'd copy: its weight gradient reads it as the forward did and backward never pads
        # x again.  Exception: the tensor-core weight gradient of the transposed layer gathers from dy and reads x on
        # its own (unpadded) grid.
        keep = xin
        if spec.transposed and (not spec.circular or _convT_wgrad_tc(x.dtype, g)):
            keep = x
        ctx.save_for_backward(keep, weight, bias)
        ctx.spec, ctx.g, ctx.has_res, ctx.link, ctx.skip = spec, g, residual is not None, link, skip
        if skip is not None and skip[0] == 'park':
            skip[1]['expect_skip'] = True
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias = ctx.saved_tensors
        dy = dy.contiguous()
        skip = ctx.skip
        dgrad_res = _take_skip(skip[1]) if (skip is not None and skip[0] == 'take' and ctx.needs_input_grad[0]) else None
        dx, gw_ret, gb_ret = _conv_backward(x, weight, bias, ctx.spec, ctx.g, dy, ctx.needs_input_grad[0], ctx.link,
                                            dgrad_res)
        if skip is not None and skip[0] == 'park':
            skip[1]['skip'] = dx
            dx = None
        return dx, gw_ret, gb_ret, (dy if ctx.has_res else None), None, None, None


# Weight-gradient kernels only feed the optimizer: inside TrainEngine they are launched on a side stream so that they
# overlap the (latency-bound) dgrad / normalisation chain of the remaining layers.  Operand tensors are kept alive until
# the join (they were allocated on the main stream).
_SIDE = {'stream': None, 'keep': [], 'active': False}


def side_stream_begin():
    if _SIDE['stream'] is None:
        _SIDE['stream'] = torch.cuda.Stream()
    _SIDE['active'] = True
    _SIDE['keep'] = []


def side_stream_join():
    if _SIDE['active']:
        torch.cuda.current_stream().wait_stream(_SIDE['stream'])
        _SIDE['keep'] = []
        _SIDE['active'] = False


_FORK = {'stream': None}


def fork_stream():
    """a second stream that has been made to wait for everything queued on the current one"""
    if _FORK['stream'] is None:
        _FORK['stream'] = torch.cuda.Stream()
    _FORK['stream'].wait_stream(torch.cuda.current_stream())
    return _FORK['stream']


def _wgrad_stream(*operands):
    """stream handle for a wgrad-type launch whose operands are ready on the current stream"""
    if not _SIDE['active']:
        return stream()
    side = _SIDE['stream']
    side.wait_stream(torch.cuda.current_stream())
    _SIDE['keep'].extend(operands)
    return side.cuda_stream


def _conv_backward(x, weight, bias, spec, g, dy, need_dx, link=None, dgrad_residual=None):
    """dgrad + wgrad (+ bias gradient) of one convolution; returns (dx, grad_weight, grad_bias) as autograd expects.
    dgrad_residual (same shape as x) is added to dx in the dgrad epilogue."""
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad = g
    dx = None
    # circular layer: x is the halo'd input copy (regular conv) and dy gets its own wrapped halo for the dgrad (and for
    # the transposed layer's weight gradient, which gathers from dy)
    need_dgrad = need_dx or dgrad_residual is not None
    dyh = wrap_pad(dy, spec.dgrad_halo) if spec.circular and (need_dgrad or spec.transposed) else None
    if need_dgrad:
        dx = torch.empty(B, H, W, Cin, device=x.device, dtype=x.dtype)
        # dgrad: roles of input/output swap; regular conv -> transposed gather and vice versa.
        # For stride 1 the transposed gather equals a regular conv with the flipped kernel, which the
        # dgrad packing already encodes (pad' = K-1-pad), so the tensor-core kernel can take it.
        if stride == 1 and not spec.transposed:
            gd = (B, Ho, Wo, Cout, H, W, Cin, KH, KW, 1, KH - 1 - pad)
        else:
            gd = (B, Ho, Wo, Cout, H, W, Cin, KH, KW, stride, pad)
        tr_d = not spec.transposed and stride != 1
        dy_d = dy
        if dyh is not None:
            dy_d, gd = dyh, _halo_geometry(gd, spec.dgrad_halo, tr_d)
        _conv_launch(dy_d, spec.wp_dgrad, None, dgrad_residual, dx, gd, tr_d)
    gw_buf, gw_ret = _grad_buffer(weight)
    gb_buf, gb_ret = (None, None) if bias is None else _grad_buffer(bias)
    if link is not None and 'dbias' in link:
        # the consuming GroupNorm's backward already reduced dy over pixels (= this conv's bias gradient)
        gb_buf, gb_ret = None, link.pop('dbias')
    use_tc = _STATE['use_tc'] and x.dtype == torch.bfloat16
    tc_conv = (use_tc and not spec.transposed
               and call('pidm_conv2d_wgrad_tc_supported', B, Ho, Wo, Cin, Cout, KH, KW, stride))
    # the forward of a circular layer saved either its halo'd input (read as the forward read it) or, for the
    # tensor-core weight gradient of the transposed layer, x itself
    x_halo = spec.circular and x.shape[1] != H
    if spec.circular and spec.transposed:
        tc_convT = not x_halo
    else:
        tc_convT = spec.transposed and use_tc and call('pidm_conv2d_wgrad_tc_supported', B, H, W, Cout, Cin, KH, KW,
                                                       stride)
    # gathered operands as the kernels read them: (tensor, H, W, pad)
    xa, dya = (x, H, W, pad), (dy, Ho, Wo, pad)
    if x_halo:
        xa = (x, x.shape[1], x.shape[2], pad + 2 if spec.transposed else 0)
    elif spec.circular:
        dya = (dyh, Ho + 2, Wo + 2, 0)
    ws = _wgrad_stream(xa[0], dy, dya[0])
    if tc_conv:
        # D[(tap, ci)][co]: gathered operand = x, reduction grid = output pixels
        call('pidm_conv2d_wgrad_tc', xa[0], dy, gw_buf, B, xa[1], xa[2], Cin, spec.cin_real, Ho, Wo, Cout, KH, KW,
             stride, xa[3], spec.w_stride_c, spec.w_stride_n, ws)
        if gb_buf is not None:
            call('pidm_colsum', dy, gb_buf, B * Ho * Wo, Cout, _code(dy), ws)
    elif tc_convT:
        # ConvTranspose: D[(tap, co)][ci]: gathered operand = dy (sampled with the stride), grid = input pixels
        call('pidm_conv2d_wgrad_tc', dya[0], x, gw_buf, B, dya[1], dya[2], Cout, Cout, H, W, Cin, KH, KW, stride,
             dya[3], spec.w_stride_n, spec.w_stride_c, ws)
        if gb_buf is not None:
            call('pidm_colsum', dy, gb_buf, B * Ho * Wo, Cout, _code(dy), ws)
    else:
        call('pidm_conv2d_wgrad_simt', xa[0], dy, gw_buf, gb_buf, B, xa[1], xa[2], Cin, spec.cin_real, Ho, Wo, Cout,
             KH, KW, stride, xa[3], 1 if spec.transposed else 0, spec.w_stride_n, spec.w_stride_c, _code(x), ws)
    return dx, gw_ret, gb_ret


def conv2d(x, weight, bias, spec, residual=None, gn_link=None, skip=None):
    return _Conv2d.apply(x.contiguous(), weight, bias, None if residual is None else residual.contiguous(), spec,
                         gn_link, skip)


# ----------------------------------------------------------------------------------------------
# GroupNorm -> FiLM -> SiLU ; channel LayerNorm
# ----------------------------------------------------------------------------------------------
class _GroupNormSilu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, scale_shift, groups, eps, link, residual):
        B, H, W, C = x.shape
        y = torch.empty_like(x)
        pre = link is not None and link.get('sums') is not None
        sums = link['sums'] if pre else torch.empty(B, groups, 2, device=x.device, dtype=torch.float32)
        call('pidm_groupnorm_silu_fwd', x, gamma, beta, scale_shift, residual, y, sums, 1 if pre else 0, B, H * W, C,
             groups, eps, _code(x), stream())
        ctx.save_for_backward(x, gamma, beta, scale_shift, sums)
        ctx.groups, ctx.eps, ctx.link, ctx.has_res = groups, eps, link, residual is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, ss, sums = ctx.saved_tensors
        B, H, W, C = x.shape
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        gg_buf, gg_ret = _grad_buffer(gamma)
        gb_buf, gb_ret = _grad_buffer(beta)
        dss = None if ss is None else torch.empty_like(ss)
        ws = torch.empty(B * C * 2, device=x.device, dtype=torch.float32)
        dbias = None
        link = ctx.link
        if link is not None and link.get('bias') is not None:
            dbias, dbias_ret = _grad_buffer(link['bias'])
            link['dbias'] = dbias_ret             # picked up by the producing convolution's backward
        call('pidm_groupnorm_silu_bwd', x, dy, sums, gamma, beta, ss, dx, gg_buf, gb_buf, dss, dbias, ws, B, H * W, C,
             ctx.groups, ctx.eps, _code(x), stream())
        return dx, gg_ret, gb_ret, dss, None, None, None, (dy if ctx.has_res else None)


def groupnorm_silu(x, gamma, beta, scale_shift, groups, eps=1e-5, gn_link=None, residual=None):
    """residual (optional): added after the SiLU (ResnetBlock `h + x` with an identity res_conv)."""
    return _GroupNormSilu.apply(x.contiguous(), gamma, beta, scale_shift, groups, eps, gn_link,
                                None if residual is None else residual.contiguous())


class _LayerNormC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, eps, skip_link):
        C = x.shape[-1]
        y = torch.empty_like(x)
        call('pidm_layernorm_c_fwd', x, gamma, y, x.numel() // C, C, eps, _code(x), stream())
        ctx.save_for_backward(x, gamma)
        ctx.eps, ctx.skip_link = eps, skip_link
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma = ctx.saved_tensors
        C = x.shape[-1]
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        gg_buf, gg_ret = _grad_buffer(gamma)
        call('pidm_layernorm_c_bwd', x, dy, gamma, dx, gg_buf,
             _take_skip(ctx.skip_link) if ctx.needs_input_grad[0] else None, x.numel() // C, C, ctx.eps,
             _code(x), stream())
        return dx, gg_ret, None, None


def layernorm_c(x, gamma, eps=1e-5, skip_link=None):
    """gamma: the reference's [1,C,1,1,1] parameter (contiguous, so it is a flat [C] buffer).
    skip_link: dict shared with stash_grad() -- the parked skip-connection gradient is added to dx."""
    return _LayerNormC.apply(x.contiguous(), gamma, eps, skip_link)


# ----------------------------------------------------------------------------------------------
# attention cores
# ----------------------------------------------------------------------------------------------
class _LinAttn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, heads):
        B, H, W, C3 = qkv.shape
        N = H * W
        hid = heads * 32
        assert C3 == 3 * hid
        out = torch.empty(B, H, W, hid, device=qkv.device, dtype=qkv.dtype)
        ctxm = torch.empty(B, heads, 32, 32, device=qkv.device, dtype=torch.float32)
        kmax = torch.empty(B, heads, 32, device=qkv.device, dtype=torch.float32)
        kzinv = torch.empty_like(kmax)
        ws = torch.empty(call('pidm_linattn_workspace_floats', B, N, heads), device=qkv.device, dtype=torch.float32)
        call('pidm_linattn_fwd', qkv, out, ctxm, kmax, kzinv, ws, B, N, heads, _code(qkv), stream())
        ctx.save_for_backward(qkv, ctxm, kmax, kzinv)
        ctx.heads = heads
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, ctxm, kmax, kzinv = ctx.saved_tensors
        B, H, W, _ = qkv.shape
        dout = dout.contiguous()
        dqkv = torch.empty_like(qkv)
        dctx = torch.empty_like(ctxm)
        call('pidm_linattn_bwd', qkv, dout, ctxm, kmax, kzinv, dqkv, dctx, B, H * W, ctx.heads, _code(qkv), stream())
        return dqkv, None


class _LinAttnBlock(torch.autograd.Function):
    """The whole linear-attention block at the 32-channel levels: y = residual + to_out(attention(to_qkv(xn))) with a 1x1
    32 -> 768 to_qkv (no bias) and a 1x1 256 -> C to_out (with bias) (reference unet_model.py:275-297).  Neither the
    [B, N, 768] qkv nor the [B, N, 256] attention output, nor their gradients, are written: the kernels recompute q, k, v
    per head from xn, forward projects each head's output tile on chip, and backward recomputes it and dout per head
    from dy; a second pass over (xn, dy) on the weight-gradient stream accumulates both projections' weight gradients.
    Like the to_out convolution it replaces, it hands dy back as the residual's gradient."""

    @staticmethod
    def forward(ctx, xn, w_qkv, spec_qkv, w_out, b_out, spec_out, residual, heads):
        B, H, W, C = xn.shape
        N = H * W
        y = torch.empty_like(residual)
        ctxm = torch.empty(B, heads, 32, 32, device=xn.device, dtype=torch.float32)
        kmax = torch.empty(B, heads, 32, device=xn.device, dtype=torch.float32)
        kzinv = torch.empty_like(kmax)
        ws = torch.empty(call('pidm_linattn_block_workspace_floats', B, N), device=xn.device, dtype=torch.float32)
        call('pidm_linattn_block_fwd', xn, spec_qkv.wp_fwd, spec_out.wp_fwd, b_out, residual, y, ctxm, kmax, kzinv, ws,
             B, N, stream())
        ctx.save_for_backward(xn, w_qkv, w_out, b_out, ctxm, kmax, kzinv)
        ctx.specs = (spec_qkv, spec_out)
        return y

    @staticmethod
    def backward(ctx, dy):
        xn, w_qkv, w_out, b_out, ctxm, kmax, kzinv = ctx.saved_tensors
        sq, so = ctx.specs
        B, H, W, _ = xn.shape
        N = H * W
        dy = dy.contiguous()
        dx = torch.empty_like(xn)
        dctx = torch.empty_like(ctxm)
        call('pidm_linattn_block_bwd', xn, sq.wp_fwd, so.wp_fwd, dy, ctxm, kmax, kzinv, dx, dctx, B, N, stream())
        gq_buf, gq_ret = _grad_buffer(w_qkv)
        go_buf, go_ret = _grad_buffer(w_out)
        gb_buf, gb_ret = _grad_buffer(b_out)
        ws = _wgrad_stream(xn, sq.wp_fwd, so.wp_fwd, dy, ctxm, dctx, kmax, kzinv)
        call('pidm_linattn_block_wgrad', xn, sq.wp_fwd, so.wp_fwd, dy, ctxm, dctx, kmax, kzinv, gq_buf, sq.w_stride_n,
             sq.w_stride_c, go_buf, so.w_stride_n, so.w_stride_c, B, N, ws)
        call('pidm_colsum', dy, gb_buf, B * N, dy.shape[-1], _code(dy), ws)
        return (dx if ctx.needs_input_grad[0] else None), gq_ret, None, go_ret, gb_ret, None, dy, None


def linear_attention_block_supported(xn, spec_qkv, spec_out, b_out, heads):
    B, H, W, C = xn.shape
    return (_STATE['use_tc'] and xn.is_cuda and b_out is not None
            and spec_qkv.kh == 1 and spec_qkv.kw == 1 and spec_qkv.cout == 3 * heads * 32
            and spec_out.kh == 1 and spec_out.kw == 1 and not spec_out.transposed
            and spec_out.cin == heads * 32 and spec_out.cout == C
            and bool(call('pidm_linattn_block_supported', C, heads, H * W, _code(xn))))


def linear_attention_block(xn, w_qkv, spec_qkv, w_out, b_out, spec_out, residual, heads):
    """y = residual + to_out(linear_attention(to_qkv(xn))); to_qkv 1x1 without bias, to_out 1x1 256 -> C with bias."""
    return _LinAttnBlock.apply(xn.contiguous(), w_qkv, spec_qkv, w_out, b_out, spec_out, residual.contiguous(), heads)


def linear_attention(qkv, heads):
    return _LinAttn.apply(qkv.contiguous(), heads)


class _Attn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, heads):
        B, H, W, C3 = qkv.shape
        out = torch.empty(B, H, W, heads * 32, device=qkv.device, dtype=qkv.dtype)
        call('pidm_attn_fwd', qkv, out, B, H * W, heads, _code(qkv), stream())
        ctx.save_for_backward(qkv)
        ctx.heads = heads
        return out

    @staticmethod
    def backward(ctx, dout):
        (qkv,) = ctx.saved_tensors
        B, H, W, _ = qkv.shape
        dqkv = torch.empty_like(qkv)
        call('pidm_attn_bwd', qkv, dout.contiguous(), dqkv, B, H * W, ctx.heads, _code(qkv), stream())
        return dqkv, None


def softmax_attention(qkv, heads):
    return _Attn.apply(qkv.contiguous(), heads)


# ----------------------------------------------------------------------------------------------
# time conditioning
# ----------------------------------------------------------------------------------------------
class _TimeEmbed(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t, W1, b1, W2, b2):
        B = t.shape[0]
        td, dim = W1.shape
        dev = W1.device
        emb = torch.empty(B, dim, device=dev, dtype=torch.float32)
        h1 = torch.empty(B, td, device=dev, dtype=torch.float32)
        temb = torch.empty_like(h1)
        silu_t = torch.empty_like(h1)
        call('pidm_time_embed_fwd', t, W1, b1, W2, b2, emb, h1, temb, silu_t, B, dim, td, stream())
        ctx.save_for_backward(emb, h1, temb, W1, b1, W2, b2)
        ctx.mark_non_differentiable(temb)
        return silu_t, temb

    @staticmethod
    def backward(ctx, d_silu, _unused):
        emb, h1, temb, W1, b1, W2, b2 = ctx.saved_tensors
        B, td = h1.shape
        gW1, rW1 = _grad_buffer(W1)
        gb1, rb1 = _grad_buffer(b1)
        gW2, rW2 = _grad_buffer(W2)
        gb2, rb2 = _grad_buffer(b2)
        d_silu = d_silu.contiguous()
        ws = torch.empty(2 * B * td, device=h1.device, dtype=torch.float32)
        args = (d_silu, emb, h1, temb, W2, gW1, gb1, gW2, gb2, ws, B, emb.shape[1], td)
        call('pidm_time_embed_bwd', *args, 2, stream())                      # activation gradients (critical path)
        # weight gradients feed the optimizer only.  EVERY tensor the side-stream kernel reads must be kept alive until
        # the join: autograd releases this node's saved tensors (emb, h1) as soon as backward returns, and the caching
        # allocator would hand their memory to the next main-stream allocation while the kernel is still reading it
        call('pidm_time_embed_bwd', *args, 1, _wgrad_stream(ws, emb, h1))
        return None, rW1, rb1, rW2, rb2


def time_embed(t, W1, b1, W2, b2):
    """Returns (SiLU(time_mlp(t)), time_mlp(t)); the second output is for inspection only."""
    return _TimeEmbed.apply(t.to(torch.int64).contiguous(), W1, b1, W2, b2)


class _BlockMlps(torch.autograd.Function):
    """All ResnetBlock time-MLPs in one launch.  `table` is a MlpTable (packing.py); one output per block."""

    @staticmethod
    def forward(ctx, silu_t, table, *wb):
        B, td = silu_t.shape
        outs = [torch.empty(B, n, device=silu_t.device, dtype=torch.float32) for n in table.rows]
        call('pidm_block_mlps_fwd', table.device_table(outs), table.n, table.max_rows, silu_t, B, td, stream())
        ctx.save_for_backward(silu_t, *wb)
        ctx.table = table
        return tuple(outs)

    @staticmethod
    def backward(ctx, *d_outs):
        silu_t, *wb = ctx.saved_tensors
        table = ctx.table
        B, td = silu_t.shape
        bufs, rets = [], []
        for p in wb:
            b_, r_ = _grad_buffer(p)
            bufs.append(b_)
            rets.append(r_)
        d_outs = [d.contiguous() for d in d_outs]
        d_silu = torch.empty_like(silu_t)
        tab = table.device_table(None, d_outs, bufs)
        # (side stream: keep silu_t -- a saved tensor, released when this backward returns -- the incoming gradients
        #  and the device table alive until the join, see _TimeEmbed.backward)
        call('pidm_block_mlps_bwd', tab, table.n, table.max_rows, silu_t, d_silu, B, td, 1,
             _wgrad_stream(silu_t, tab, *d_outs))
        call('pidm_block_mlps_bwd', tab, table.n, table.max_rows, silu_t, d_silu, B, td, 2, stream())
        return (d_silu, None, *rets)


def block_mlps(silu_t, table):
    """-> tuple of [B, 2*C_out] tensors (scale | shift), one per ResnetBlock with a time MLP."""
    return _BlockMlps.apply(silu_t, table, *table.params)


# ----------------------------------------------------------------------------------------------
# output head (1x1 conv to NCHW fp32, optional sigmoid on the last channel)
# ----------------------------------------------------------------------------------------------
class _Head(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, sigmoid_last):
        B, H, W, C = x.shape
        O = w.shape[0]
        y = torch.empty(B, O, H, W, device=x.device, dtype=torch.float32)
        call('pidm_head_fwd', x, w, b, y, B, H * W, C, O, int(sigmoid_last), _code(x), stream())
        ctx.save_for_backward(x, w, b, y)
        ctx.sig = int(sigmoid_last)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, b, y = ctx.saved_tensors
        B, H, W, C = x.shape
        O = w.shape[0]
        dx = torch.empty_like(x)
        gw, rw = _grad_buffer(w)
        gb, rb = _grad_buffer(b)
        call('pidm_head_bwd', x, w, y, dy.contiguous().float(), dx, gw, gb, B, H * W, C, O, ctx.sig, _code(x), stream())
        return dx, rw, rb, None


def head(x, w, b, sigmoid_last=False):
    return _Head.apply(x.contiguous(), w, b, sigmoid_last)


# ----------------------------------------------------------------------------------------------
# diffusion element-wise + Darcy residual / loss
# ----------------------------------------------------------------------------------------------
def q_sample(x0, noise, t, sqrt_ab, sqrt_1mab):
    _need_cuda(x0, noise, t)
    _need_f32(sqrt_ab=sqrt_ab, sqrt_1mab=sqrt_1mab)
    x0 = x0.contiguous().float()
    xt = torch.empty_like(x0)
    call('pidm_qsample', x0, noise.contiguous().float(), t.to(torch.int64).contiguous(), sqrt_ab, sqrt_1mab, xt,
         x0.shape[0], x0[0].numel(), stream())
    return xt


def posterior_step(x_t, x0_pred, z, c1, c2, sigma):
    out = torch.empty_like(x_t)
    call('pidm_posterior_step', x_t.contiguous(), x0_pred.contiguous(), z.contiguous(), out, float(c1), float(c2),
         float(sigma), x_t.numel(), stream())
    return out


def mech_sample_input(x, planes, out):
    """U-Net input of a conditional sampling step of the topology-optimisation model, written into `out`
    [B,3+nc,P,P]: the sample x [B,3,P+1,P+1] resized to P x P, then the constant planes [B,nc,P,P]."""
    _need_cuda(x, planes, out)
    _need_f32(x=x, planes=planes, out=out)
    B, nc, P, _ = planes.shape
    assert x.shape == (B, 3, P + 1, P + 1) and out.shape == (B, 3 + nc, P, P), (x.shape, planes.shape, out.shape)
    call('pidm_mech_sample_input', x.contiguous(), planes.contiguous(), out, B, nc, P, stream())
    return out


def mech_posterior_step(y, x, z, t, c1, c2, sigma, out):
    """Posterior step of the topology-optimisation sampler from the network output y [B,3,P,P], written into `out`
    [B,3,P+1,P+1] (may be x): c1[t] model_out + c2[t] x + sigma[t] z, model_out = (u_x, u_y resized to P+1, rho
    zero-padded); t [B] int64 stays on the device."""
    _need_cuda(y, x, z, t, out)
    _need_f32(y=y, x=x, z=z, c1=c1, c2=c2, sigma=sigma)
    B, _, P, _ = y.shape
    assert x.shape == out.shape == z.shape == (B, 3, P + 1, P + 1) and t.dtype == torch.int64, (x.shape, y.shape, t.dtype)
    call('pidm_mech_posterior_step', y.contiguous(), x.contiguous(), z.contiguous(), t, c1, c2, sigma, out, B, P, stream())
    return out


class _DarcyResidual(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0hat, f_s, geom):
        B, C, P, _ = x0hat.shape
        r = torch.empty(B, P * P, 3, device=x0hat.device, dtype=torch.float32)
        call('pidm_darcy_residual_fwd', x0hat, f_s, r, B, P, *geom, stream())
        ctx.save_for_backward(x0hat, f_s)
        ctx.geom = geom
        return r

    @staticmethod
    def backward(ctx, gr):
        x0hat, f_s = ctx.saved_tensors
        B, C, P, _ = x0hat.shape
        gx = torch.empty_like(x0hat)
        call('pidm_darcy_residual_bwd', x0hat, f_s, gr.contiguous(), gx, B, P, *ctx.geom, stream())
        return gx, None, None


DARCY_PIXELS_AT_BOUNDARY = 1      # flag bits of the Darcy C ABI (pidm.h)
DARCY_PERIODIC = 2


def darcy_flags(pixels_at_boundary, periodic=False):
    """The flags word of the Darcy entry points: pixels_at_boundary (bit 0) and bcs='periodic' (bit 1)."""
    return (DARCY_PIXELS_AT_BOUNDARY if pixels_at_boundary else 0) | (DARCY_PERIODIC if periodic else 0)


def darcy_residual(x0hat, f_s, domain_length=1.0, reverse_d1=True, pixels_at_boundary=True, periodic=False):
    _need_cuda(x0hat)
    _need_f32(f_s=f_s)
    assert x0hat.shape[1] == 2, 'Darcy fields are (p, K)'
    return _DarcyResidual.apply(x0hat.contiguous().float(), f_s,
                                (float(domain_length), int(reverse_d1), darcy_flags(pixels_at_boundary, periodic)))


class _DarcyPidmLoss(torch.autograd.Function):
    """loss = c_data * mean_b(p2[t_b] mse_b) + mean(c_res * 0.5 r^2 / var_t); residual never materialised.
    The gradient is produced in the forward pass (one kernel) and only scaled in backward.
    model_out=None means "the data term uses x0hat itself" (x0_estimation: mean)."""

    @staticmethod
    def forward(ctx, x0hat, model_out, target, t, f_s, p2w, pvar, c_data, c_res, geom):
        B, C, P, _ = x0hat.shape
        same = model_out is None
        sums = torch.empty(3, device=x0hat.device, dtype=torch.float32)
        need = x0hat.requires_grad or (model_out is not None and model_out.requires_grad)
        gx = torch.empty_like(x0hat) if need else None
        gm = None if (same or not need) else torch.empty_like(model_out)
        call('pidm_darcy_pidm_loss', x0hat, x0hat if same else model_out, target, f_s, t, p2w, pvar, float(c_data),
             float(c_res), sums, gx, gm, B, P, *geom, stream())
        ctx.save_for_backward(gx, gm)
        ctx.mark_non_differentiable(sums)
        return sums[0] + sums[1], sums

    @staticmethod
    def backward(ctx, g, _unused):
        gx, gm = ctx.saved_tensors
        g = g.contiguous().float()
        # out of place: the saved gradients stay intact, so a second backward (retain_graph) scales the originals again
        ox = torch.empty_like(gx)
        call('pidm_scale', gx, g, ox, gx.numel(), stream())
        om = None
        if gm is not None:
            om = torch.empty_like(gm)
            call('pidm_scale', gm, g, om, gm.numel(), stream())
        return ox, om, None, None, None, None, None, None, None, None


def darcy_pidm_loss(x0hat, model_out, target, t, f_s, p2w, pvar, c_data, c_res, domain_length=1.0, reverse_d1=True,
                    pixels_at_boundary=True, periodic=False):
    """Returns (loss, sums) with sums = [data_loss, residual_loss, mean|r|] on the device."""
    _need_cuda(x0hat, target)
    _need_f32(f_s=f_s, p2w=p2w, pvar=pvar)
    geom = (float(domain_length), int(reverse_d1), darcy_flags(pixels_at_boundary, periodic))
    if model_out is not None and model_out is x0hat:
        model_out = None
    return _DarcyPidmLoss.apply(x0hat.contiguous().float(),
                                None if model_out is None else model_out.contiguous().float(),
                                target.contiguous().float(), t.to(torch.int64).contiguous(), f_s, p2w, pvar, c_data, c_res,
                                geom)
