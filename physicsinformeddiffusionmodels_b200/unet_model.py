"""`Unet3D` with the reference's constructor, state_dict and call surface (reference
src/unet_model.py:406-623), executed entirely by libpidm CUDA kernels on NHWC activations.

The module tree exists to own the parameters under the reference's 317 state_dict keys (including the
members the reference forward never touches: temporal attentions, rotary freqs, relative position bias,
signal embedding, to_q/to_k/to_v side projections, emb_conv/combine_conv).  Standard torch.nn layers are
used as PARAMETER HOLDERS ONLY -- constructed in the reference's order so that the same seed gives the same
initial weights -- their forward() is never called.  `Unet3D.forward` drives the kernels through ops.py.
"""
import math

import torch
from torch import nn

from . import ops
from .packing import ConvSpec, MlpTable, WeightPacker


def exists(x):
    return x is not None


def default(val, d):
    if exists(val):
        return val
    return d() if callable(d) else d


def _round_up(x, m):
    return (x + m - 1) // m * m


def draw_null_mask(B, prob, device, draw_shard=None):
    """The classifier-free mask of the reference's prob_mask_like (unet_model.py:63-69): [B] bool, True = the sample's
    conditioning is dropped.  draw_shard=(rank, world): drawn for the global batch of world * B samples and this rank's
    rows sliced out, so ranks with identical generator states consume the draw of the one-process run."""
    if prob == 1:
        return torch.ones(B, device=device, dtype=torch.bool)
    if prob == 0:
        return torch.zeros(B, device=device, dtype=torch.bool)
    rank, world = draw_shard if draw_shard is not None else (0, 1)
    return (torch.zeros(B * world, device=device).float().uniform_(0, 1) < prob)[rank * B:(rank + 1) * B]


# ---- parameter holders (names = reference attribute names) ---------------------------------------------
class RotaryEmbedding(nn.Module):
    """Holder for the frozen `freqs` of rotary_embedding_torch.RotaryEmbedding (unet_model.py:439); the
    reference forward never rotates anything (temporal attention is skipped)."""

    def __init__(self, dim, theta=10000):
        super().__init__()
        freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: (dim // 2)].float() / dim))
        self.freqs = nn.Parameter(freqs, requires_grad=False)


class RelativePositionBias(nn.Module):
    def __init__(self, heads=8, num_buckets=32, max_distance=128):
        super().__init__()
        self.relative_attention_bias = nn.Embedding(num_buckets, heads)


class LayerNorm(nn.Module):
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.gamma = nn.Parameter(torch.ones(1, dim, 1, 1, 1))


class PreNorm(nn.Module):
    def __init__(self, dim, fn):
        super().__init__()
        self.fn = fn
        self.norm = LayerNorm(dim)


class Residual(nn.Module):
    def __init__(self, fn):
        super().__init__()
        self.fn = fn


class EinopsToAndFrom(nn.Module):
    def __init__(self, fn):
        super().__init__()
        self.fn = fn


class Attention(nn.Module):
    """Softmax attention parameters (unet_model.py:317-339).  `to_out` is the bias-free Linear: in the
    reference the second assignment overwrites the Conv2d (which still consumed RNG, replicated here)."""

    def __init__(self, dim, heads=4, dim_head=32, rotary_emb=None, cond_dim=64):
        super().__init__()
        self.heads, self.dim_head = heads, dim_head
        hidden = dim_head * heads
        self.rotary_emb = rotary_emb
        self.to_qkv = nn.Linear(dim, hidden * 3, bias=False)
        self.to_q = nn.Linear(dim, hidden, bias=False)
        self.to_k = nn.Linear(cond_dim, hidden, bias=False)
        self.to_v = nn.Linear(cond_dim, hidden, bias=False)
        self.to_out = nn.Conv2d(hidden, dim, 1)
        self.to_out = nn.Linear(hidden, dim, bias=False)


class SpatialLinearAttention(nn.Module):
    def __init__(self, dim, heads=4, dim_head=32, cond_dim=64):
        super().__init__()
        self.heads = heads
        hidden = dim_head * heads
        self.to_qkv = nn.Conv2d(dim, hidden * 3, 1, bias=False)
        self.to_q = nn.Conv2d(dim, hidden, 1, bias=False)
        self.to_k = nn.Linear(cond_dim, hidden, bias=False)
        self.to_v = nn.Linear(cond_dim, hidden, bias=False)
        self.to_out = nn.Conv2d(hidden, dim, 1)


class Block(nn.Module):
    def __init__(self, dim, dim_out, groups=8):
        super().__init__()
        self.proj = nn.Conv3d(dim, dim_out, (1, 3, 3), padding=(0, 1, 1))
        self.norm = nn.GroupNorm(groups, dim_out)


class ResnetBlock(nn.Module):
    def __init__(self, dim, dim_out, *, time_emb_dim=None, groups=8):
        super().__init__()
        self.mlp = nn.Sequential(nn.SiLU(), nn.Linear(time_emb_dim, dim_out * 2)) if exists(time_emb_dim) else None
        self.block1 = Block(dim, dim_out, groups=groups)
        self.block2 = Block(dim_out, dim_out, groups=groups)
        self.res_conv = nn.Conv3d(dim, dim_out, 1) if dim != dim_out else nn.Identity()
        self.groups = groups


class CircularUpsample(nn.Module):
    """Holder for the circular up-sampling layer (unet_model.py:161-194): the reference pads by 2 circularly and runs a
    ConvTranspose3d with padding 5; its state_dict keys are `conv_transpose.weight|bias`.  The engine runs it as the
    periodic 4x4/stride-2 transposed convolution over a 1-pixel wrapped halo (ops._halo_geometry)."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.conv_transpose = nn.ConvTranspose3d(in_channels, out_channels, (1, 4, 4), (1, 2, 2), padding=(0, 5, 5))


def _up_conv(up):
    """the ConvTranspose3d that holds an up-sampling layer's parameters"""
    return up.conv_transpose if isinstance(up, CircularUpsample) else up


class SignalEmbedding(nn.Module):
    """Holder for sign_emb_CNN (unet_model.py:370-404, only used by an ablation that forward never reaches)."""

    def __init__(self, init_channel, channel_upsamplings):
        super().__init__()
        scale = [init_channel, *channel_upsamplings]
        mods = []
        for ci, co in zip(scale[:-1], scale[1:]):
            mods += [nn.Conv1d(ci, co, kernel_size=4, stride=2, padding=1), nn.SiLU()]
        self.emb_model = nn.Sequential(*mods)


class Unet3D(nn.Module):
    def __init__(self, dim, out_dim=None, dim_mults=(1, 2, 4, 8), channels=2, self_condition=False, attn_heads=8,
                 attn_dim_head=32, init_dim=None, init_kernel_size=7, use_sparse_linear_attn=True, resnet_groups=8,
                 cond_bias=False, cond_attention='none', cond_attention_tokens=6, cond_to_time='add',
                 padding_mode='zeros', sigmoid_last_channel=False):
        super().__init__()
        if padding_mode not in ('zeros', 'circular'):
            raise ValueError('Unknown padding mode: {}'.format(padding_mode))
        if not use_sparse_linear_attn:
            raise NotImplementedError('use_sparse_linear_attn=False is not used by the reference drivers')
        if attn_dim_head != 32:
            raise NotImplementedError('attention kernels are built for dim_head = 32 (reference default)')
        if self_condition:
            raise NotImplementedError('self_condition=True is not used by the reference drivers')
        assert init_kernel_size % 2 == 1
        self.input_channels = channels
        self.self_condition = self_condition
        self.dim = dim
        time_dim = dim * 4
        self.cond_dim = time_dim
        self.cond_to_time = cond_to_time
        self.padding_mode = padding_mode
        self.heads = attn_heads
        self.groups = resnet_groups
        self.init_kernel_size = init_kernel_size

        # ---- parameter holders, in the reference construction order (unet_model.py:438-526) ----
        rotary_emb = RotaryEmbedding(min(32, attn_dim_head))

        def temporal_attn(d):
            return EinopsToAndFrom(Attention(d, heads=attn_heads, dim_head=attn_dim_head, rotary_emb=rotary_emb,
                                             cond_dim=self.cond_dim))
        self.time_rel_pos_bias = RelativePositionBias(heads=attn_heads, max_distance=32)
        init_dim = default(init_dim, dim)
        pad = init_kernel_size // 2
        self.init_conv = nn.Conv3d(channels, init_dim, (1, init_kernel_size, init_kernel_size), padding=(0, pad, pad))
        self.init_temporal_attn = Residual(PreNorm(init_dim, temporal_attn(init_dim)))
        dims = [init_dim, *map(lambda m: dim * m, dim_mults)]
        in_out = list(zip(dims[:-1], dims[1:]))
        self.time_mlp = nn.Sequential(nn.Identity(), nn.Linear(dim, time_dim), nn.GELU(), nn.Linear(time_dim, time_dim))
        self.sign_emb_CNN = SignalEmbedding(1, (16, 32, 64, 128, self.cond_dim))
        self.downs = nn.ModuleList([])
        self.ups = nn.ModuleList([])
        n_res = len(in_out)
        tdim = time_dim + int(self.cond_dim or 0) if cond_to_time == 'concat' else self.cond_dim

        def rb(a, b, time=True):
            return ResnetBlock(a, b, time_emb_dim=tdim if time else None, groups=resnet_groups)

        def lin_attn(d):
            return Residual(PreNorm(d, SpatialLinearAttention(d, heads=attn_heads, cond_dim=self.cond_dim)))
        for ind, (di, do) in enumerate(in_out):
            is_last = ind >= (n_res - 1)
            self.downs.append(nn.ModuleList([
                rb(di, do), rb(do, do), lin_attn(do),
                nn.Conv3d(do, do, (1, 4, 4), (1, 2, 2), (0, 1, 1)) if not is_last else nn.Identity()]))
        mid = dims[-1]
        self.mid_block1 = rb(mid, mid)
        spatial_attn = EinopsToAndFrom(Attention(mid, heads=attn_heads, cond_dim=self.cond_dim))
        self.mid_spatial_attn = Residual(PreNorm(mid, spatial_attn))
        self.mid_temporal_attn = Residual(PreNorm(mid, temporal_attn(mid)))
        self.mid_block2 = rb(mid, mid)
        def upsample(d):
            if padding_mode == 'circular':
                return CircularUpsample(d, d)
            return nn.ConvTranspose3d(d, d, (1, 4, 4), (1, 2, 2), (0, 1, 1))
        for ind, (di, do) in enumerate(reversed(in_out)):
            is_last = ind >= (n_res - 1)
            self.ups.append(nn.ModuleList([
                rb(do * 2, di), rb(di, di), lin_attn(di), upsample(di) if not is_last else nn.Identity()]))
        out_dim = default(out_dim, channels)
        self.out_dim = out_dim
        self.final_conv = nn.Sequential(rb(dim * 2, dim, time=False), nn.Conv3d(dim, out_dim, 1))
        self.emb_conv = nn.Sequential(nn.Conv2d(channels, init_dim, kernel_size=1), nn.GELU(),
                                      nn.Conv2d(init_dim, init_dim, kernel_size=3, padding=1))
        self.combine_conv = nn.Conv2d(init_dim * 2, init_dim, kernel_size=1)
        self.sigmoid_last_channel = sigmoid_last_channel

        self._build_plan()

    # ---- execution plan: conv specs + tables over the holders above -----------------------------------
    def _build_plan(self):
        pk = WeightPacker()
        self._packer = pk
        # the 2-channel (10 for mechanics) input is zero-padded to 32 channels so that the 7x7 stem runs on the
        # tensor-core kernels too (K step = 32 channels = one 64-byte swizzle span)
        self._cin_pad = _round_up(self.input_channels, 32)
        k = self.init_kernel_size
        self._spec = {}

        # padding_mode='circular' reaches every padded spatial convolution except emb_conv[2], which the reference
        # hard-codes to zero padding (unet_model.py:524)
        circ = self.padding_mode == 'circular'

        def conv(mod, kh, stride, pad, kind='conv', cin_pad=None, need_dgrad=True, circular=circ):
            s = pk.add(ConvSpec(mod.weight, kind, kh, kh, stride, pad, cin_pad=cin_pad, need_dgrad=need_dgrad,
                                circular=circular))
            self._spec[id(mod)] = s
            return s
        conv(self.init_conv, k, 1, k // 2, cin_pad=self._cin_pad, need_dgrad=False)
        mlps = []

        def plan_rb(block):
            conv(block.block1.proj, 3, 1, 1)
            conv(block.block2.proj, 3, 1, 1)
            if not isinstance(block.res_conv, nn.Identity):
                conv(block.res_conv, 1, 1, 0)
            if block.mlp is not None:
                block._mlp_index = len(mlps)
                mlps.append(block.mlp[1])

        def plan_la(res):
            conv(res.fn.fn.to_qkv, 1, 1, 0)
            conv(res.fn.fn.to_out, 1, 1, 0)
        self._early_specs = 0
        for b1, b2, la, down in self.downs:
            plan_rb(b1); plan_rb(b2); plan_la(la)
            if self._early_specs == 0:
                self._early_specs = len(pk.specs)      # stem + first resolution level: packed by a first launch
            if not isinstance(down, nn.Identity):
                conv(down, 4, 2, 1)
        plan_rb(self.mid_block1)
        att = self.mid_spatial_attn.fn.fn.fn
        conv(att.to_qkv, 1, 1, 0)
        conv(att.to_out, 1, 1, 0)
        plan_rb(self.mid_block2)
        for b1, b2, la, up in self.ups:
            plan_rb(b1); plan_rb(b2); plan_la(la)
            if not isinstance(up, nn.Identity):
                conv(_up_conv(up), 4, 2, 1, kind='convT')
        plan_rb(self.final_conv[0])
        # residual-gradient guidance branch (only executed when forward() is given cond=..., reference :585-603);
        # emb_conv[0] (1x1, 2 channels in) runs fused with its GELU in ops.cond_embed, from the fp32 cond
        conv(self.emb_conv[2], 3, 1, 1, circular=False)
        conv(self.combine_conv, 1, 1, 0)
        self._mlp_table = MlpTable(mlps)

    def unused_parameter_names(self, guidance=False):
        """Trainable parameters that Unet3D.forward never touches (they exist for state_dict parity with the reference:
        temporal attentions, relative position bias, signal embedding, the to_q / to_k / to_v side projections and,
        without residual-gradient guidance (cond=None: the configuration of model.yaml), emb_conv and combine_conv).
        They never receive a gradient -- in the reference their .grad stays None (checked against the reference-generated
        tests/golden/params_without_grad.txt and, guidance=True, params_without_grad_guidance.txt) -- so a data-parallel
        step need not exchange them."""
        dead = []
        prefixes = ('time_rel_pos_bias.', 'sign_emb_CNN.', 'init_temporal_attn.', 'mid_temporal_attn.')
        if not guidance:
            prefixes += ('emb_conv.', 'combine_conv.')
        for name, p in self.named_parameters():
            if not p.requires_grad:
                continue
            parts = name.split('.')
            if name.startswith(prefixes) or parts[-2] in ('to_q', 'to_k', 'to_v'):
                dead.append(name)
        return dead

    # ---- kernels ----------------------------------------------------------------------------------------
    # set by engine.TrainEngine: called during backward when the gradients of a parameter group are complete
    _boundary_cb = None

    def _boundary(self, group, h):
        cb = self._boundary_cb
        if cb is not None and h.requires_grad:
            h.register_hook(lambda g, _cb=cb, _k=group: _cb(_k))       # returns None: the gradient is left untouched
        return h

    def _conv(self, mod, x, residual=None, gn_link=None, skip=None):
        return ops.conv2d(x, mod.weight, getattr(mod, 'bias', None), self._spec[id(mod)], residual=residual,
                          gn_link=gn_link, skip=skip)

    def _resblock(self, block, x, ss_list):
        ss = ss_list[block._mlp_index] if (block.mlp is not None and ss_list is not None) else None
        # conv -> GroupNorm pairs are linked: statistics come out of the conv epilogue, the conv's bias gradient
        # out of the GroupNorm backward
        l1, l2 = {'groups': block.groups}, {'groups': block.groups}
        # x feeds both the first conv and the residual branch: the residual branch parks its gradient (ops._Stash /
        # a 'park' conv) and the first conv's dgrad adds it in its epilogue -- no separate accumulation kernel
        sk = {}
        h = self._conv(block.block1.proj, x, gn_link=l1, skip=('take', sk))
        h = ops.groupnorm_silu(h, block.block1.norm.weight, block.block1.norm.bias, ss, block.groups,
                               block.block1.norm.eps, gn_link=l1)
        h = self._conv(block.block2.proj, h, gn_link=l2)
        if isinstance(block.res_conv, nn.Identity):       # `+ x` rides on the GroupNorm/SiLU pass
            return ops.groupnorm_silu(h, block.block2.norm.weight, block.block2.norm.bias, None, block.groups,
                                      block.block2.norm.eps, gn_link=l2, residual=ops.stash_grad(x, sk))
        h = ops.groupnorm_silu(h, block.block2.norm.weight, block.block2.norm.bias, None, block.groups,
                               block.block2.norm.eps, gn_link=l2)
        return self._conv(block.res_conv, x, residual=h, skip=('park', sk))

    def _linear_attention(self, res, x):
        pre = res.fn
        sk = {}                                    # gradient of the `+ x` skip is added inside the LayerNorm backward
        xn = ops.layernorm_c(x, pre.norm.gamma, pre.norm.eps, skip_link=sk)
        to_qkv = pre.fn.to_qkv
        spec = self._spec[id(to_qkv)]
        to_out = pre.fn.to_out
        b_out = getattr(to_out, 'bias', None)
        if (getattr(to_qkv, 'bias', None) is None
                and ops.linear_attention_block_supported(xn, spec, self._spec[id(to_out)], b_out, pre.fn.heads)):
            # to_qkv, the attention, to_out and the `+ x`: the [B, N, 256] attention output is never materialised
            return ops.linear_attention_block(xn, to_qkv.weight, spec, to_out.weight, b_out, self._spec[id(to_out)],
                                              ops.stash_grad(x, sk), pre.fn.heads)
        qkv = self._conv(to_qkv, xn)
        a = ops.linear_attention(qkv, pre.fn.heads)
        return self._conv(to_out, a, residual=ops.stash_grad(x, sk))

    def _mid_attention(self, res, x):
        pre = res.fn
        att = pre.fn.fn
        sk = {}
        xn = ops.layernorm_c(x, pre.norm.gamma, pre.norm.eps, skip_link=sk)
        qkv = self._conv(att.to_qkv, xn)
        a = ops.softmax_attention(qkv, att.heads)
        return self._conv(att.to_out, a, residual=ops.stash_grad(x, sk))

    def forward_with_guidance_scale(self, *args, **kwargs):
        """classifier-free guidance at sampling time (reference :530-540): null + (cond - null) * scale"""
        from .denoising_utils import _axpby
        guidance_scale = kwargs.pop('guidance_scale', 3.)
        logits = self.forward(*args, null_cond_prob=0., **kwargs)
        if guidance_scale == 1:
            return logits
        null_logits = self.forward(*args, null_cond_prob=1., **kwargs)
        B = logits.shape[0]
        full = lambda v: torch.full((B,), float(v), device=logits.device, dtype=torch.float32)   # noqa: E731
        return _axpby(full(guidance_scale), logits, full(1. - guidance_scale), null_logits, full(0.), null_logits)

    # the classifier-free mask of the last guided forward, [B] bool, written in place (a CUDA-graph replay leaves the mask
    # it drew there)
    _null_mask_last = None

    def _cond_embedding(self, h, cond, null_cond_prob, draw_shard=None):
        """x <- combine_conv(cat(x, emb_conv(cond))) with cond zeroed for the samples drawn as "unconditional"
        (classifier-free guidance, reference :585-603).  cond [B, P*P, 2] is data (the residual gradient): no gradient."""
        if cond.dim() != 3:
            raise ValueError('Input must be [BxP*PxC].')
        B, N, _ = cond.shape
        P = int(math.isqrt(N))
        mask = getattr(self, '_null_mask_override', None)          # tests inject the reference's draw
        if mask is None:
            mask = draw_null_mask(B, null_cond_prob, cond.device, draw_shard)
        last = self._null_mask_last
        if last is None or last.shape != mask.shape or last.device != mask.device:
            last = self._null_mask_last = torch.empty(B, device=cond.device, dtype=torch.bool)
        last.copy_(mask)
        e = ops.cond_embed(cond, last, self.emb_conv[0].weight, self.emb_conv[0].bias, P)
        e = self._conv(self.emb_conv[2], e)
        return self._conv(self.combine_conv, ops.concat(h, e))

    def forward(self, x, time, x_self_cond=None, cond=None, null_cond_prob=0., draw_shard=None):
        """x: [B, P*P, C] (as handed over by the residual operators), [B, C, P, P] or [B, C, 1, P, P].
        Returns fp32 [B, out_dim, P, P] ([B, out_dim, 1, P, P] for 5-D input), reference :542-623.
        draw_shard=(rank, world): the classifier-free mask is drawn for the global batch and sliced (draw_null_mask)."""
        if exists(x_self_cond):
            raise NotImplementedError('self-conditioning is not used by the reference drivers')
        video = False
        if x.dim() == 3:
            B, N, C = x.shape
            P = int(math.isqrt(N))
            assert P * P == N, 'number of pixels must be a perfect square'
            x = x.reshape(B, P, P, C).permute(0, 3, 1, 2)
        elif x.dim() == 5:
            if x.shape[2] != 1:
                raise NotImplementedError('image sequences with F > 1 frames are not used by the reference drivers')
            x = x[:, :, 0]
            video = True
        elif x.dim() != 4:
            raise ValueError('Input must be image [BxCxPxP] or image sequence [BxCxFxPxP].')
        if not x.is_cuda:
            raise RuntimeError('Unet3D (CUDA engine) needs CUDA tensors: no CPU fallback on the product path')
        dt = ops.act_dtype()
        # the weight re-packing (one launch over all layers) runs on a forked stream and overlaps the input layout
        # change and the time-conditioning MLPs; it is joined before the first convolution
        # Inference (no_grad): the packed copy is reused as long as no parameter changed (tensor version counters;
        # engine.TrainEngine invalidates explicitly because its optimizer kernel writes the flat buffer directly), so a
        # 250-step sampling loop packs once instead of 250 times.
        pack_stream = ops.fork_stream()
        early_packed = None
        if torch.is_grad_enabled() or self._packer.stale(dt):
            with torch.cuda.stream(pack_stream):
                early_packed = self._packer.refresh(dt, early_specs=0 if exists(cond) else self._early_specs)
        # pre-zeroed scratch for the GroupNorm statistics that the conv epilogues accumulate (<= 64 norms)
        ops.zero_pool_begin(64 * (x.shape[0] * self.groups * 2 + 32), x.device)
        h = ops.nchw_to_nhwc(x.float(), self._cin_pad, dt)
        tm = self.time_mlp
        if time.dim() == 0:
            time = time.reshape(1).expand(x.shape[0])
        silu_t, _ = ops.time_embed(time, tm[1].weight, tm[1].bias, tm[3].weight, tm[3].bias)
        ss = ops.block_mlps(silu_t, self._mlp_table)
        # the stem and the first resolution level only need the first pack launch; the rest is joined below
        if early_packed is not None:
            torch.cuda.current_stream().wait_event(early_packed)
        else:
            torch.cuda.current_stream().wait_stream(pack_stream)
        h = self._conv(self.init_conv, h)
        if exists(cond):
            h = self._cond_embedding(h, cond, null_cond_prob, draw_shard)
        r = h
        skips = []
        for lvl, (b1, b2, la, down) in enumerate(self.downs):
            if lvl == 2:
                h = self._boundary(1, h)       # backward has finished downs[2:], mid (and everything after them)
            h = self._resblock(b1, h, ss)
            h = self._resblock(b2, h, ss)
            h = self._linear_attention(la, h)
            skips.append(h)
            if lvl == 0 and early_packed is not None:
                torch.cuda.current_stream().wait_stream(pack_stream)
            if not isinstance(down, nn.Identity):
                h = self._conv(down, h)
        h = self._resblock(self.mid_block1, h, ss)
        h = self._mid_attention(self.mid_spatial_attn, h)
        h = self._resblock(self.mid_block2, h, ss)
        h = self._boundary(2, h)               # backward has finished the up path and the output head
        for b1, b2, la, up in self.ups:
            h = ops.concat(h, skips.pop())
            h = self._resblock(b1, h, ss)
            h = self._resblock(b2, h, ss)
            h = self._linear_attention(la, h)
            if not isinstance(up, nn.Identity):
                h = self._conv(_up_conv(up), h)
        h = ops.concat(h, r)
        h = self._resblock(self.final_conv[0], h, None)
        fc = self.final_conv[1]
        y = ops.head(h, fc.weight, fc.bias, self.sigmoid_last_channel)
        ops.zero_pool_end()
        return y.unsqueeze(2) if video else y
