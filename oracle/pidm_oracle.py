"""CPU ORACLE for the physics-informed-diffusion hot path.  TEST INFRASTRUCTURE ONLY.

This file restates, in plain functional PyTorch (float32 or float64, CPU), the algorithm of the
reference hot path (jhbastek/PhysicsInformedDiffusionModels).  It is the checker for the CUDA
path: only `tests/`, `__graft_entry__.smoke()` and `bench.py` (cpu_baseline / `--impl reference`
legs) may import it.  The product package never imports anything from `oracle/`.

Pinned against the real reference: `oracle/make_golden.py` imports the untouched reference modules
from the original project (through the import shims in `oracle/ref_shims/`), runs them on seeded inputs
and writes `tests/golden/*.pt`; `tests/test_oracle_golden.py` checks every function below against
those fixtures.  Where the reference's own third-party dependency is absent (findiff stencil
tables, solidspy Q4 stiffness, the authors' mesh files) parity is pinned analytically only -- see
DESIGN.md "Oracle" for the list.

Each function cites the reference file:line it follows (paths relative to the original project's root).

The study options are arguments of the functions they change, so that they combine as in the product: `periodic`
(bcs='periodic') of the Darcy functions, cfg['padding_mode'] (Unet3D(padding_mode='circular')) of the U-Net, CoCoGen
corrections in `p_sample_loop`, and the conditional topology-optimisation sampler `mechanics_p_sample_loop`.  Their
defaults run the reference's default path.
"""
import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------------
# A1/A2  schedule tables            (src/denoising_utils.py:315-370, extract :302-306)
# --------------------------------------------------------------------------------------------


def golden_sample(t, n=8192):
    """Fixed, seeded sample of n elements of a flattened tensor (all of it when it is smaller).  The large activation
    taps and weight gradients in tests/golden are stored this way so that every fixture stays small; the tests compare
    the same elements of what they compute."""
    flat = t.reshape(-1)
    if flat.numel() <= n:
        return flat.clone()
    idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:n]
    return flat[idx.to(flat.device)]


def cosine_betas(n_steps, s=0.008):
    """Cosine schedule, denoising_utils.py:362-369 (float32 arithmetic exactly as the reference)."""
    x = torch.linspace(0, n_steps, n_steps + 1)
    ac = torch.cos(((x / n_steps) + s) / (1 + s) * torch.pi * 0.5) ** 2
    ac = ac / ac[0]
    betas = 1 - (ac[1:] / ac[:-1])
    return torch.clip(betas, 0, 0.999)


def diffusion_tables(n_steps):
    """The 18 derived tables of DenoisingDiffusion.create_diff_dict, denoising_utils.py:315-352."""
    d = OrderedDict()
    b = cosine_betas(n_steps)
    d['betas'] = b
    a = 1.0 - b
    d['alphas'] = a
    d['sqrt_recip_alphas'] = torch.sqrt(1.0 / a)
    ap = torch.cumprod(a, 0)
    d['alphas_prod'] = ap
    d['alphas_prod_p'] = torch.cat([torch.ones(1), ap[:-1]], 0)
    d['alphas_bar_sqrt'] = torch.sqrt(ap)
    d['sqrt_recip_alphas_cumprod'] = torch.sqrt(1.0 / ap)
    d['sqrt_recipm1_alphas_cumprod'] = torch.sqrt(1.0 / ap - 1)
    d['one_minus_alphas_bar_log'] = torch.log(1 - ap)
    d['one_minus_alphas_bar_sqrt'] = torch.sqrt(1 - ap)
    app = F.pad(ap[:-1], (1, 0), value=1.0)
    d['alphas_prod_prev'] = app
    d['posterior_mean_coef1'] = b * torch.sqrt(app) / (1.0 - ap)
    d['posterior_mean_coef2'] = (1.0 - app) * torch.sqrt(a) / (1.0 - ap)
    d['noise_mean_coeff'] = torch.sqrt(1.0 / a) * (1.0 - a) / torch.sqrt(1.0 - ap)
    pv = b * (1.0 - app) / (1.0 - ap)
    d['posterior_variance'] = pv
    pvc = pv.clone()
    pvc[0] = pv[1]
    d['posterior_variance_clipped'] = pvc
    d['posterior_log_variance_clipped'] = torch.log(pvc)
    snr = ap / (1.0 - ap)
    d['p2_loss_weight'] = torch.minimum(snr, torch.full_like(snr, 5.0))
    return d


def q_sample(x0, t, noise, tables):
    """x_t = sqrt(abar_t) x0 + sqrt(1-abar_t) eps, denoising_utils.py:373-378 / inline :633-638."""
    a = tables['alphas_bar_sqrt'].to(x0.dtype)[t].view(-1, *([1] * (x0.ndim - 1)))
    s = tables['one_minus_alphas_bar_sqrt'].to(x0.dtype)[t].view(-1, *([1] * (x0.ndim - 1)))
    return x0 * a + noise * s


# --------------------------------------------------------------------------------------------
# A6  Unet3D.forward, executed subset   (src/unet_model.py:542-623 and blocks :147-367)
# --------------------------------------------------------------------------------------------


def unet_config(dim=32, channels=2, out_dim=None, dim_mults=(1, 2, 4, 8), heads=8, dim_head=32,
                groups=8, sigmoid_last_channel=False, padding_mode='zeros'):
    return dict(dim=dim, channels=channels, out_dim=channels if out_dim is None else out_dim,
                dim_mults=tuple(dim_mults), heads=heads, dim_head=dim_head, groups=groups,
                sigmoid_last_channel=sigmoid_last_channel, padding_mode=padding_mode)


def _up_key(cfg, i):
    # with padding_mode='circular' the up-sampling layer is the periodic transposed-conv module (unet_model.py:164-194)
    return f'ups.{i}.3.conv_transpose' if cfg['padding_mode'] == 'circular' else f'ups.{i}.3'


def unet_param_shapes(cfg):
    """Every state_dict key of the reference Unet3D with its shape, in reference order
    (unet_model.py:406-528).  Includes the parameter holders that forward never touches.  The order, and so the weights
    make_test_state_dict draws, is the same for both padding modes; only the six up-sampling keys differ."""
    dim, ch, od = cfg['dim'], cfg['channels'], cfg['out_dim']
    hid = cfg['heads'] * cfg['dim_head']
    td = dim * 4
    S = OrderedDict()

    def temporal(prefix, c):
        S[prefix + '.fn.fn.fn.rotary_emb.freqs'] = (min(32, cfg['dim_head']) // 2,)
        S[prefix + '.fn.fn.fn.to_qkv.weight'] = (hid * 3, c)
        S[prefix + '.fn.fn.fn.to_q.weight'] = (hid, c)
        S[prefix + '.fn.fn.fn.to_k.weight'] = (hid, td)
        S[prefix + '.fn.fn.fn.to_v.weight'] = (hid, td)
        S[prefix + '.fn.fn.fn.to_out.weight'] = (c, hid)
        S[prefix + '.fn.norm.gamma'] = (1, c, 1, 1, 1)

    def resblock(prefix, ci, co, time=True):
        if time:
            S[prefix + '.mlp.1.weight'] = (co * 2, td)
            S[prefix + '.mlp.1.bias'] = (co * 2,)
        for b, c_in in (('block1', ci), ('block2', co)):
            S[f'{prefix}.{b}.proj.weight'] = (co, c_in, 1, 3, 3)
            S[f'{prefix}.{b}.proj.bias'] = (co,)
            S[f'{prefix}.{b}.norm.weight'] = (co,)
            S[f'{prefix}.{b}.norm.bias'] = (co,)
        if ci != co:
            S[prefix + '.res_conv.weight'] = (co, ci, 1, 1, 1)
            S[prefix + '.res_conv.bias'] = (co,)

    def linattn(prefix, c):
        S[prefix + '.fn.fn.to_qkv.weight'] = (hid * 3, c, 1, 1)
        S[prefix + '.fn.fn.to_q.weight'] = (hid, c, 1, 1)
        S[prefix + '.fn.fn.to_k.weight'] = (hid, td)
        S[prefix + '.fn.fn.to_v.weight'] = (hid, td)
        S[prefix + '.fn.fn.to_out.weight'] = (c, hid, 1, 1)
        S[prefix + '.fn.fn.to_out.bias'] = (c,)
        S[prefix + '.fn.norm.gamma'] = (1, c, 1, 1, 1)

    S['time_rel_pos_bias.relative_attention_bias.weight'] = (32, cfg['heads'])
    S['init_conv.weight'] = (dim, ch, 1, 7, 7)
    S['init_conv.bias'] = (dim,)
    temporal('init_temporal_attn', dim)
    S['time_mlp.1.weight'] = (td, dim)
    S['time_mlp.1.bias'] = (td,)
    S['time_mlp.3.weight'] = (td, td)
    S['time_mlp.3.bias'] = (td,)
    chans = [1, 16, 32, 64, 128, td]
    for i in range(5):
        S[f'sign_emb_CNN.emb_model.{2 * i}.weight'] = (chans[i + 1], chans[i], 4)
        S[f'sign_emb_CNN.emb_model.{2 * i}.bias'] = (chans[i + 1],)
    dims = [dim] + [dim * m for m in cfg['dim_mults']]
    in_out = list(zip(dims[:-1], dims[1:]))
    nres = len(in_out)
    for i, (ci, co) in enumerate(in_out):
        resblock(f'downs.{i}.0', ci, co)
        resblock(f'downs.{i}.1', co, co)
        linattn(f'downs.{i}.2', co)
        if i < nres - 1:
            S[f'downs.{i}.3.weight'] = (co, co, 1, 4, 4)
            S[f'downs.{i}.3.bias'] = (co,)
    for i, (ci, co) in enumerate(reversed(in_out)):
        resblock(f'ups.{i}.0', co * 2, ci)
        resblock(f'ups.{i}.1', ci, ci)
        linattn(f'ups.{i}.2', ci)
        if i < nres - 1:
            S[_up_key(cfg, i) + '.weight'] = (ci, ci, 1, 4, 4)
            S[_up_key(cfg, i) + '.bias'] = (ci,)
    mid = dims[-1]
    resblock('mid_block1', mid, mid)
    S['mid_spatial_attn.fn.fn.fn.to_qkv.weight'] = (hid * 3, mid)
    S['mid_spatial_attn.fn.fn.fn.to_q.weight'] = (hid, mid)
    S['mid_spatial_attn.fn.fn.fn.to_k.weight'] = (hid, td)
    S['mid_spatial_attn.fn.fn.fn.to_v.weight'] = (hid, td)
    S['mid_spatial_attn.fn.fn.fn.to_out.weight'] = (mid, hid)
    S['mid_spatial_attn.fn.norm.gamma'] = (1, mid, 1, 1, 1)
    temporal('mid_temporal_attn', mid)
    resblock('mid_block2', mid, mid)
    resblock('final_conv.0', dim * 2, dim, time=False)
    S['final_conv.1.weight'] = (od, dim, 1, 1, 1)
    S['final_conv.1.bias'] = (od,)
    S['emb_conv.0.weight'] = (dim, ch, 1, 1)
    S['emb_conv.0.bias'] = (dim,)
    S['emb_conv.2.weight'] = (dim, dim, 3, 3)
    S['emb_conv.2.bias'] = (dim,)
    S['combine_conv.weight'] = (dim, dim * 2, 1, 1)
    S['combine_conv.bias'] = (dim,)
    return S


def make_test_state_dict(cfg, seed=0, dtype=torch.float32):
    """Deterministic, architecture-shaped random weights (CPU generator) used by the golden script
    and by the tests so that no 40 MB checkpoint has to be committed.  Fan-in scaled so activations
    stay O(1); norm gains near 1, biases small but NON-zero so every term is exercised."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for k, shp in unet_param_shapes(cfg).items():
        if k.endswith('rotary_emb.freqs'):
            n = shp[0] * 2
            sd[k] = 1.0 / (10000 ** (torch.arange(0, n, 2)[: n // 2].float() / n))
        elif k.endswith('norm.gamma') or k.endswith('norm.weight'):
            sd[k] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith('.bias'):
            sd[k] = 0.05 * torch.randn(shp, generator=g)
        else:
            fan_in = 1
            for s in shp[1:]:
                fan_in *= s
            sd[k] = torch.randn(shp, generator=g) / math.sqrt(max(fan_in, 1))
        sd[k] = sd[k].to(dtype)
    return sd


def _gn_silu(x, w, b, groups, scale_shift=None):
    # Block.forward, unet_model.py:233-241
    x = F.group_norm(x, groups, w, b, eps=1e-5)
    if scale_shift is not None:
        sc, sh = scale_shift
        x = x * (sc + 1) + sh
    return F.silu(x)


def _conv(x, w, b, pad, padding_mode, stride=1):
    # a padded Conv3d on F=1 frames; padding_mode='circular' wraps the pad (unet_model.py:196,226,452)
    if padding_mode == 'circular':
        return F.conv2d(F.pad(x, (pad,) * 4, mode='circular'), w, b, stride=stride)
    return F.conv2d(x, w, b, stride=stride, padding=pad)


def conv_transpose_circular(x, w, b):
    """The periodic 4x4 / stride-2 up-sampling of padding_mode='circular' (unet_model.py:164-194): circular pad 1, then
    conv_transpose2d with padding 3 -- equal to the reference's pad 2 / padding 5."""
    return F.conv_transpose2d(F.pad(x, (1,) * 4, mode='circular'), w, b, stride=2, padding=3)


def _resblock(sd, p, x, temb, groups, padding_mode='zeros'):
    # ResnetBlock.forward, unet_model.py:255-267
    ss = None
    if temb is not None and (p + '.mlp.1.weight') in sd:
        e = F.linear(F.silu(temb), sd[p + '.mlp.1.weight'], sd[p + '.mlp.1.bias'])
        ss = e[:, :, None, None].chunk(2, dim=1)
    h = _conv(x, sd[p + '.block1.proj.weight'][:, :, 0], sd[p + '.block1.proj.bias'], 1, padding_mode)
    h = _gn_silu(h, sd[p + '.block1.norm.weight'], sd[p + '.block1.norm.bias'], groups, ss)
    h = _conv(h, sd[p + '.block2.proj.weight'][:, :, 0], sd[p + '.block2.proj.bias'], 1, padding_mode)
    h = _gn_silu(h, sd[p + '.block2.norm.weight'], sd[p + '.block2.norm.bias'], groups)
    if (p + '.res_conv.weight') in sd:
        x = F.conv2d(x, sd[p + '.res_conv.weight'][:, :, 0], sd[p + '.res_conv.bias'])
    return h + x


def _chan_layernorm(x, gamma, eps=1e-5):
    # LayerNorm.forward, unet_model.py:207-210 (biased variance, gain only)
    var = x.var(dim=1, unbiased=False, keepdim=True)
    mean = x.mean(dim=1, keepdim=True)
    return (x - mean) / (var + eps).sqrt() * gamma.reshape(1, -1, 1, 1)


def _linear_attention(sd, p, x, heads, dim_head):
    # Residual(PreNorm(SpatialLinearAttention)), unet_model.py:139-145,212-220,281-299
    b, c, h, w = x.shape
    xn = _chan_layernorm(x, sd[p + '.fn.norm.gamma'])
    qkv = F.conv2d(xn, sd[p + '.fn.fn.to_qkv.weight'])
    q, k, v = qkv.reshape(b, 3, heads, dim_head, h * w).unbind(1)
    q = q.softmax(dim=-2) * dim_head ** -0.5
    k = k.softmax(dim=-1)
    v = v / (h * w)
    ctx = torch.einsum('bhdn,bhen->bhde', k, v)
    out = torch.einsum('bhde,bhdn->bhen', ctx, q).reshape(b, heads * dim_head, h, w)
    out = F.conv2d(out, sd[p + '.fn.fn.to_out.weight'], sd[p + '.fn.fn.to_out.bias'])
    return out + x


def _mid_attention(sd, p, x, heads, dim_head):
    # Residual(PreNorm(EinopsToAndFrom('b c f h w','b f (h w) c', Attention))), unet_model.py:341-367,497-499
    b, c, h, w = x.shape
    xn = _chan_layernorm(x, sd[p + '.fn.norm.gamma'])
    tok = xn.reshape(b, c, h * w).transpose(1, 2)                       # b n c
    qkv = F.linear(tok, sd[p + '.fn.fn.fn.to_qkv.weight'])
    q, k, v = qkv.reshape(b, h * w, 3, heads, dim_head).permute(2, 0, 3, 1, 4)  # b h n d
    sim = torch.einsum('bhid,bhjd->bhij', q * dim_head ** -0.5, k)
    attn = (sim - sim.amax(dim=-1, keepdim=True)).softmax(dim=-1)
    o = torch.einsum('bhij,bhjd->bhid', attn, v).permute(0, 2, 1, 3).reshape(b, h * w, heads * dim_head)
    o = F.linear(o, sd[p + '.fn.fn.fn.to_out.weight'])                  # bias-free Linear (:339 wins)
    return o.transpose(1, 2).reshape(b, c, h, w) + x


def time_embedding(sd, time, dim):
    # SinusoidalPosEmb + time_mlp, unet_model.py:147-159,464-469  (nn.GELU() = exact erf form)
    half = dim // 2
    f = torch.exp(torch.arange(half, dtype=torch.float32, device=time.device) * -(math.log(10000) / (half - 1)))
    e = time.to(torch.float32)[:, None] * f[None, :]
    e = torch.cat((e.sin(), e.cos()), dim=-1).to(sd['time_mlp.1.weight'].dtype)
    e = F.linear(e, sd['time_mlp.1.weight'], sd['time_mlp.1.bias'])
    e = F.gelu(e)
    return F.linear(e, sd['time_mlp.3.weight'], sd['time_mlp.3.bias'])


def unet_forward(sd, cfg, x, time, return_taps=False, cond=None, null_mask=None):
    """Unet3D.forward with F=1, self_condition=False (unet_model.py:542-623).
    x: [B,C,P,P] (or [B,P*P,C], converted as at :554-556).  Returns [B,out_dim,P,P].
    cond [B,C,P,P] (optional, the residual gradient of the guidance branch, :585-603) with null_mask [B] bool = samples
    whose conditioning is dropped (classifier-free guidance; the reference draws it with prob_mask_like).
    cfg['padding_mode'] = 'circular' (unet_model.py:161-199, 452): the stem, every ResnetBlock 3x3 and the down-sampling
    convolutions pad circularly and the up-sampling layers are conv_transpose_circular; emb_conv[2] stays zero-padded as
    in the reference (:524)."""
    if x.ndim == 3:
        p = int(math.isqrt(x.shape[1]))
        x = x.reshape(x.shape[0], p, p, x.shape[2]).permute(0, 3, 1, 2)
    heads, dh, groups, pm = cfg['heads'], cfg['dim_head'], cfg['groups'], cfg['padding_mode']
    taps = OrderedDict()
    x = _conv(x, sd['init_conv.weight'][:, :, 0], sd['init_conv.bias'], 3, pm)
    taps['init_conv'] = x
    if cond is not None:
        c = torch.where(null_mask[:, None, None, None], torch.zeros_like(cond), cond)
        e = F.conv2d(c, sd['emb_conv.0.weight'], sd['emb_conv.0.bias'])
        e = F.conv2d(F.gelu(e), sd['emb_conv.2.weight'], sd['emb_conv.2.bias'], padding=1)     # zeros in both modes
        x = F.conv2d(torch.cat((x, e), dim=1), sd['combine_conv.weight'], sd['combine_conv.bias'])
    r = x
    t = time_embedding(sd, time, cfg['dim'])
    taps['time_emb'] = t
    n_res = len(cfg['dim_mults'])
    skips = []
    for i in range(n_res):
        x = _resblock(sd, f'downs.{i}.0', x, t, groups, pm)
        if i == 0:
            taps['downs.0.0'] = x
        x = _resblock(sd, f'downs.{i}.1', x, t, groups, pm)
        x = _linear_attention(sd, f'downs.{i}.2', x, heads, dh)
        if i == 0:
            taps['downs.0.2'] = x
        skips.append(x)
        if i < n_res - 1:
            x = _conv(x, sd[f'downs.{i}.3.weight'][:, :, 0], sd[f'downs.{i}.3.bias'], 1, pm, stride=2)
    taps['down_out'] = x
    x = _resblock(sd, 'mid_block1', x, t, groups, pm)
    x = _mid_attention(sd, 'mid_spatial_attn', x, heads, dh)
    taps['mid_attn'] = x
    x = _resblock(sd, 'mid_block2', x, t, groups, pm)
    for i in range(n_res):
        x = torch.cat((x, skips.pop()), dim=1)
        x = _resblock(sd, f'ups.{i}.0', x, t, groups, pm)
        x = _resblock(sd, f'ups.{i}.1', x, t, groups, pm)
        x = _linear_attention(sd, f'ups.{i}.2', x, heads, dh)
        if i < n_res - 1:
            w, b = sd[_up_key(cfg, i) + '.weight'][:, :, 0], sd[_up_key(cfg, i) + '.bias']
            if pm == 'circular':
                x = conv_transpose_circular(x, w, b)
            else:
                x = F.conv_transpose2d(x, w, b, stride=2, padding=1)
        if i == 0:
            taps['ups.0'] = x
    x = torch.cat((x, r), dim=1)
    x = _resblock(sd, 'final_conv.0', x, None, groups, pm)
    x = F.conv2d(x, sd['final_conv.1.weight'][:, :, 0], sd['final_conv.1.bias'])
    if cfg['sigmoid_last_channel']:
        x = torch.cat((x[:, :-1], torch.sigmoid(x[:, -1:])), dim=1)     # :619-621 (in place there)
    if return_taps:
        return x, taps
    return x


# --------------------------------------------------------------------------------------------
# A7-A9  Darcy residual   (src/residuals_darcy.py:6-70,106-207 ; src/grad_utils.py:27-184)
# --------------------------------------------------------------------------------------------


# bcs='periodic' (grad_utils.py:76-81): the reference pads by one pixel with mode='circular' and applies the interior
# ('C', 'C') stencil, so every pixel, boundary pixels included, uses the central second-order stencil with wrapped
# neighbours.  Everything else is kept as with bcs='none': h = domain_length / (P-1) when pixels_at_boundary, f_s, and
# the two BC channels on rows 0 / P-1 and columns 0 / P-1 with the same signs (built from the wrapped p_0 / p_1).


def fd_first(u, axis, h, periodic=False):
    """Second-order first derivative along `axis` (-2 = rows = x0, -1 = cols = x1): central in the
    interior, one-sided 3-point at the two ends.  Net effect of the 9 conv2d + 9 slice-assigns at
    grad_utils.py:64-146 with the acc=2 stencils (corner assignments win).  periodic: central everywhere, neighbours
    wrapped."""
    if periodic:
        return (torch.roll(u, -1, axis) - torch.roll(u, 1, axis)) * (0.5 / h)
    u = u.movedim(axis, -1)
    d = torch.empty_like(u)
    d[..., 1:-1] = (u[..., 2:] - u[..., :-2]) * (0.5 / h)
    d[..., 0] = (-1.5 * u[..., 0] + 2.0 * u[..., 1] - 0.5 * u[..., 2]) / h
    d[..., -1] = (1.5 * u[..., -1] - 2.0 * u[..., -2] + 0.5 * u[..., -3]) / h
    return d.movedim(-1, axis)


def fd_second(u, axis, h, periodic=False):
    """Second-order second derivative: central [1,-2,1]/h^2; 4-point one-sided [2,-5,4,-1]/h^2 at ends.  periodic:
    central everywhere, neighbours wrapped."""
    if periodic:
        return (torch.roll(u, -1, axis) - 2.0 * u + torch.roll(u, 1, axis)) / (h * h)
    u = u.movedim(axis, -1)
    d = torch.empty_like(u)
    h2 = h * h
    d[..., 1:-1] = (u[..., 2:] - 2.0 * u[..., 1:-1] + u[..., :-2]) / h2
    d[..., 0] = (2.0 * u[..., 0] - 5.0 * u[..., 1] + 4.0 * u[..., 2] - u[..., 3]) / h2
    d[..., -1] = (2.0 * u[..., -1] - 5.0 * u[..., -2] + 4.0 * u[..., -3] - u[..., -4]) / h2
    return d.movedim(-1, axis)


def stencil_gradients(u, mode, d0, d1, periodic=False):
    """StencilGradients(periodic=...).forward for one mode on [..., P, P]"""
    if mode == 'd_d0':
        return fd_first(u, -2, d0, periodic)
    if mode == 'd_d1':
        return fd_first(u, -1, d1, periodic)
    if mode == 'd_d00':
        return fd_second(u, -2, d0, periodic)
    if mode == 'd_d11':
        return fd_second(u, -1, d1, periodic)
    if mode == 'd_d01':
        return fd_first(fd_first(u, -1, d1, periodic), -2, d0, periodic)
    raise ValueError(mode)


def spacing(P, domain_length=1.0, reverse_d1=True, pixels_at_boundary=True):
    """(d0, d1) of ResidualsDarcy (residuals_darcy.py:24-33)"""
    d0 = domain_length / (P - 1) if pixels_at_boundary else domain_length / P
    return d0, (-d0 if reverse_d1 else d0)


def darcy_source(pixels=64, w=0.125, r=10.0, dtype=torch.float32):
    """f_s on the pixel-centre grid, residuals_darcy.py:40-53,95-104: +r on [0,w]^2, -r on [1-w,1]^2."""
    ps = 1.0 / pixels
    c = torch.linspace(ps / 2, 1.0 - ps / 2, steps=pixels)
    X, Y = torch.meshgrid(c, c, indexing='ij')
    f = torch.zeros_like(X)
    f[(torch.abs(X - 0.5 * w) <= 0.5 * w) & (torch.abs(Y - 0.5 * w) <= 0.5 * w)] = r
    f[(torch.abs(X - 1 + 0.5 * w) <= 0.5 * w) & (torch.abs(Y - 1 + 0.5 * w) <= 0.5 * w)] = -r
    return f.to(dtype)


def darcy_residual(x0_pred, domain_length=1.0, reverse_d1=True, pixels_at_boundary=True, periodic=False):
    """ResidualsDarcy.compute_residual on a given x0_pred [B,2,P,P] (residuals_darcy.py:134-183).
    Returns residual [B, P*P, 3] = (eq_0, bc_x0, bc_x1).
    eq_0 = -(K p_00 + K_0 p_0) - (K p_11 + K_1 p_1) - f_s.  periodic: bcs='periodic' (see fd_first)."""
    B, C, P, _ = x0_pred.shape
    d0, d1 = spacing(P, domain_length, reverse_d1, pixels_at_boundary)
    p, K = x0_pred[:, 0], x0_pred[:, 1]
    p0, p1 = fd_first(p, -2, d0, periodic), fd_first(p, -1, d1, periodic)
    p00, p11 = fd_second(p, -2, d0, periodic), fd_second(p, -1, d1, periodic)
    K0, K1 = fd_first(K, -2, d0, periodic), fd_first(K, -1, d1, periodic)
    fs = darcy_source(P, dtype=x0_pred.dtype).to(x0_pred.device)     # (device-aware: bench's torch-CUDA leg runs this on the GPU)
    eq0 = (-K * p00 - K0 * p0) + (-K * p11 - K1 * p1) - fs
    bc0 = torch.zeros_like(p)
    bc1 = torch.zeros_like(p)
    bc0[:, 0, :] = -p0[:, 0, :]
    bc0[:, -1, :] = p0[:, -1, :]
    sgn = 1.0 if reverse_d1 else -1.0
    bc1[:, :, 0] = sgn * p1[:, :, 0]
    bc1[:, :, -1] = -sgn * p1[:, :, -1]
    return torch.stack([eq0, bc0, bc1], dim=-1).reshape(B, P * P, 3)


def darcy_stencils(P, periodic=False, domain_length=1.0, reverse_d1=True, pixels_at_boundary=True):
    """The stencils of darcy_residual at the geometry given (spacing) as [P,P] fp64 matrices (D1_0, D2_0, D1_1, D2_1):
    fd_first(u, -2, d0) = D1_0 u and fd_first(u, -1, d1) = u D1_1^T, likewise fd_second with D2.  Their absolute values
    bound every rounding of an fp32 evaluation of the stencils."""
    mats = []
    for h in spacing(P, domain_length, reverse_d1, pixels_at_boundary):
        D1 = torch.zeros(P, P, dtype=torch.float64)
        D2 = torch.zeros(P, P, dtype=torch.float64)
        for i in range(P):
            if periodic or 0 < i < P - 1:
                D1[i, (i - 1) % P] -= 0.5
                D1[i, (i + 1) % P] += 0.5
                D2[i, (i - 1) % P] += 1.
                D2[i, i] -= 2.
                D2[i, (i + 1) % P] += 1.
            elif i == 0:
                D1[0, :3] = torch.tensor([-1.5, 2., -0.5], dtype=torch.float64)
                D2[0, :4] = torch.tensor([2., -5., 4., -1.], dtype=torch.float64)
            else:
                D1[-1, -3:] = torch.tensor([0.5, -2., 1.5], dtype=torch.float64)
                D2[-1, -4:] = torch.tensor([-1., 4., -5., 2.], dtype=torch.float64)
        mats += [D1 / h, D2 / (h * h)]
    return mats


def along_rows(M, u):
    """M applied along axis -2 of u [B,P,P]"""
    return torch.einsum('ij,bjk->bik', M, u)


def along_cols(M, u):
    """M applied along axis -1 of u [B,P,P]"""
    return torch.einsum('kj,bij->bik', M, u)


def darcy_residual_matrix(x, periodic=False, absolute=False, stencils=None, domain_length=1.0, reverse_d1=True,
                          pixels_at_boundary=True):
    """darcy_residual from the darcy_stencils matrices, x [B,2,P,P] fp64 -> [B,P*P,3]: the fp64 reference the GPU tests
    compare fp32 kernels with.  absolute=True evaluates it with |stencils|, |fields| and |f_s|, which bounds every
    intermediate of an fp32 evaluation.  `stencils` replaces darcy_stencils(P, periodic, <geometry>); reverse_d1 also
    sets the sign of the bc_x1 channel, as in darcy_residual."""
    P = x.shape[-1]
    geom = dict(domain_length=domain_length, reverse_d1=reverse_d1, pixels_at_boundary=pixels_at_boundary)
    mats = darcy_stencils(P, periodic, **geom) if stencils is None else stencils
    if absolute:      # |x| as a select, not x.abs(): the derivative of abs vanishes at an exact zero, which would drop
        mats, x = [m.abs() for m in mats], torch.where(x < 0, -x, x)     # that pixel from darcy_residual_vjp's bound
    D1a, D2a, D1b, D2b = (m.to(x.device) for m in mats)
    p, K = x[:, 0], x[:, 1]
    p0, p1, K0, K1 = along_rows(D1a, p), along_cols(D1b, p), along_rows(D1a, K), along_cols(D1b, K)
    lap = along_rows(D2a, p) + along_cols(D2b, p)
    fs = darcy_source(P, dtype=torch.float64).to(x.device)
    bc0, bc1 = torch.zeros_like(p), torch.zeros_like(p)
    if absolute:
        eq0 = K * lap + K0 * p0 + K1 * p1 + fs.abs()
        bc0[:, 0], bc0[:, -1] = p0[:, 0], p0[:, -1]
        bc1[:, :, 0], bc1[:, :, -1] = p1[:, :, 0], p1[:, :, -1]
    else:
        eq0 = -K * lap - K0 * p0 - K1 * p1 - fs
        bc0[:, 0], bc0[:, -1] = -p0[:, 0], p0[:, -1]
        sgn = 1.0 if reverse_d1 else -1.0
        bc1[:, :, 0], bc1[:, :, -1] = sgn * p1[:, :, 0], -sgn * p1[:, :, -1]
    return torch.stack([eq0, bc0, bc1], dim=-1).reshape(x.shape[0], P * P, 3)


def darcy_residual_vjp(x, cot, periodic=False, absolute=False, **geom):
    """J^T cot of darcy_residual_matrix in fp64; absolute=True: |J|^T |cot| at |x| (the residual is bilinear in (p, K)
    with non-negative coefficients in its absolute form, so this gradient bounds every product of the adjoint).
    geom: the geometry keywords of darcy_residual_matrix."""
    xa = (x.abs() if absolute else x).clone().requires_grad_(True)
    with torch.enable_grad():
        r = darcy_residual_matrix(xa, periodic, absolute, **geom)
        if absolute:
            r = r - darcy_residual_matrix(torch.zeros_like(xa), periodic, True, **geom)      # drop the constant |f_s|
        return torch.autograd.grad((r * (cot.abs() if absolute else cot)).sum(), xa)[0]


# --------------------------------------------------------------------------------------------
# A3/A10  training loss   (src/denoising_utils.py:554-558, 616-710)
# --------------------------------------------------------------------------------------------


def darcy_residual_gradient(x_t, periodic=False):
    """d mean|r(x_t)| / d x_t (residuals_darcy.py:117-120), [B,2,P,P]; a constant for the network (no graph kept)."""
    with torch.enable_grad():
        x = x_t.detach().clone().requires_grad_(True)
        return torch.autograd.grad(darcy_residual(x, periodic=periodic).abs().mean(), x)[0]


def pidm_loss_from_x0pred(x0, x0_pred, residual, t, tables, c_data=1.0, c_residual=1e-3):
    """loss = c_data * mean_b(p2[t] * mean_chw (x0 - x0_pred)^2) + mean(c_residual * 0.5 r^2 / var_t)."""
    B = x0.shape[0]
    dt = x0_pred.dtype
    mse = ((x0 - x0_pred) ** 2).reshape(B, -1).mean(dim=1)
    data = c_data * (mse * tables['p2_loss_weight'].to(dt)[t]).mean()
    var = tables['posterior_variance_clipped'].to(dt)[t].view(B, *([1] * (residual.ndim - 1)))
    res = (c_residual * 0.5 * residual ** 2 / var).mean()
    return data + res, data, residual.abs().mean()


def darcy_training_loss(sd, cfg, x0, t, noise, tables, c_data=1.0, c_residual=1e-3, use_ddim_x0=False,
                        guidance_null_mask=None, periodic=False):
    """model_estimation_loss for gov_eqs='darcy' with t and eps supplied (so it is RNG-free).
    guidance_null_mask [B] bool: residual-gradient guidance on (residuals_darcy.py:114-126) with that classifier-free mask.
    periodic: bcs='periodic' in the residual and in the guidance gradient."""
    xt = q_sample(x0, t, noise, tables)
    if guidance_null_mask is not None:
        cond = darcy_residual_gradient(xt, periodic)
        model_out = unet_forward(sd, cfg, xt, t, cond=cond, null_mask=guidance_null_mask)
        x0_hat = model_out
    elif use_ddim_x0:
        x0_hat, model_out = ddim_x0(sd, cfg, xt, t, tables)
    else:
        model_out = unet_forward(sd, cfg, xt, t)
        x0_hat = model_out
    r = darcy_residual(x0_hat, periodic=periodic)
    loss, data, rabs = pidm_loss_from_x0pred(x0, model_out, r, t, tables, c_data, c_residual)
    return loss, dict(data=data, residual_abs=rabs, model_out=model_out, x0_hat=x0_hat, residual=r, x_t=xt)


def jacobian_max(x0_pred, periodic=False):
    """max_dr_dp [B]: the largest entry (signed, zeros included, as torch.max) of d residual / d p per sample, with the
    reference's clamp(max=1e12).  The reference obtains the Jacobian with vmap(jacfwd); the residual is affine in p, so
    here its columns are residual(e_j, K) - residual(0, K) for the P*P unit fields e_j (one batched call per sample)."""
    B, _, P, _ = x0_pred.shape
    out = torch.empty(B, dtype=x0_pred.dtype)
    for b in range(B):
        basis = torch.zeros(P * P + 1, 2, P, P, dtype=x0_pred.dtype)
        basis[:, 1] = x0_pred[b, 1].detach()
        basis[torch.arange(P * P), 0, torch.arange(P * P) // P, torch.arange(P * P) % P] = 1.0
        rr = darcy_residual(basis, periodic=periodic)
        out[b] = torch.clamp((rr[:-1] - rr[-1:]).max(), max=1e12)
    return out


def cocogen_steps(x0_pred, steps, periodic=False):
    """`steps` successive ResidualsDarcy.residual_correction calls (residuals_darcy.py:209-240) on x0_pred [B,2,P,P]:
    p <- p - (1e-6 / jacobian_max) * d(sum r^2)/dp.  A correction changes p only, so K and the step size stay fixed over
    successive corrections of a field.  Returns (x, residual of x, [p after each correction])."""
    eps = (1e-6 / jacobian_max(x0_pred, periodic)).view(-1, 1, 1)
    x = x0_pred.detach().clone()
    p_iterates = []
    for _ in range(steps):
        with torch.enable_grad():
            xg = x.clone().requires_grad_(True)
            dr_dp = torch.autograd.grad((darcy_residual(xg, periodic=periodic) ** 2).sum(), xg)[0][:, 0]
        x[:, 0] = x[:, 0] - eps * dr_dp
        p_iterates.append(x[:, 0].clone())
    return x, darcy_residual(x, periodic=periodic), p_iterates


def cocogen_correction(x0_pred, periodic=False):
    """One residual_correction: (corrected x0_pred, its residual)."""
    x, r, _ = cocogen_steps(x0_pred, 1, periodic)
    return x, r


# --------------------------------------------------------------------------------------------
# A11/A12  sampling   (src/denoising_utils.py:388-545, 571-574, 712-787)
# --------------------------------------------------------------------------------------------


def posterior_step(x_t, x0_pred, z, i, tables, suppress_noise=True):
    """One ancestral step, denoising_utils.py:441-455: mean = c1[t] x0 + c2[t] x_t; + sqrt(beta_t) z (t>0)."""
    dt = x_t.dtype
    mean = tables['posterior_mean_coef1'].to(dt)[i] * x0_pred + tables['posterior_mean_coef2'].to(dt)[i] * x_t
    sig = tables['betas'].to(dt)[i].sqrt()
    mask = 0.0 if (suppress_noise and i == 0) else 1.0
    return mean + mask * sig * z


def ddim_x0(sd, cfg, xt, t, tables, ddim_steps=0, mechanics=False):
    """ddim_sample_x0 with eta=0 (denoising_utils.py:712-787), per-sample grids linspace(0,t,steps+2).
    Reference quirk kept: every network call sees the ORIGINAL x_t (model_input never updated, :741-753).
    mechanics: gov_eqs='mechanics', xt is the network input and the walk runs on its three solution channels.  The walk
    draws a noise tensor that eta = 0 never uses (the reference draws it for RNG parity), so there is none here."""
    B = xt.shape[0]
    dt = xt.dtype
    seqs, seqs_next = [], []
    for ti in t.tolist():
        # np.linspace as the reference: torch.linspace rounds some points differently (t = 58, ddim_steps = 13 gives 28
        # where numpy's int() gives 29)
        seq = [int(v) for v in np.linspace(0, ti, ddim_steps + 2, endpoint=True, dtype=float)]
        seqs.append(list(reversed(seq)))
        seqs_next.append(list(reversed([-1] + seq[:-1])))
    cur_t = torch.tensor(seqs).T
    nxt_t = torch.tensor(seqs_next).T
    cur_x = xt[:, :3] if mechanics else xt
    model_out = None
    v4 = lambda name, idx: tables[name].to(dt)[idx].view(B, 1, 1, 1)
    for k in range(cur_t.shape[0]):
        tt, tn = cur_t[k], nxt_t[k]
        x0p = unet_forward(sd, cfg, xt, tt)
        if k == 0:
            model_out = x0p
        if int(tn[0]) < 0:
            cur_x = x0p
            continue
        mean = v4('posterior_mean_coef1', tt) * x0p + v4('posterior_mean_coef2', tt) * cur_x
        eps = (v4('sqrt_recip_alphas', tt) * cur_x - mean) / v4('noise_mean_coeff', tt)
        a_next = v4('alphas_prod', tn)
        new_x = x0p * a_next.sqrt() + (1 - a_next).sqrt() * eps
        mask = (tt == tn).to(dt).view(B, 1, 1, 1)
        cur_x = mask * cur_x + (1 - mask) * new_x
    return cur_x, model_out


def p_sample_loop(sd, cfg, x_T, noises, tables, n_steps, periodic=False, N_correction=0, M_correction=0,
                  correction_mode='none', trajectory=False):
    """Ancestral loop for Darcy, mean-mode x0 (denoising_utils.py:508-545).  noises[k] is the z drawn
    at loop iteration k (drawn even at t=0).  Returns (x_0 sample, residual of the last x0_pred).
    CoCoGen corrections (the correction branches of denoising_utils.py:433-459,517-540): while t < N_correction the x0
    estimate ('x0') or the new sample ('xt') is corrected once and the step's residual is the corrected one; then
    M_correction corrections of the final sample, and the residual is that of the last correction.
    trajectory=True returns [x_T, one entry per step, one per post-loop correction] in place of the sample."""
    x = x_T
    seq = [x]
    r = None
    for k, i in enumerate(reversed(range(n_steps))):
        tt = torch.full((x.shape[0],), i, dtype=torch.long)
        x0p = unet_forward(sd, cfg, x, tt)
        r = darcy_residual(x0p, periodic=periodic)
        correct = i < N_correction
        if correct and correction_mode == 'x0':
            x0p, r = cocogen_correction(x0p, periodic)
        x = posterior_step(x, x0p, noises[k], i, tables)
        if correct and correction_mode == 'xt':
            x, r = cocogen_correction(x, periodic)
        seq.append(x)
    for _ in range(M_correction):
        x, r = cocogen_correction(x, periodic)
        seq.append(x)
    return (seq if trajectory else x), r


# --------------------------------------------------------------------------------------------
# A13  mechanics residual, matrix-free restatement (src/residuals_mechanics_K.py:10-103,166-274)
# --------------------------------------------------------------------------------------------


def q4_plane_stress_stiffness(E=1.0, nu=0.3, dtype=torch.float64):
    """Closed form of the unit-square Q4 plane-stress stiffness (the '99-line topopt' KE), node order
    counter-clockwise from the lower-left corner, dofs (u1x,u1y,...,u4y)."""
    k = [1 / 2 - nu / 6, 1 / 8 + nu / 8, -1 / 4 - nu / 12, -1 / 8 + 3 * nu / 8,
         -1 / 4 + nu / 12, -1 / 8 - nu / 8, nu / 6, 1 / 8 - 3 * nu / 8]
    idx = [[0, 1, 2, 3, 4, 5, 6, 7], [1, 0, 7, 6, 5, 4, 3, 2], [2, 7, 0, 5, 6, 3, 4, 1],
           [3, 6, 5, 0, 7, 2, 1, 4], [4, 5, 6, 7, 0, 1, 2, 3], [5, 4, 3, 2, 1, 0, 7, 6],
           [6, 3, 4, 1, 2, 7, 0, 5], [7, 2, 1, 4, 3, 6, 5, 0]]
    KE = torch.tensor([[k[j] for j in row] for row in idx], dtype=dtype) * (E / (1 - nu ** 2))
    return KE


def mechanics_mesh(nel=64):
    """The generated unit-square mesh convention used by BOTH oracle and engine (the authors' mesh
    files are an external download, SURVEY.md section 8c): node id = row*(nel+1)+col, dof = 2*node+d.
    Element (er,ec) connects, counter-clockwise in (x=col, y=-row... ) a stated convention:
    n1=(er+1,ec), n2=(er+1,ec+1), n3=(er,ec+1), n4=(er,ec).  Returns LongTensor [nel*nel, 8] of dofs."""
    nn_ = nel + 1
    er, ec = torch.meshgrid(torch.arange(nel), torch.arange(nel), indexing='ij')
    nodes = torch.stack([(er + 1) * nn_ + ec, (er + 1) * nn_ + ec + 1, er * nn_ + ec + 1, er * nn_ + ec], dim=-1)
    nodes = nodes.reshape(-1, 4)
    return torch.stack([2 * nodes, 2 * nodes + 1], dim=-1).reshape(-1, 8)


def bilinear_resize(x, size):
    """torchvision Resize(antialias=False) == F.interpolate(bilinear, align_corners=False),
    residuals_mechanics_K.py:10-21."""
    return F.interpolate(x, size=(size, size), mode='bilinear', align_corners=False, antialias=False)


def mechanics_residual(x0_pred, bcs, vf, KE=None):
    """Matrix-free restatement of ResidualsMechanics.compute_residual on a given x0_pred
    [B,3,64,64] = (u_x,u_y,rho) and bcs [B,4,65,65] = (bc_x, bc_y, load_x, load_y):
       r = K(rho) u - f with BC rows replaced by identity rows (columns NOT symmetrised) and f zeroed
       there; compliance = u^T K u (same modified K); inequality = mean(rho) - vf."""
    B = x0_pred.shape[0]
    dt = x0_pred.dtype
    nel = x0_pred.shape[-1]
    KE = (q4_plane_stress_stiffness() if KE is None else KE).to(dt)
    dofs = mechanics_mesh(nel)
    u_img = bilinear_resize(x0_pred[:, :2], nel + 1)                       # [B,2,65,65]
    u = u_img.permute(0, 2, 3, 1).reshape(B, -1)                           # dof = 2*(row*65+col)+d
    rho = x0_pred[:, 2].reshape(B, -1)
    ue = u[:, dofs]                                                        # [B,nel^2,8]
    fe = torch.einsum('ij,bej->bei', KE, ue) * rho[:, :, None]
    Ku = torch.zeros_like(u).index_add_(1, dofs.reshape(-1), fe.reshape(B, -1))
    bc_mask = (bcs[:, :2].permute(0, 2, 3, 1).reshape(B, -1) != 0)
    f = bcs[:, 2:4].permute(0, 2, 3, 1).reshape(B, -1)
    f = torch.where(bc_mask, torch.zeros_like(f), f)
    Ku = torch.where(bc_mask, u, Ku)                                       # identity rows
    residual = Ku - f
    compliance = (u * Ku).sum(dim=1)
    ineq = rho.mean(dim=1) - vf
    return residual, compliance, ineq


def mechanics_matfree(u, rho, bcs, KE=None, absolute=False):
    """pidm_mechanics_residual_fwd on its own operands, any nel: u [B,2,nn,nn] nodal displacements, rho [B,nel,nel],
    bcs [B,4,nn,nn] = (bc_x, bc_y, load_x, load_y), nn = nel + 1.  Returns (residual [B, 2 nn^2] in the dof order
    2*node + d, compliance [B]):
       residual = K(rho) u - f with the Dirichlet rows (bcs[:, :2] != 0) replaced by identity rows and f zeroed there,
       compliance = u^T (that modified K) u.
    K(rho) u is formed from four shifted views of the node planes, one per local node of the Q4 element, so it shares no
    indexing with mechanics_mesh.  Differentiable: its VJP comes from autograd.  absolute=True evaluates it with |KE|,
    |u|, |rho| and |f|, which bounds every intermediate of an fp32 evaluation."""
    KE = (q4_plane_stress_stiffness() if KE is None else torch.as_tensor(KE)).to(u)
    fixed = bcs[:, :2] != 0
    if absolute:      # selects, not abs(): as in darcy_residual_matrix, a VJP through them keeps exact zeros
        KE, u, rho, bcs = (torch.where(v < 0, -v, v) for v in (KE, u, rho, bcs))
    nel = rho.shape[-1]
    corners = ((1, 0), (1, 1), (0, 1), (0, 0))              # local nodes n1..n4 of element (er, ec): (er + dr, ec + dc)
    ue = torch.stack([u[:, d, dr:dr + nel, dc:dc + nel] for dr, dc in corners for d in (0, 1)], dim=1)
    fe = torch.einsum('ij,bjrc->birc', KE, ue) * rho[:, None]
    Ku = sum(F.pad(fe[:, 2 * k:2 * k + 2], (dc, 1 - dc, dr, 1 - dr)) for k, (dr, dc) in enumerate(corners))
    f = torch.where(fixed, torch.zeros_like(u), bcs[:, 2:4])
    w = torch.where(fixed, u, Ku)
    r = w + f if absolute else w - f
    return r.permute(0, 2, 3, 1).reshape(u.shape[0], -1), (u * w).sum(dim=(1, 2, 3))


def mechanics_training_loss(sd, cfg, inp, t, noise, tables, c_data=1.0, c_residual=1e-2, c_ineq=0.0, lambda_opt=0.0):
    """model_estimation_loss for gov_eqs='mechanics', mean-mode x0, with t and eps supplied (denoising_utils.py:616-710,
    residuals_mechanics_K.py:166-274).  inp [B,10,65,65] = (vf, strain energy, von Mises | disp_x, disp_y, E | bc_x,
    bc_y, load_x, load_y).  Returns (loss, dict of the tracked scalars and intermediates)."""
    B = inp.shape[0]
    cond, x0, bcs = torch.tensor_split(inp, (3, 6), dim=1)
    xt = q_sample(x0, t, noise, tables)
    net_in = torch.cat((bilinear_resize(torch.cat((xt, cond), dim=1), 64), bilinear_resize(bcs, 64)), dim=1)
    y = unet_forward(sd, cfg, net_in, t)
    vf = cond[:, 0, 0, 0]
    r, comp, ineq = mechanics_residual(y, bcs, vf)
    out = torch.cat((bilinear_resize(y[:, :2], 65), F.pad(y[:, 2], (0, 1, 0, 1)).unsqueeze(1)), dim=1)
    mse = ((x0 - out) ** 2).reshape(B, -1).mean(dim=1)
    data = c_data * (mse * tables['p2_loss_weight'].to(mse.dtype)[t]).mean()
    var = tables['posterior_variance_clipped'].to(mse.dtype)[t]
    loss = data + (c_residual * 0.5 * r ** 2 / var[:, None]).mean()
    if c_ineq > 0:
        # reference :679,:694: var is extracted with the residual's rank ([B,1]) while the inequality is [B]: the
        # quotient broadcasts to [B,B]
        loss = loss + (c_ineq * 0.5 * ineq[None, :] ** 2 / var[:, None]).mean()
    loss = loss + (lambda_opt * comp).mean()
    return loss, dict(data=data, residual_abs=r.abs().mean(), inequality=ineq.mean(), compliance=comp.mean(), model_out=out,
                      residual=r)


def mechanics_p_sample_loop(sd, cfg, x_T, noises, conditioning, bcs, tables, n_steps, use_ddim_x0=False, ddim_steps=0):
    """The reference's ancestral loop with a conditioning input (denoising_utils.py:388-545 with
    residuals_mechanics_K.py:176-205).  x_T [B,3,65,65], noises[k] = the posterior z of loop iteration k (drawn at t = 0
    too), conditioning [B,3,65,65], bcs [B,4,65,65].  Returns dict(x_first, x_final, x0_pred_last, residual, compliance,
    inequality); the residual terms are those of the last step (t = 0)."""
    x, out = x_T, {}
    vf = conditioning[:, 0, 0, 0]
    bcs_red = bilinear_resize(bcs, 64)
    for k, i in enumerate(reversed(range(n_steps))):
        tt = torch.full((x.shape[0],), i, dtype=torch.long)
        net_in = torch.cat((bilinear_resize(torch.cat((x, conditioning), dim=1), 64), bcs_red), dim=1)
        if use_ddim_x0:
            x0p, mo = ddim_x0(sd, cfg, net_in, tt, tables, ddim_steps, mechanics=True)
        else:
            x0p = mo = unet_forward(sd, cfg, net_in, tt)
        model_out = torch.cat((bilinear_resize(mo[:, :2], 65), F.pad(mo[:, 2], (0, 1, 0, 1)).unsqueeze(1)), dim=1)
        x = posterior_step(x, model_out, noises[k], i, tables)
        if k == 0:
            out['x_first'] = x
    r, comp, ineq = mechanics_residual(x0p, bcs, vf)
    out.update(x_final=x, x0_pred_last=x0p, residual=r, compliance=comp, inequality=ineq)
    return out


def reduced_system(rho, bcs, KE=None):
    """rho [nel,nel], bcs [4,nel+1,nel+1] -> (K scipy CSC fp64, f fp64) in the dof order 2*node + d: K(rho) with the
    reference's modification (Dirichlet rows replaced by identity rows, columns kept, f zeroed on the Dirichlet dofs;
    residuals_mechanics_K.py:296-325)."""
    import numpy as np
    import scipy.sparse as sp
    rho = np.asarray(rho, dtype=np.float64)
    bcs = np.asarray(bcs, dtype=np.float64)
    nel = rho.shape[-1]
    n = 2 * (nel + 1) ** 2
    KE = (q4_plane_stress_stiffness() if KE is None else torch.as_tensor(KE)).double().numpy()
    dofs = mechanics_mesh(nel).numpy()                                            # [nel^2, 8]
    vals = rho.reshape(-1)[:, None, None] * KE[None]
    rows = np.broadcast_to(dofs[:, :, None], vals.shape)
    cols = np.broadcast_to(dofs[:, None, :], vals.shape)
    K = sp.coo_matrix((vals.ravel(), (rows.ravel(), cols.ravel())), shape=(n, n)).tocsr()
    fixed = np.stack((bcs[0].ravel(), bcs[1].ravel()), axis=1).ravel() != 0
    f = np.stack((bcs[2].ravel(), bcs[3].ravel()), axis=1).ravel()
    f[fixed] = 0.
    K = sp.diags((~fixed).astype(np.float64)) @ K + sp.diags(fixed.astype(np.float64))
    return K.tocsc(), f


def fem_solve(rho, bcs, KE=None):
    """u [B,2,nel+1,nel+1] fp64 with K(rho) u = f on the free dofs, u = 0 on the Dirichlet dofs: scipy's sparse direct
    solve of reduced_system, the ground truth for the iterative solvers."""
    import scipy.sparse.linalg as spla
    rho, bcs = torch.as_tensor(rho), torch.as_tensor(bcs)
    out = []
    for b in range(rho.shape[0]):
        K, f = reduced_system(rho[b].cpu().numpy(), bcs[b].cpu().numpy(), KE)
        nn_ = bcs.shape[-1]
        out.append(torch.from_numpy(spla.spsolve(K, f).reshape(nn_ * nn_, 2).T.reshape(2, nn_, nn_).copy()))
    return torch.stack(out)


# --------------------------------------------------------------------------------------------
# A15  toy study on [B, D] points   (main_toy.py:48-79, src/denoising_toy_utils.py:171-199, 267-333, 372-383, 436-511)
# --------------------------------------------------------------------------------------------


def toy_model_forward(sd, x, t):
    """ConditionalModel: softplus(embed1[t] * lin1(x)) -> softplus(embed2[t] * lin2(.)) -> lin3 (:171-199)"""
    h = F.softplus(sd['lin1.embed.weight'][t] * F.linear(x, sd['lin1.lin.weight'], sd['lin1.lin.bias']))
    h = F.softplus(sd['lin2.embed.weight'][t] * F.linear(h, sd['lin2.lin.weight'], sd['lin2.lin.bias']))
    return F.linear(h, sd['lin3.weight'], sd['lin3.bias'])


def toy_ddim_x0(sd, xt, t, tables, mode):
    """ddim_sample_x0 with reduced_n_steps = 0, eta = 0 (:267-333): grid (t, 0) then (0, -1); cur_x advances."""
    tz = torch.zeros_like(t)
    out = toy_model_forward(sd, xt, t)
    ra, rm = tables['sqrt_recip_alphas_cumprod'][t, None], tables['sqrt_recipm1_alphas_cumprod'][t, None]
    if mode == 'eps':
        eps, x0p = out, ra * xt - rm * out
    else:
        x0p = out
        mean = tables['posterior_mean_coef1'][t, None] * x0p + tables['posterior_mean_coef2'][t, None] * xt
        eps = (tables['sqrt_recip_alphas'][t, None] * xt - mean) / tables['noise_mean_coeff'][t, None]
    a_next = tables['alphas_prod'][tz, None]
    cur = x0p * a_next.sqrt() + (1 - a_next).sqrt() * eps
    mask = (t == tz).float()[:, None]
    cur = mask * xt + (1 - mask) * cur
    out = toy_model_forward(sd, cur, tz)
    if mode == 'eps':
        return tables['sqrt_recip_alphas_cumprod'][tz, None] * cur - tables['sqrt_recipm1_alphas_cumprod'][tz, None] * out
    return out


def toy_training_loss(sd, x0, t, noise, tables, mode='x0', use_ddim_x0=False, c_data=1.0, c_residual=0.005, c_ineq=0.0,
                      lambda_opt=0.0):
    """model_estimation_loss of the toy study (:436-511) with the callables of main_toy.py:48-79: residual
    |x|^2 - 1, inequality relu(|x|_1 - 1), optimisation x[:, 0].  Returns (loss, ["data loss" as the reference reports it, mean|r|, mean ineq, mean opt])."""
    tables = {k: v.to(x0.dtype) for k, v in tables.items()}
    x = tables['alphas_bar_sqrt'][t, None] * x0 + tables['one_minus_alphas_bar_sqrt'][t, None] * noise
    out = toy_model_forward(sd, x, t)
    if mode == 'eps':
        data = ((noise - out) ** 2).mean()
        x0p = tables['sqrt_recip_alphas_cumprod'][t, None] * x - tables['sqrt_recipm1_alphas_cumprod'][t, None] * out
    else:
        data = (((x0 - out) ** 2).mean(dim=1) * tables['p2_loss_weight'][t]).mean()
        x0p = out
    data = c_data * data
    ev = toy_ddim_x0(sd, x, t, tables, mode) if use_ddim_x0 else x0p
    var = tables['posterior_variance_clipped'][t]

    def nll(v):
        return -torch.clamp(-0.5 * v ** 2 / var, min=-27.6310211159)
    r = (ev ** 2).sum(dim=1) - 1.0
    q = torch.relu(ev.abs().sum(dim=1) - 1.0)
    o = ev[:, 0]
    loss = data + c_residual * nll(r).mean() + c_ineq * nll(q).mean() + lambda_opt * o.mean()
    # reference quirk (:477-478,:491): `data_loss = loss` aliases the tensor that `loss += ...` then updates in place, so
    # the "data loss" it reports is the TOTAL loss
    return loss, [loss.detach(), r.abs().mean(), q.mean(), o.mean()]


# --------------------------------------------------------------------------------------------
# A14  step glue: clip + Adam + EMA     (main.py:163-166,178-183,316 ; denoising_utils.py:163-205)
# --------------------------------------------------------------------------------------------


def adam_ema_step(params, grads, m, v, ema, step, lr=1e-4, b1=0.9, b2=0.999, eps=1e-8, max_norm=1.0,
                  ema_mu=0.99, ema_on=True):
    """Reference semantics of clip_grad_norm_(1.0) -> Adam(lr,default betas/eps) -> EMA(0.99) on lists
    of tensors; in place.  `step` is the 1-based Adam step count."""
    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads)).float()
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    for p, g, mi, vi, e in zip(params, grads, m, v, ema):
        g = g * coef
        mi.mul_(b1).add_(g, alpha=1 - b1)
        vi.mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = (vi.sqrt() / math.sqrt(bc2)).add_(eps)
        p.addcdiv_(mi, denom, value=-lr / bc1)
        if ema_on:
            e.mul_(ema_mu).add_(p, alpha=1 - ema_mu)
    return total
