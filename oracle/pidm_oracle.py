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
"""
import math
from collections import OrderedDict

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
                groups=8, sigmoid_last_channel=False):
    return dict(dim=dim, channels=channels, out_dim=channels if out_dim is None else out_dim,
                dim_mults=tuple(dim_mults), heads=heads, dim_head=dim_head, groups=groups,
                sigmoid_last_channel=sigmoid_last_channel)


def unet_param_shapes(cfg):
    """Every state_dict key of the reference Unet3D with its shape, in reference order
    (unet_model.py:406-528).  Includes the parameter holders that forward never touches."""
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
            S[f'ups.{i}.3.weight'] = (ci, ci, 1, 4, 4)
            S[f'ups.{i}.3.bias'] = (ci,)
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


def _resblock(sd, p, x, temb, groups):
    # ResnetBlock.forward, unet_model.py:255-267
    ss = None
    if temb is not None and (p + '.mlp.1.weight') in sd:
        e = F.linear(F.silu(temb), sd[p + '.mlp.1.weight'], sd[p + '.mlp.1.bias'])
        ss = e[:, :, None, None].chunk(2, dim=1)
    h = F.conv2d(x, sd[p + '.block1.proj.weight'][:, :, 0], sd[p + '.block1.proj.bias'], padding=1)
    h = _gn_silu(h, sd[p + '.block1.norm.weight'], sd[p + '.block1.norm.bias'], groups, ss)
    h = F.conv2d(h, sd[p + '.block2.proj.weight'][:, :, 0], sd[p + '.block2.proj.bias'], padding=1)
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
    whose conditioning is dropped (classifier-free guidance; the reference draws it with prob_mask_like)."""
    if x.ndim == 3:
        p = int(math.isqrt(x.shape[1]))
        x = x.reshape(x.shape[0], p, p, x.shape[2]).permute(0, 3, 1, 2)
    heads, dh, groups = cfg['heads'], cfg['dim_head'], cfg['groups']
    taps = OrderedDict()
    x = F.conv2d(x, sd['init_conv.weight'][:, :, 0], sd['init_conv.bias'], padding=3)
    taps['init_conv'] = x
    if cond is not None:
        c = torch.where(null_mask[:, None, None, None], torch.zeros_like(cond), cond)
        e = F.conv2d(c, sd['emb_conv.0.weight'], sd['emb_conv.0.bias'])
        e = F.conv2d(F.gelu(e), sd['emb_conv.2.weight'], sd['emb_conv.2.bias'], padding=1)
        x = F.conv2d(torch.cat((x, e), dim=1), sd['combine_conv.weight'], sd['combine_conv.bias'])
    r = x
    t = time_embedding(sd, time, cfg['dim'])
    taps['time_emb'] = t
    n_res = len(cfg['dim_mults'])
    skips = []
    for i in range(n_res):
        x = _resblock(sd, f'downs.{i}.0', x, t, groups)
        if i == 0:
            taps['downs.0.0'] = x
        x = _resblock(sd, f'downs.{i}.1', x, t, groups)
        x = _linear_attention(sd, f'downs.{i}.2', x, heads, dh)
        if i == 0:
            taps['downs.0.2'] = x
        skips.append(x)
        if i < n_res - 1:
            x = F.conv2d(x, sd[f'downs.{i}.3.weight'][:, :, 0], sd[f'downs.{i}.3.bias'], stride=2, padding=1)
    taps['down_out'] = x
    x = _resblock(sd, 'mid_block1', x, t, groups)
    x = _mid_attention(sd, 'mid_spatial_attn', x, heads, dh)
    taps['mid_attn'] = x
    x = _resblock(sd, 'mid_block2', x, t, groups)
    for i in range(n_res):
        x = torch.cat((x, skips.pop()), dim=1)
        x = _resblock(sd, f'ups.{i}.0', x, t, groups)
        x = _resblock(sd, f'ups.{i}.1', x, t, groups)
        x = _linear_attention(sd, f'ups.{i}.2', x, heads, dh)
        if i < n_res - 1:
            x = F.conv_transpose2d(x, sd[f'ups.{i}.3.weight'][:, :, 0], sd[f'ups.{i}.3.bias'], stride=2, padding=1)
        if i == 0:
            taps['ups.0'] = x
    x = torch.cat((x, r), dim=1)
    x = _resblock(sd, 'final_conv.0', x, None, groups)
    x = F.conv2d(x, sd['final_conv.1.weight'][:, :, 0], sd['final_conv.1.bias'])
    if cfg['sigmoid_last_channel']:
        x = torch.cat((x[:, :-1], torch.sigmoid(x[:, -1:])), dim=1)     # :619-621 (in place there)
    if return_taps:
        return x, taps
    return x


# --------------------------------------------------------------------------------------------
# A7-A9  Darcy residual   (src/residuals_darcy.py:6-70,106-207 ; src/grad_utils.py:27-184)
# --------------------------------------------------------------------------------------------


def fd_first(u, axis, h):
    """Second-order first derivative along `axis` (-2 = rows = x0, -1 = cols = x1): central in the
    interior, one-sided 3-point at the two ends.  Net effect of the 9 conv2d + 9 slice-assigns at
    grad_utils.py:64-146 with the acc=2 stencils (corner assignments win)."""
    u = u.movedim(axis, -1)
    d = torch.empty_like(u)
    d[..., 1:-1] = (u[..., 2:] - u[..., :-2]) * (0.5 / h)
    d[..., 0] = (-1.5 * u[..., 0] + 2.0 * u[..., 1] - 0.5 * u[..., 2]) / h
    d[..., -1] = (1.5 * u[..., -1] - 2.0 * u[..., -2] + 0.5 * u[..., -3]) / h
    return d.movedim(-1, axis)


def fd_second(u, axis, h):
    """Second-order second derivative: central [1,-2,1]/h^2; 4-point one-sided [2,-5,4,-1]/h^2 at ends."""
    u = u.movedim(axis, -1)
    d = torch.empty_like(u)
    h2 = h * h
    d[..., 1:-1] = (u[..., 2:] - 2.0 * u[..., 1:-1] + u[..., :-2]) / h2
    d[..., 0] = (2.0 * u[..., 0] - 5.0 * u[..., 1] + 4.0 * u[..., 2] - u[..., 3]) / h2
    d[..., -1] = (2.0 * u[..., -1] - 5.0 * u[..., -2] + 4.0 * u[..., -3] - u[..., -4]) / h2
    return d.movedim(-1, axis)


def darcy_source(pixels=64, w=0.125, r=10.0, dtype=torch.float32):
    """f_s on the pixel-centre grid, residuals_darcy.py:40-53,95-104: +r on [0,w]^2, -r on [1-w,1]^2."""
    ps = 1.0 / pixels
    c = torch.linspace(ps / 2, 1.0 - ps / 2, steps=pixels)
    X, Y = torch.meshgrid(c, c, indexing='ij')
    f = torch.zeros_like(X)
    f[(torch.abs(X - 0.5 * w) <= 0.5 * w) & (torch.abs(Y - 0.5 * w) <= 0.5 * w)] = r
    f[(torch.abs(X - 1 + 0.5 * w) <= 0.5 * w) & (torch.abs(Y - 1 + 0.5 * w) <= 0.5 * w)] = -r
    return f.to(dtype)


def darcy_residual(x0_pred, domain_length=1.0, reverse_d1=True, pixels_at_boundary=True):
    """ResidualsDarcy.compute_residual on a given x0_pred [B,2,P,P] (residuals_darcy.py:134-183).
    Returns residual [B, P*P, 3] = (eq_0, bc_x0, bc_x1).
    eq_0 = -(K p_00 + K_0 p_0) - (K p_11 + K_1 p_1) - f_s."""
    B, C, P, _ = x0_pred.shape
    d0 = domain_length / (P - 1) if pixels_at_boundary else domain_length / P
    d1 = -d0 if reverse_d1 else d0
    p, K = x0_pred[:, 0], x0_pred[:, 1]
    p0, p1 = fd_first(p, -2, d0), fd_first(p, -1, d1)
    p00, p11 = fd_second(p, -2, d0), fd_second(p, -1, d1)
    K0, K1 = fd_first(K, -2, d0), fd_first(K, -1, d1)
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


# --------------------------------------------------------------------------------------------
# A3/A10  training loss   (src/denoising_utils.py:554-558, 616-710)
# --------------------------------------------------------------------------------------------


def darcy_residual_gradient(x_t):
    """d mean|r(x_t)| / d x_t (residuals_darcy.py:117-120), [B,2,P,P]; a constant for the network (no graph kept)."""
    with torch.enable_grad():
        x = x_t.detach().clone().requires_grad_(True)
        return torch.autograd.grad(darcy_residual(x).abs().mean(), x)[0]


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
                        guidance_null_mask=None):
    """model_estimation_loss for gov_eqs='darcy' with t and eps supplied (so it is RNG-free).
    guidance_null_mask [B] bool: residual-gradient guidance on (residuals_darcy.py:114-126) with that classifier-free mask."""
    xt = q_sample(x0, t, noise, tables)
    if guidance_null_mask is not None:
        model_out = unet_forward(sd, cfg, xt, t, cond=darcy_residual_gradient(xt), null_mask=guidance_null_mask)
        x0_hat = model_out
    elif use_ddim_x0:
        x0_hat, model_out = ddim_x0(sd, cfg, xt, t, tables)
    else:
        model_out = unet_forward(sd, cfg, xt, t)
        x0_hat = model_out
    r = darcy_residual(x0_hat)
    loss, data, rabs = pidm_loss_from_x0pred(x0, model_out, r, t, tables, c_data, c_residual)
    return loss, dict(data=data, residual_abs=rabs, model_out=model_out, x0_hat=x0_hat, residual=r, x_t=xt)


def cocogen_correction(x0_pred):
    """ResidualsDarcy.residual_correction (residuals_darcy.py:209-240) on x0_pred [B,2,P,P]:
    p <- p - (1e-6 / max(dr/dp)) * d(sum r^2)/dp, then the residual of the corrected field.  The reference obtains the
    Jacobian dr/dp with vmap(jacfwd); the residual is affine in p, so here its columns are residual(e_j, K) - residual(0, K)
    for the 4096 unit fields e_j (one batched call per sample)."""
    B, _, P, _ = x0_pred.shape
    x = x0_pred.detach().clone().requires_grad_(True)
    r = darcy_residual(x)
    dr_dp = torch.autograd.grad((r ** 2).sum(), x)[0][:, 0]
    out = x0_pred.detach().clone()
    for b in range(B):
        K = x0_pred[b, 1].detach()
        basis = torch.zeros(P * P + 1, 2, P, P, dtype=x0_pred.dtype)
        basis[:, 1] = K
        basis[torch.arange(P * P), 0, torch.arange(P * P) // P, torch.arange(P * P) % P] = 1.0
        rr = darcy_residual(basis)
        J = rr[:-1] - rr[-1:]                                    # [column j][row (pixel, channel)]
        mx = torch.clamp(J.max(), max=1e12)
        out[b, 0] = out[b, 0] - (1e-6 / mx) * dr_dp[b]
    return out, darcy_residual(out)


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


def ddim_x0(sd, cfg, xt, t, tables, ddim_steps=0):
    """ddim_sample_x0 with eta=0 (denoising_utils.py:712-787), per-sample grids linspace(0,t,steps+2).
    Reference quirk kept: every network call sees the ORIGINAL x_t (model_input never updated, :741-753)."""
    B = xt.shape[0]
    dt = xt.dtype
    seqs, seqs_next = [], []
    for ti in t.tolist():
        seq = [int(v) for v in torch.linspace(0, ti, ddim_steps + 2, dtype=torch.float64).tolist()]
        seqs.append(list(reversed(seq)))
        seqs_next.append(list(reversed([-1] + seq[:-1])))
    cur_t = torch.tensor(seqs).T
    nxt_t = torch.tensor(seqs_next).T
    cur_x = xt
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


def p_sample_loop(sd, cfg, x_T, noises, tables, n_steps):
    """Ancestral loop for Darcy, mean-mode x0 (denoising_utils.py:508-545).  noises[k] is the z drawn
    at loop iteration k (drawn even at t=0).  Returns (x_0 sample, residual of the last x0_pred)."""
    x = x_T
    r = None
    for k, i in enumerate(reversed(range(n_steps))):
        tt = torch.full((x.shape[0],), i, dtype=torch.long)
        x0p = unet_forward(sd, cfg, x, tt)
        r = darcy_residual(x0p)
        x = posterior_step(x, x0p, noises[k], i, tables)
    return x, r


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
