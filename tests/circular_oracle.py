"""CPU oracle for Unet3D(padding_mode='circular') (reference src/unet_model.py:161-199).  TEST INFRASTRUCTURE ONLY.

The circular restatement of oracle.pidm_oracle.unet_forward in plain PyTorch (float32 or float64, CPU): the stem, every
ResnetBlock 3x3 and the three down-sampling convolutions pad circularly; the up-sampling layers are the periodic 4x4 /
stride-2 transposed convolution (circular pad 1, then conv_transpose2d with padding 3 -- equal to the reference's pad 2 /
padding 5); emb_conv[2] stays zero-padded as in the reference (:524).  It takes the CIRCULAR state_dict (the up-sampling
weights under `ups.{i}.3.conv_transpose.*`).  Pinned against the reference by tests/test_oracle_circular.py.
"""
import torch
import torch.nn.functional as F

from oracle import pidm_oracle as O


def conv_circ(x, w, b, pad, stride=1):
    return F.conv2d(F.pad(x, (pad,) * 4, mode='circular'), w, b, stride=stride)


def up_circ(x, w, b):
    return F.conv_transpose2d(F.pad(x, (1,) * 4, mode='circular'), w, b, stride=2, padding=3)


def circular_state_dict(sd):
    """zeros-mode state_dict (oracle.make_test_state_dict) -> the circular model's keys"""
    out = {}
    for k, v in sd.items():
        parts = k.split('.')
        if parts[0] == 'ups' and parts[2] == '3':
            k = '.'.join(parts[:3] + ['conv_transpose'] + parts[3:])
        out[k] = v
    return out


def _resblock(sd, p, x, temb, groups):
    ss = None
    if temb is not None and (p + '.mlp.1.weight') in sd:
        e = F.linear(F.silu(temb), sd[p + '.mlp.1.weight'], sd[p + '.mlp.1.bias'])
        ss = e[:, :, None, None].chunk(2, dim=1)
    h = conv_circ(x, sd[p + '.block1.proj.weight'][:, :, 0], sd[p + '.block1.proj.bias'], 1)
    h = O._gn_silu(h, sd[p + '.block1.norm.weight'], sd[p + '.block1.norm.bias'], groups, ss)
    h = conv_circ(h, sd[p + '.block2.proj.weight'][:, :, 0], sd[p + '.block2.proj.bias'], 1)
    h = O._gn_silu(h, sd[p + '.block2.norm.weight'], sd[p + '.block2.norm.bias'], groups)
    if (p + '.res_conv.weight') in sd:
        x = F.conv2d(x, sd[p + '.res_conv.weight'][:, :, 0], sd[p + '.res_conv.bias'])
    return h + x


def unet_forward(sd, cfg, x, time, return_taps=False, cond=None, null_mask=None):
    """O.unet_forward with padding_mode='circular'; same arguments and taps"""
    if x.ndim == 3:
        p = int(x.shape[1] ** 0.5)
        x = x.reshape(x.shape[0], p, p, x.shape[2]).permute(0, 3, 1, 2)
    heads, dh, groups = cfg['heads'], cfg['dim_head'], cfg['groups']
    taps = {}
    x = conv_circ(x, sd['init_conv.weight'][:, :, 0], sd['init_conv.bias'], 3)
    taps['init_conv'] = x
    if cond is not None:
        c = torch.where(null_mask[:, None, None, None], torch.zeros_like(cond), cond)
        e = F.conv2d(c, sd['emb_conv.0.weight'], sd['emb_conv.0.bias'])
        e = F.conv2d(F.gelu(e), sd['emb_conv.2.weight'], sd['emb_conv.2.bias'], padding=1)     # zero-padded
        x = F.conv2d(torch.cat((x, e), dim=1), sd['combine_conv.weight'], sd['combine_conv.bias'])
    r = x
    t = O.time_embedding(sd, time, cfg['dim'])
    n_res = len(cfg['dim_mults'])
    skips = []
    for i in range(n_res):
        x = _resblock(sd, f'downs.{i}.0', x, t, groups)
        if i == 0:
            taps['downs.0.0'] = x
        x = _resblock(sd, f'downs.{i}.1', x, t, groups)
        x = O._linear_attention(sd, f'downs.{i}.2', x, heads, dh)
        if i == 0:
            taps['downs.0.2'] = x
        skips.append(x)
        if i < n_res - 1:
            x = conv_circ(x, sd[f'downs.{i}.3.weight'][:, :, 0], sd[f'downs.{i}.3.bias'], 1, stride=2)
    x = _resblock(sd, 'mid_block1', x, t, groups)
    x = O._mid_attention(sd, 'mid_spatial_attn', x, heads, dh)
    taps['mid_attn'] = x
    x = _resblock(sd, 'mid_block2', x, t, groups)
    for i in range(n_res):
        x = torch.cat((x, skips.pop()), dim=1)
        x = _resblock(sd, f'ups.{i}.0', x, t, groups)
        x = _resblock(sd, f'ups.{i}.1', x, t, groups)
        x = O._linear_attention(sd, f'ups.{i}.2', x, heads, dh)
        if i < n_res - 1:
            x = up_circ(x, sd[f'ups.{i}.3.conv_transpose.weight'][:, :, 0], sd[f'ups.{i}.3.conv_transpose.bias'])
        if i == 0:
            taps['ups.0'] = x
    x = torch.cat((x, r), dim=1)
    x = _resblock(sd, 'final_conv.0', x, None, groups)
    x = F.conv2d(x, sd['final_conv.1.weight'][:, :, 0], sd['final_conv.1.bias'])
    if cfg['sigmoid_last_channel']:
        x = torch.cat((x[:, :-1], torch.sigmoid(x[:, -1:])), dim=1)
    if return_taps:
        return x, taps
    return x
