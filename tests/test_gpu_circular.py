"""Unet3D(padding_mode='circular') on the GPU: the wrap-pad (halo) kernel, every circular convolution geometry of the
Darcy network (forward, dgrad, weight gradient) per element against fp64, the plans the halo'd operands get, and the
network's forward, roll equivariance and guidance loss against fixtures of the UNMODIFIED reference
(oracle/make_golden.py circular).  The circular training loss, graph-replayed step and sampling engine are the
'circular' rows of test_gpu_e2e.py and test_gpu_parity_bench_path.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from checks import rel
from oracle import pidm_oracle as O
from study import build_darcy

pytestmark = pytest.mark.gpu
DEV = 'cuda'
U = 2.0 ** -24


# ---- halo kernel --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
@pytest.mark.parametrize('B,H,C', [(1, 64, 32), (3, 32, 64), (32, 64, 32), (3, 16, 256), (32, 8, 512), (3, 8, 2048)])
@pytest.mark.parametrize('halo', [1, 2, 3])
def test_wrap_pad_is_bitwise_circular_pad(dtype, B, H, C, halo):
    from physicsinformeddiffusionmodels_b200 import _lib
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + C + halo)
    x = torch.randn(B, H, H, C, device=DEV, generator=g).to(dtype)
    n = B * (H + 2 * halo) ** 2 * C
    guard = 4096
    buf = torch.full((n + 2 * guard,), float('nan'), device=DEV, dtype=dtype)
    y = buf[guard:guard + n].view(B, H + 2 * halo, H + 2 * halo, C)
    _lib.call('pidm_wrap_pad_nhwc', x, y, B, H, H, C, halo, _lib.DTYPE_CODE[dtype], _lib.stream())
    ref = F.pad(x.permute(0, 3, 1, 2), (halo,) * 4, mode='circular').permute(0, 2, 3, 1)
    assert torch.equal(y, ref)
    assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + n:]).all()


# ---- every circular convolution geometry of the Darcy (dim=32) and mechanics (dim=128) networks ------------------------
def _geometries(model, P=64):
    """distinct (kind, k, stride, Cin, Cin_real, Cout, H) of a circular model's padded layers, H = input size"""
    out, res = set(), P
    for s in model._packer.specs:                # registration order = execution order
        if s.circular:
            out.add((s.kind, s.kh, s.stride, s.cin, s.cin_real, s.cout, res))
        if s.kind == 'conv' and s.stride == 2:
            res //= 2
        elif s.kind == 'convT':
            res *= 2
    return sorted(out)


def _models():
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    return {'darcy': Unet3D(dim=32, channels=2, padding_mode='circular'),
            'mechanics': Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True, padding_mode='circular')}


_GEOMS = {k: _geometries(m) for k, m in _models().items()}
# batch 32 for the Darcy layers (the benchmarked step); batch 8 for the mechanics layers keeps the fp64 references of
# the 128..2048-channel layers affordable (the plans at batch 32 are checked below)
LAYERS = [pytest.param(g, 32, id='darcy-' + '-'.join(map(str, g))) for g in _GEOMS['darcy']] + [
    pytest.param(g, 8, id='mechanics-' + '-'.join(map(str, g))) for g in _GEOMS['mechanics']]


def _ref_conv(kind, x, w, stride, pad, edit=None):
    """fp64 reference; edit = 'row' / 'col' leaves the first halo row / last halo column unwrapped (zero)"""
    xp = F.pad(x, ((pad if kind == 'conv' else 1),) * 4, mode='circular')
    if edit == 'row':
        xp = torch.cat((torch.zeros_like(xp[:, :, :1]), xp[:, :, 1:]), 2)
    elif edit == 'col':
        xp = torch.cat((xp[..., :-1], torch.zeros_like(xp[..., -1:])), 3)
    if kind == 'conv':
        return F.conv2d(xp, w, stride=stride)
    return F.conv_transpose2d(xp, w, stride=2, padding=3)


def _layer(geom, B):
    from physicsinformeddiffusionmodels_b200 import ops, packing
    kind, k, stride, Cin, Cin_real, Cout, H = geom
    pad = k // 2 if stride == 1 else 1
    g = torch.Generator().manual_seed(k * 100000 + Cin * 100 + Cout + H)
    x = torch.zeros(B, Cin, H, H, dtype=torch.float64)
    x[:, :Cin_real] = torch.randn(B, Cin_real, H, H, generator=g).bfloat16().double()
    shape = (Cout, Cin_real, 1, k, k) if kind == 'conv' else (Cin, Cout, 1, k, k)
    w = (torch.randn(*shape, generator=g) / math.sqrt(Cin_real * k * k)).bfloat16().double()
    Ho = H // stride if kind == 'conv' else 2 * H
    cot = torch.randn(B, Cout, Ho, Ho, generator=g).bfloat16().double()
    wd = torch.nn.Parameter(w.float().to(DEV))
    need_dgrad = Cin == Cin_real                 # the channel-padded stem has no input gradient (its input is data)
    spec = packing.ConvSpec(wd, kind, k, k, stride, pad, cin_pad=Cin, need_dgrad=need_dgrad, circular=True)
    pk = packing.WeightPacker()
    pk.add(spec)
    pk.refresh(torch.bfloat16)
    xd = x.permute(0, 2, 3, 1).contiguous().to(DEV).bfloat16().requires_grad_(need_dgrad)
    ops.set_precision('bf16')
    y = ops.conv2d(xd, wd, None, spec)
    y.backward(cot.permute(0, 2, 3, 1).contiguous().to(DEV).bfloat16())
    torch.cuda.synchronize()
    out = dict(kind=kind, stride=stride, x=x[:, :Cin_real].to(DEV), w=w[:, :, 0].to(DEV), cot=cot.to(DEV), pad=pad,
               y=y.permute(0, 3, 1, 2).double(), dw=wd.grad[:, :, 0].double())
    if need_dgrad:
        out['dx'] = xd.grad.permute(0, 3, 1, 2).double()
    return out


def _refs(L, edit=None):
    """fp64 references and per-element bounds: |y - r| <= 2^-8 |r| + sqrt(K) 2^-24 A for the bf16 outputs (y, dx),
    sqrt(K') 2^-24 A for the fp32 weight gradient (A = the same sums over absolute values)"""
    kind, stride, x, w, cot, pad = L['kind'], L['stride'], L['x'], L['w'], L['cot'], L['pad']
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    yr = _ref_conv(kind, xr, wr, stride, pad, edit)
    yr.backward(cot)
    xa, wa = x.abs().requires_grad_(True), w.abs().requires_grad_(True)
    ya = _ref_conv(kind, xa, wa, stride, pad)
    ya.backward(cot.abs())
    cin, cout = (w.shape[1], w.shape[0]) if kind == 'conv' else (w.shape[0], w.shape[1])
    taps = w.shape[-1] * w.shape[-2]
    k_w = x.shape[0] * cot.shape[-1] * cot.shape[-2]
    return {'y': (yr.detach(), 2.0 ** -8 * yr.detach().abs() + math.sqrt(cin * taps) * U * ya.detach()),
            'dx': (xr.grad, 2.0 ** -8 * xr.grad.abs() + math.sqrt(cout * taps) * U * xa.grad),
            'dw': (wr.grad, math.sqrt(k_w) * U * wa.grad)}


def _passes(got, ref, bound):
    return bool(((got - ref).abs() <= bound).all())


@pytest.mark.parametrize('geom,B', LAYERS)
def test_circular_layer_per_element_against_fp64(geom, B):
    L = _layer(geom, B)
    for name, (ref, bound) in _refs(L).items():
        if name in L:
            err = (L[name] - ref).abs()
            assert (err <= bound).all(), (name, (err / bound).max().item())


def _pick(kind, k):
    return next(g for g in _GEOMS['darcy'] if g[0] == kind and g[1] == k)


@pytest.mark.parametrize('geom', [_pick('conv', 7), _pick('conv', 3), _pick('conv', 4), _pick('convT', 4)],
                         ids=['stem', '3x3', 'down', 'up'])
@pytest.mark.parametrize('edit', ['row', 'col'])
def test_circular_layer_bound_rejects_an_unwrapped_halo_line(geom, edit):
    """one halo row or column left unwrapped in the reference: the forward, input gradient and weight gradient of the
    kernels all fail the bound"""
    L = _layer(geom, 32)
    refs = _refs(L, edit)
    for name in ('y', 'dx', 'dw'):
        if name in L:
            assert not _passes(L[name], *refs[name]), name


@pytest.mark.parametrize('geom,name', [(_pick('convT', 4), 'y'), (_pick('conv', 4), 'dx')], ids=['up-fwd', 'down-dgrad'])
@pytest.mark.parametrize('cls', [(0, 0), (1, 1)])
def test_circular_gather_bound_rejects_a_shifted_parity_class(geom, name, cls):
    """the four-class transposed gather (up-sampling forward, down-sampling dgrad): a reference in which ONE output
    parity class is shifted by one pixel fails the bound"""
    L = _layer(geom, 32)
    ref, bound = _refs(L)[name]
    assert _passes(L[name], ref, bound)
    a, b = cls
    edited = ref.clone()
    edited[:, :, a::2, b::2] = torch.roll(ref[:, :, a::2, b::2], 1, 2)
    assert not _passes(L[name], edited, bound)


@pytest.mark.parametrize('model', ['darcy', 'mechanics'])
def test_circular_plans_match_the_zero_padded_layers(model):
    """at batch 32 the halo'd operands get the same tensor-core plans as the zero-padded layers: row-group staging for
    the stride-1 layers with 16-row tiles, the four-class gather for the up-sampling forward, and the tap-complete 3x3
    weight-gradient kernel"""
    from physicsinformeddiffusionmodels_b200._lib import call
    import ctypes
    B = 32
    for kind, k, s, ci, _, co, H in _GEOMS[model]:
        pad = k // 2 if s == 1 else 1
        out_z, out_c = (ctypes.c_int * 12)(), (ctypes.c_int * 12)()
        if kind == 'conv':
            Ho = H // s
            call('pidm_conv2d_tc_plan', B, H, H, ci, Ho, Ho, co, k, k, s, pad, 0, out_z)
            call('pidm_conv2d_tc_plan', B, H + 2 * pad, H + 2 * pad, ci, Ho, Ho, co, k, k, s, 0, 0, out_c)
        else:
            call('pidm_conv2d_tc_plan', B, H, H, ci, 2 * H, 2 * H, co, k, k, 2, 1, 1, out_z)
            call('pidm_conv2d_tc_plan', B, H + 2, H + 2, ci, 2 * H, 2 * H, co, k, k, 2, 3, 1, out_c)
        assert list(out_z)[:10] == list(out_c)[:10], (kind, k, ci, co, H)
        if kind == 'conv' and s == 1:
            assert out_c[2] == (1 if H % 16 == 0 else 0)
        if kind == 'conv' and k == 3:
            wz, wc = (ctypes.c_int * 12)(), (ctypes.c_int * 12)()
            call('pidm_conv2d_wgrad_tc_plan', B, H, H, ci, ci, H, H, co, 3, 3, 1, 1, 9, ci * 9, wz)
            call('pidm_conv2d_wgrad_tc_plan', B, H + 2, H + 2, ci, ci, H, H, co, 3, 3, 1, 0, 9, ci * 9, wc)
            assert wc[0] == 1 and list(wz) == list(wc), (ci, co, H)


# ---- end to end -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from physicsinformeddiffusionmodels_b200 import ops
    yield ops
    ops.set_precision('bf16')


@pytest.mark.parametrize('mode,tol', [('fp32', 1e-4), ('bf16', 3e-2)])
def test_circular_unet_forward_matches_reference(ops, golden, mode, tol):
    ops.set_precision(mode)
    gd = golden('unet_circular_fwd.pt')
    model, _, _ = build_darcy('circular')
    with torch.no_grad():
        y = model(gd['x'].to(DEV), gd['t'].to(DEV))
    assert rel(y, gd['y']) < tol, rel(y, gd['y'])


@pytest.mark.parametrize('mode,tol', [('fp32', 1e-4), ('bf16', 3e-2)])
def test_circular_unet_rolls_with_its_input(ops, mode, tol):
    """rolling the input by (8, 16) pixels rolls the output; the zero-padded network fails the same check"""
    ops.set_precision(mode)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 2, 64, 64, generator=g).to(DEV)
    t = torch.tensor([3, 77], device=DEV)
    errs = {}
    for study in ('circular', 'periodic'):                  # 'periodic': periodic residual, zero-padded network
        model, _, _ = build_darcy(study)
        with torch.no_grad():
            y = model(x, t)
            ys = model(torch.roll(x, (8, 16), (2, 3)), t)
        errs[study] = rel(ys, torch.roll(y, (8, 16), (2, 3)))
    assert errs['circular'] < tol, errs
    assert errs['periodic'] > 0.1, errs


@pytest.mark.parametrize('mode,tol_loss,tol_grad', [('fp32', 5e-5, 1e-3), ('bf16', 3e-2, 8e-2)])
def test_circular_guidance_loss_matches_reference(ops, golden, mode, tol_loss, tol_grad):
    """residual-gradient guidance: emb_conv[2] stays zero-padded inside the circular network"""
    ops.set_precision(mode)
    gd = golden('darcy_guidance_circular.pt')
    model, diff, res = build_darcy('circular', residual_grad_guidance=True)
    model._null_mask_override = gd['null_mask'].to(DEV)
    loss, _, _, _, _ = diff.darcy_loss_from_draws(gd['x0'].to(DEV), gd['t'].to(DEV), gd['noise'].to(DEV), res, 1.0, 1e-3)
    model._null_mask_override = None
    assert abs(loss.item() / gd['loss'].item() - 1) < tol_loss, (loss.item(), gd['loss'].item())
    loss.backward()
    named = dict(model.named_parameters())
    for k, gk in (('emb_conv.2.weight', 'grad_emb2'), ('emb_conv.0.weight', 'grad_emb0'),
                  ('final_conv.1.weight', 'grad_final_w')):
        assert rel(named[k].grad, gd[gk]) < tol_grad, (k, rel(named[k].grad, gd[gk]))


@pytest.mark.parametrize('mode,tol', [('fp32', 1e-4), ('bf16', 3e-2)])
def test_circular_mechanics_model_forward_matches_oracle(ops, mode, tol):
    """Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True, padding_mode='circular') at batch 2 against
    the circular oracle (fp64 on the device)"""
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    ops.set_precision(mode)
    cfg = O.unet_config(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True, padding_mode='circular')
    sd = O.make_test_state_dict(cfg, 5)
    model = Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True, padding_mode='circular').to(DEV)
    model.load_state_dict(sd)
    model.eval()
    g = torch.Generator().manual_seed(21)
    x = torch.randn(2, 10, 64, 64, generator=g).to(DEV)
    t = torch.tensor([5, 60], device=DEV)
    with torch.no_grad():
        y = model(x, t)
        ref = O.unet_forward({k: v.to(DEV).double() for k, v in sd.items()}, cfg, x.double(), t)
    assert y.shape == (2, 3, 64, 64)
    assert rel(y, ref) < tol, rel(y, ref)
