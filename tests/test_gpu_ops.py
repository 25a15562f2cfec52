"""Per-operator parity of the libpidm CUDA kernels (through the C ABI) against plain PyTorch fp32 references
/ the CPU oracle.  fp32-activation mode must agree tightly (only summation order differs); bf16 mode within
bf16 rounding of the operands.  Tolerances are written next to each check."""
import math

import pytest
import torch
import torch.nn.functional as F

from checks import rel

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def nhwc(x, dtype):      # test-side layout helper: NCHW fp32 -> NHWC activations
    return x.permute(0, 2, 3, 1).contiguous().to(dtype)


def nchw(x):
    return x.float().permute(0, 3, 1, 2).contiguous()


@pytest.fixture(scope='module')
def pk():
    from physicsinformeddiffusionmodels_b200 import ops, packing
    return ops, packing


DTYPES = [(torch.float32, 2e-5), (torch.bfloat16, 2e-2)]


# ----------------------------------------------------------------------------------------------
# convolution: every geometry the U-Net uses, forward + dgrad + wgrad, CUDA-core kernel
# ----------------------------------------------------------------------------------------------
CONV_CASES = [
    # name, kind, Cin, Cout, k, stride, pad, H
    ('3x3', 'conv', 32, 64, 3, 1, 1, 16),
    ('1x1', 'conv', 64, 32, 1, 1, 0, 16),
    ('7x7stem', 'conv', 2, 32, 7, 1, 3, 16),
    ('down4x4s2', 'conv', 32, 32, 4, 2, 1, 16),
    ('up4x4s2T', 'convT', 32, 32, 4, 2, 1, 8),
    ('3x3wide', 'conv', 64, 96, 3, 1, 1, 8),
]


@pytest.mark.parametrize('dtype,tol', DTYPES)
@pytest.mark.parametrize('case', CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_simt(pk, case, dtype, tol):
    ops, packing = pk
    ops.set_tensor_core_conv(False)
    name, kind, Cin, Cout, k, stride, pad, H = case
    B = 3
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, Cin, H, H, generator=g)
    if kind == 'conv':
        w = torch.randn(Cout, Cin, 1, k, k, generator=g) / math.sqrt(Cin * k * k)
    else:
        w = torch.randn(Cin, Cout, 1, k, k, generator=g) / math.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g) * 0.1
    if dtype == torch.bfloat16:   # compare on identical (bf16-representable) operands
        x, w = x.bfloat16().float(), w.bfloat16().float()
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    if kind == 'conv':
        yr = F.conv2d(xr, wr[:, :, 0], br, stride=stride, padding=pad)
    else:
        yr = F.conv_transpose2d(xr, wr[:, :, 0], br, stride=stride, padding=pad)
    cot = torch.randn(yr.shape, generator=g)
    if dtype == torch.bfloat16:
        cot = cot.bfloat16().float()
    (yr * cot).sum().backward()

    cpad = (Cin + 7) // 8 * 8
    wd = torch.nn.Parameter(w.to(DEV))
    bd = torch.nn.Parameter(b.to(DEV))
    spec = packing.ConvSpec(wd, kind, k, k, stride, pad, cin_pad=cpad, need_dgrad=(cpad == Cin))
    packer = packing.WeightPacker()
    packer.add(spec)
    packer.refresh(dtype)
    xin = torch.zeros(B, H, H, cpad)
    xin[..., :Cin] = x.permute(0, 2, 3, 1)
    xd = xin.to(DEV).to(dtype).requires_grad_(cpad == Cin)
    y = ops.conv2d(xd, wd, bd, spec)
    assert rel(nchw(y), yr) < tol, f'{name} fwd'
    (y.float() * nhwc(cot, torch.float32).to(DEV)).sum().backward()
    assert rel(wd.grad, wr.grad) < tol, f'{name} wgrad'
    assert rel(bd.grad, br.grad) < tol, f'{name} bgrad'
    if cpad == Cin:
        assert rel(nchw(xd.grad), xr.grad) < tol, f'{name} dgrad'
    ops.set_tensor_core_conv(True)


TC_CASES = [
    # B, H, Cin, Cout, k, bias, residual
    (2, 64, 32, 32, 3, True, False),
    (2, 32, 64, 64, 3, True, True),
    (4, 16, 128, 128, 3, True, False),
    (4, 8, 256, 256, 3, True, False),
    (3, 8, 256, 256, 3, False, False),      # odd batch: TN=2 box runs out of bounds in the batch dimension
    (2, 64, 32, 768, 1, False, False),      # to_qkv
    (2, 64, 256, 32, 1, True, True),        # to_out + residual
    (2, 16, 256, 64, 3, True, False),       # ups.1.0.block1
    (2, 8, 512, 128, 3, True, False),
    (2, 32, 768, 64, 1, False, False),      # dgrad of to_qkv
]


@pytest.mark.parametrize('case', TC_CASES, ids=[f'B{c[0]}_H{c[1]}_C{c[2]}x{c[3]}_k{c[4]}' for c in TC_CASES])
def test_conv_tcgen05_matches_reference(pk, case):
    """wgmma/TMA kernel vs fp32 F.conv2d on bf16-representable operands: only accumulation order and the bf16
    rounding of the OUTPUT differ -> 1e-2 relative (bf16 has 8 mantissa bits: 2^-9 per element)."""
    ops, packing = pk
    from physicsinformeddiffusionmodels_b200._lib import call
    B, H, Cin, Cout, k, has_bias, has_res = case
    assert call('pidm_conv2d_tc_general_supported', B, H, H, Cin, H, H, Cout, k, k, 1, k // 2, 0) == 1
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(B, Cin, H, H, generator=g)).bfloat16().float()
    w = (torch.randn(Cout, Cin, 1, k, k, generator=g) / math.sqrt(Cin * k * k)).bfloat16().float()
    b = torch.randn(Cout, generator=g) if has_bias else None
    res = torch.randn(B, Cout, H, H, generator=g).bfloat16().float() if has_res else None
    yr = F.conv2d(x, w[:, :, 0], b, padding=k // 2)
    if has_res:
        yr = yr + res
    wd = torch.nn.Parameter(w.to(DEV))
    spec = packing.ConvSpec(wd, 'conv', k, k, 1, k // 2)
    packer = packing.WeightPacker()
    packer.add(spec)
    packer.refresh(torch.bfloat16)
    xd = nhwc(x, torch.bfloat16).to(DEV)
    ops.set_tensor_core_conv(True)
    with torch.no_grad():
        y = ops.conv2d(xd, wd, None if b is None else b.to(DEV), spec,
                       residual=None if res is None else nhwc(res, torch.bfloat16).to(DEV))
        ops.set_tensor_core_conv(False)
        y_simt = ops.conv2d(xd, wd, None if b is None else b.to(DEV), spec,
                            residual=None if res is None else nhwc(res, torch.bfloat16).to(DEV))
        ops.set_tensor_core_conv(True)
    torch.cuda.synchronize()
    e_tc, e_simt = rel(nchw(y), yr), rel(nchw(y_simt), yr)
    assert e_simt < 1e-2, f'simt reference itself off: {e_simt}'
    assert e_tc < 1e-2, f'tensor-core conv off: rel {e_tc} (simt {e_simt})'


def test_conv_tcgen05_dgrad(pk):
    ops, packing = pk
    g = torch.Generator().manual_seed(3)
    B, H, Cin, Cout = 2, 32, 64, 128
    x = torch.randn(B, Cin, H, H, generator=g).bfloat16().float().requires_grad_(True)
    w = (torch.randn(Cout, Cin, 1, 3, 3, generator=g) / 24).bfloat16().float()
    yr = F.conv2d(x, w[:, :, 0], None, padding=1)
    cot = torch.randn(yr.shape, generator=g).bfloat16().float()
    (yr * cot).sum().backward()
    wd = torch.nn.Parameter(w.to(DEV))
    spec = packing.ConvSpec(wd, 'conv', 3, 3, 1, 1)
    packer = packing.WeightPacker()
    packer.add(spec)
    packer.refresh(torch.bfloat16)
    xd = nhwc(x.detach(), torch.bfloat16).to(DEV).requires_grad_(True)
    ops.set_tensor_core_conv(True)
    y = ops.conv2d(xd, wd, None, spec)
    y.backward(nhwc(cot, torch.bfloat16).to(DEV))
    assert rel(nchw(xd.grad), x.grad) < 1e-2
    wr = w.clone().requires_grad_(True)
    (F.conv2d(x.detach(), wr[:, :, 0], None, padding=1) * cot).sum().backward()
    assert rel(wd.grad, wr.grad) < 1e-2


# ----------------------------------------------------------------------------------------------
# normalisation
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype,tol', DTYPES)
@pytest.mark.parametrize('C,H,with_ss', [(32, 16, True), (64, 8, False), (256, 8, True)])
def test_groupnorm_silu(pk, C, H, with_ss, dtype, tol):
    ops, _ = pk
    g = torch.Generator().manual_seed(4)
    B, G = 3, 8
    x = (torch.randn(B, C, H, H, generator=g) * 1.5 + 0.3)
    if dtype == torch.bfloat16:
        x = x.bfloat16().float()
    gamma = (1 + 0.2 * torch.randn(C, generator=g))
    beta = 0.1 * torch.randn(C, generator=g)
    ss = 0.3 * torch.randn(B, 2 * C, generator=g) if with_ss else None
    xr, gr, br = x.clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    sr = ss.clone().requires_grad_(True) if with_ss else None
    h = F.group_norm(xr, G, gr, br, eps=1e-5)
    if with_ss:
        sc, sh = sr[:, :C, None, None], sr[:, C:, None, None]
        h = h * (sc + 1) + sh
    yr = F.silu(h)
    cot = torch.randn(yr.shape, generator=g)
    if dtype == torch.bfloat16:
        cot = cot.bfloat16().float()
    (yr * cot).sum().backward()
    xd = nhwc(x, dtype).to(DEV).requires_grad_(True)
    gd, bd = torch.nn.Parameter(gamma.to(DEV)), torch.nn.Parameter(beta.to(DEV))
    sd = ss.to(DEV).requires_grad_(True) if with_ss else None
    y = ops.groupnorm_silu(xd, gd, bd, sd, G)
    assert rel(nchw(y), yr) < tol
    y.backward(nhwc(cot, dtype).to(DEV))
    assert rel(nchw(xd.grad), xr.grad) < 2 * tol
    assert rel(gd.grad, gr.grad) < 2 * tol and rel(bd.grad, br.grad) < 2 * tol
    if with_ss:
        assert rel(sd.grad, sr.grad) < 2 * tol


@pytest.mark.parametrize('C,H,dtype,tol', [(32, 64, torch.bfloat16, 2e-2), (64, 32, torch.bfloat16, 2e-2),
                                           (128, 16, torch.bfloat16, 2e-2), (256, 8, torch.bfloat16, 2e-2),
                                           (32, 32, torch.bfloat16, 2e-2), (64, 16, torch.bfloat16, 2e-2),
                                           (128, 8, torch.bfloat16, 2e-2), (32, 64, torch.float32, 2e-5),
                                           (256, 8, torch.float32, 2e-5), (128, 64, torch.bfloat16, 2e-2),
                                           (1024, 8, torch.bfloat16, 2e-2)])
def test_groupnorm_silu_at_benchmarked_shapes(pk, C, H, dtype, tol):
    """Every GroupNorm geometry of the B=32 training step (and two of the dim=128 mechanics model): the backward
    planner picks (channel slab, cluster size 1..8, vectors per thread) from the shape, so each level of the U-Net runs
    a different instantiation.  Also checks the producer-bias gradient that rides on the backward (column sums of dx)."""
    ops, _ = pk
    g = torch.Generator().manual_seed(40 + C + H)
    B, G = (32 if C * H * H <= 32 * 64 * 64 * 2 else 4), 8
    x = torch.randn(B, C, H, H, generator=g) * 1.5 + 0.3
    cot = torch.randn(B, C, H, H, generator=g)
    if dtype == torch.bfloat16:
        x, cot = x.bfloat16().float(), cot.bfloat16().float()
    gamma, beta = 1 + 0.2 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    ss = 0.3 * torch.randn(B, 2 * C, generator=g)
    xr, gr, br, sr = (t.clone().requires_grad_(True) for t in (x, gamma, beta, ss))
    h = F.group_norm(xr, G, gr, br, eps=1e-5) * (sr[:, :C, None, None] + 1) + sr[:, C:, None, None]
    yr = F.silu(h)
    (yr * cot).sum().backward()
    xd = nhwc(x, dtype).to(DEV).requires_grad_(True)
    gd, bd = torch.nn.Parameter(gamma.to(DEV)), torch.nn.Parameter(beta.to(DEV))
    sd = ss.to(DEV).requires_grad_(True)
    link = {'groups': G, 'sums': None, 'bias': torch.nn.Parameter(torch.zeros(C, device=DEV))}
    y = ops.groupnorm_silu(xd, gd, bd, sd, G, gn_link=link)
    assert rel(nchw(y), yr) < tol
    y.backward(nhwc(cot, dtype).to(DEV))
    assert rel(nchw(xd.grad), xr.grad) < 2 * tol
    assert rel(gd.grad, gr.grad) < 2 * tol and rel(bd.grad, br.grad) < 2 * tol
    assert rel(sd.grad, sr.grad) < 2 * tol
    # column sums of a mean-free-per-group quantity: compare on the scale of |dx| summed, not of the (tiny) result
    dbias_ref = xr.grad.sum(dim=(0, 2, 3))
    scale = xr.grad.abs().sum(dim=(0, 2, 3)).max()
    assert ((link['dbias'].cpu() - dbias_ref).abs().max() / scale).item() < (2e-3 if dtype == torch.bfloat16 else 1e-5)


@pytest.mark.parametrize('dtype,tol', DTYPES)
@pytest.mark.parametrize('C', [32, 64, 256, 512])
def test_layernorm_c(pk, C, dtype, tol):
    ops, _ = pk
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, C, 8, 8, generator=g) * 2 + 0.5
    if dtype == torch.bfloat16:
        x = x.bfloat16().float()
    gamma = 1 + 0.2 * torch.randn(1, C, 1, 1, 1, generator=g)
    xr, gr = x.clone().requires_grad_(True), gamma.clone().requires_grad_(True)
    var = xr.var(dim=1, unbiased=False, keepdim=True)
    yr = (xr - xr.mean(dim=1, keepdim=True)) / (var + 1e-5).sqrt() * gr.reshape(1, C, 1, 1)
    cot = torch.randn(yr.shape, generator=g)
    (yr * cot).sum().backward()
    xd = nhwc(x, dtype).to(DEV).requires_grad_(True)
    gd = torch.nn.Parameter(gamma.to(DEV))
    y = ops.layernorm_c(xd, gd)
    assert rel(nchw(y), yr) < tol
    y.backward(nhwc(cot, dtype).to(DEV))
    assert rel(nchw(xd.grad), xr.grad) < 2 * tol
    assert rel(gd.grad, gr.grad) < 2 * tol


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
def _linattn_ref(qkv, heads):      # qkv [B, 3*hid, H, W]
    b, c3, h, w = qkv.shape
    q, k, v = qkv.reshape(b, 3, heads, 32, h * w).unbind(1)
    q = q.softmax(dim=-2) * 32 ** -0.5
    k = k.softmax(dim=-1)
    v = v / (h * w)
    ctx = torch.einsum('bhdn,bhen->bhde', k, v)
    return torch.einsum('bhde,bhdn->bhen', ctx, q).reshape(b, heads * 32, h, w)


@pytest.mark.parametrize('dtype,tol', DTYPES)
@pytest.mark.parametrize('H', [8, 16, 32, 64])      # 8, 16: one-CTA-per-head kernel (bf16); 32, 64: streaming kernels
def test_linear_attention(pk, H, dtype, tol):
    ops, _ = pk
    g = torch.Generator().manual_seed(6)
    B, heads = 2, 8
    qkv = torch.randn(B, 3 * heads * 32, H, H, generator=g) * 1.5
    if dtype == torch.bfloat16:
        qkv = qkv.bfloat16().float()
    qr = qkv.clone().requires_grad_(True)
    yr = _linattn_ref(qr, heads)
    cot = torch.randn(yr.shape, generator=g)
    (yr * cot).sum().backward()
    qd = nhwc(qkv, dtype).to(DEV).requires_grad_(True)
    y = ops.linear_attention(qd, heads)
    assert rel(nchw(y), yr) < tol
    y.backward(nhwc(cot, dtype).to(DEV))
    assert rel(nchw(qd.grad), qr.grad) < 2 * tol


@pytest.mark.parametrize('B,H', [(2, 64), (3, 16), (1, 32), (4, 64), (3, 32)])
def test_block_op_matches_unfused_composition(pk, B, H):
    """The linear-attention block op (to_qkv 1x1, linear attention, to_out 1x1 with bias and the residual add in one op;
    neither qkv nor the attention output is written) vs an fp32 torch reference on bf16-representable operands, and vs
    the unfused libpidm composition conv2d(to_qkv) -> linear_attention -> conv2d(to_out, bias, residual=x).  The
    residual and the bias are scaled to the rms of the attention term, so that all three terms of y count.  bf16
    activations: 3e-2 on y and 6e-2 on the gradients against fp32, like the other bf16 attention tests; the two libpidm
    compositions differ by the bf16 rounding of q, k, v, the attention output and its gradient, which only the unfused
    one materialises: 1e-2 / 2e-2.  The block's launches are checked per element against fp64 in
    test_gpu_launch_census.py, the standalone linear attention's in test_gpu_attention_census.py."""
    ops, packing = pk
    ops.set_precision('bf16')
    ops.set_tensor_core_conv(True)
    g = torch.Generator().manual_seed(66)
    heads, C = 8, 32
    bf = lambda t: t.bfloat16().float()
    xn = bf(torch.randn(B, C, H, H, generator=g))
    wq = bf(torch.randn(3 * heads * 32, C, 1, 1, 1, generator=g) * (1.5 / math.sqrt(C)))
    wo = bf(torch.randn(C, heads * 32, 1, 1, 1, generator=g) / math.sqrt(heads * 32))
    s = F.conv2d(_linattn_ref(F.conv2d(xn, wq[:, :, 0]), heads), wo[:, :, 0]).pow(2).mean().sqrt().item()
    x = bf(torch.randn(B, C, H, H, generator=g) * s)
    bo = torch.randn(C, generator=g) * s
    dy = bf(torch.randn(B, C, H, H, generator=g))
    ref = [t.clone().requires_grad_(True) for t in (xn, x, wq, wo, bo)]
    xnr, xr, wqr, wor, bor = ref
    yr = xr + F.conv2d(_linattn_ref(F.conv2d(xnr, wqr[:, :, 0]), heads), wor[:, :, 0], bor)
    (yr * dy).sum().backward()
    ref = [yr.detach()] + [t.grad for t in ref]

    def run(block):
        wqd, wod, bod = (torch.nn.Parameter(t.to(DEV)) for t in (wq, wo, bo))
        sq, so = packing.ConvSpec(wqd, 'conv', 1, 1, 1, 0), packing.ConvSpec(wod, 'conv', 1, 1, 1, 0)
        pkr = packing.WeightPacker(); pkr.add(sq); pkr.add(so); pkr.refresh(torch.bfloat16)
        xnd = nhwc(xn, torch.bfloat16).to(DEV).requires_grad_(True)
        xd = nhwc(x, torch.bfloat16).to(DEV).requires_grad_(True)
        if block:
            assert ops.linear_attention_block_supported(xnd, sq, so, bod, heads)
            y = ops.linear_attention_block(xnd, wqd, sq, wod, bod, so, xd, heads)
        else:
            y = ops.conv2d(ops.linear_attention(ops.conv2d(xnd, wqd, None, sq), heads), wod, bod, so, residual=xd)
        y.backward(nhwc(dy, torch.bfloat16).to(DEV))
        torch.cuda.synchronize()
        return [nchw(y), nchw(xnd.grad), nchw(xd.grad), wqd.grad.float().cpu(), wod.grad.float().cpu(),
                bod.grad.float().cpu()]
    got, unf = run(True), run(False)
    names = ('y', 'dxn', 'dx', 'dWqkv', 'dWout', 'db')
    for name, a, u, r in zip(names, got, unf, ref):
        tol_ref, tol_unf = (3e-2, 1e-2) if name == 'y' else (6e-2, 2e-2)
        print(f'[block] B={B} H={H} {name}: rel vs fp32 {rel(a, r):.3g}, vs unfused {rel(a, u):.3g}')
        assert rel(a, r) < tol_ref and rel(a, u) < tol_unf, (name, rel(a, r), rel(a, u))
    assert torch.equal(got[2].cpu(), dy), 'the residual gradient is dy'


@pytest.mark.parametrize('dtype,tol', DTYPES)
def test_mid_attention(pk, dtype, tol):
    ops, _ = pk
    g = torch.Generator().manual_seed(7)
    B, heads, H = 3, 8, 8
    qkv = torch.randn(B, H * H, 3 * heads * 32, generator=g)
    if dtype == torch.bfloat16:
        qkv = qkv.bfloat16().float()
    qr = qkv.clone().requires_grad_(True)
    q, k, v = qr.reshape(B, H * H, 3, heads, 32).permute(2, 0, 3, 1, 4)
    attn = torch.einsum('bhid,bhjd->bhij', q * 32 ** -0.5, k).softmax(dim=-1)
    yr = torch.einsum('bhij,bhjd->bhid', attn, v).permute(0, 2, 1, 3).reshape(B, H * H, heads * 32)
    cot = torch.randn(yr.shape, generator=g)
    (yr * cot).sum().backward()
    qd = qkv.reshape(B, H, H, -1).to(DEV).to(dtype).requires_grad_(True)
    y = ops.softmax_attention(qd, heads)
    assert rel(y.reshape(B, H * H, -1), yr) < tol
    y.backward(cot.reshape(B, H, H, -1).to(DEV).to(dtype))
    assert rel(qd.grad.reshape(B, H * H, -1), qr.grad) < 2 * tol


# ----------------------------------------------------------------------------------------------
# output head (the time embedding and block MLPs are replayed per element in test_gpu_glue_census.py)
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype,tol', DTYPES)
@pytest.mark.parametrize('O_,sig', [(2, False), (3, True)])
def test_head(pk, O_, sig, dtype, tol):
    ops, _ = pk
    g = torch.Generator().manual_seed(9)
    B, C, H = 2, 32, 16
    x = torch.randn(B, C, H, H, generator=g)
    if dtype == torch.bfloat16:
        x = x.bfloat16().float()
    w = torch.randn(O_, C, 1, 1, 1, generator=g) / 5
    b = torch.randn(O_, generator=g) * .1
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yr = F.conv2d(xr, wr[:, :, 0], br)
    if sig:
        yr = torch.cat((yr[:, :-1], torch.sigmoid(yr[:, -1:])), 1)
    cot = torch.randn(yr.shape, generator=g)
    (yr * cot).sum().backward()
    xd = nhwc(x, dtype).to(DEV).requires_grad_(True)
    wd, bd = torch.nn.Parameter(w.to(DEV)), torch.nn.Parameter(b.to(DEV))
    y = ops.head(xd, wd, bd, sig)
    assert rel(y, yr) < tol
    y.backward(cot.to(DEV))
    assert rel(nchw(xd.grad), xr.grad) < 2 * tol
    assert rel(wd.grad, wr.grad) < 2 * tol and rel(bd.grad, br.grad) < 2 * tol


# ----------------------------------------------------------------------------------------------
# posterior step, Darcy residual + fused loss (q_sample and the optimizer: test_gpu_glue_census.py)
# ----------------------------------------------------------------------------------------------
def test_posterior_step(pk):
    ops, _ = pk
    from oracle import pidm_oracle as O
    tab = O.diffusion_tables(100)
    g = torch.Generator().manual_seed(10)
    x0, xt = torch.randn(5, 2, 64, 64, generator=g), torch.randn(5, 2, 64, 64, generator=g)
    z = torch.randn(5, 2, 64, 64, generator=g)
    for i in (0, 7, 99):
        ref = O.posterior_step(xt, x0, z, i, tab)
        sig = 0. if i == 0 else tab['betas'][i].sqrt().item()
        got = ops.posterior_step(xt.to(DEV), x0.to(DEV), z.to(DEV), tab['posterior_mean_coef1'][i].item(),
                                 tab['posterior_mean_coef2'][i].item(), sig)
        assert torch.allclose(got.cpu(), ref, rtol=1e-5, atol=1e-5)


def test_darcy_residual_golden_and_oracle(pk, golden):
    ops, _ = pk
    from oracle import pidm_oracle as O
    gd = golden('darcy_residual.pt')
    fs = O.darcy_source(64).reshape(-1).to(DEV)
    x = gd['x0_pred'].to(DEV).requires_grad_(True)
    r = ops.darcy_residual(x, fs)
    # the residual amplifies fp32 rounding of x by 1/h^2 = 3969: compare in norm (north_star: 1e-5 relative)
    assert rel(r, gd['residual']) < 1e-5
    (r * gd['cotangent'].to(DEV)).sum().backward()
    assert rel(x.grad, gd['grad_x0_pred']) < 1e-5
    # larger random batch (several samples per persistent CTA: exercises the double-buffered TMA ring)
    g = torch.Generator().manual_seed(11)
    xb = torch.randn(700, 2, 64, 64, generator=g)
    rb = ops.darcy_residual(xb.to(DEV), fs)
    assert rel(rb, O.darcy_residual(xb)) < 1e-5


def test_darcy_fused_loss_matches_oracle(pk):
    ops, _ = pk
    from oracle import pidm_oracle as O
    tab = O.diffusion_tables(100)
    g = torch.Generator().manual_seed(12)
    B = 6
    x0 = torch.randn(B, 2, 64, 64, generator=g)
    xh = (x0 + 0.3 * torch.randn(B, 2, 64, 64, generator=g)).requires_grad_(True)
    mo = (x0 + 0.2 * torch.randn(B, 2, 64, 64, generator=g)).requires_grad_(True)
    t = torch.tensor([0, 1, 40, 77, 98, 99])
    fs = O.darcy_source(64).reshape(-1).to(DEV)
    p2, pv = tab['p2_loss_weight'].to(DEV), tab['posterior_variance_clipped'].to(DEV)
    for same in (True, False):
        xh.grad = mo.grad = None
        model_out = xh if same else mo
        loss_r, data_r, rabs_r = O.pidm_loss_from_x0pred(x0, model_out, O.darcy_residual(xh), t, tab, 1.0, 1e-3)
        loss_r.backward()
        xd = xh.detach().to(DEV).requires_grad_(True)
        md = xd if same else mo.detach().to(DEV).requires_grad_(True)
        loss, sums = ops.darcy_pidm_loss(xd, md, x0.to(DEV), t.to(DEV), fs, p2, pv, 1.0, 1e-3)
        # north_star: residual loss within 1e-5 relative of the reference on identical x0_hat
        assert abs(loss.item() / loss_r.item() - 1) < 1e-5
        assert abs(sums[0].item() / data_r.item() - 1) < 1e-5 and abs(sums[2].item() / rabs_r.item() - 1) < 1e-5
        (loss * 2.0).backward()
        assert rel(xd.grad, 2 * xh.grad) < 2e-5
        if not same:
            assert rel(md.grad, 2 * mo.grad) < 2e-5


def test_fd_stencil(pk):
    from physicsinformeddiffusionmodels_b200.grad_utils import GradientsHelper
    from oracle import pidm_oracle as O
    g = torch.Generator().manual_seed(13)
    u = torch.randn(3, 64, 64, generator=g)
    gh = GradientsHelper(d0=1 / 63, d1=-1 / 63, fd_acc=2)
    ud = u.to(DEV)
    assert rel(gh.stencil_gradients(ud, 'd_d0'), O.fd_first(u, -2, 1 / 63)) < 1e-5
    assert rel(gh.stencil_gradients(ud, 'd_d1'), O.fd_first(u, -1, -1 / 63)) < 1e-5
    assert rel(gh.stencil_gradients(ud, 'd_d00'), O.fd_second(u, -2, 1 / 63)) < 1e-5
    assert rel(gh.stencil_gradients(ud, 'd_d11'), O.fd_second(u, -1, -1 / 63)) < 1e-5
    assert rel(gh.stencil_gradients(ud, 'd_d01'), O.fd_first(O.fd_first(u, -1, -1 / 63), -2, 1 / 63)) < 1e-5


def test_mechanics_residual_golden(pk, golden):
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    gd = golden('mechanics_residual.pt')
    res = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV)
    assert torch.allclose(res.KE.cpu(), gd['KE'], atol=1e-6)
    x = gd['x0_pred'].to(DEV).requires_grad_(True)
    out = res.compute_residual((x, gd['bcs'].to(DEV), gd['vf'].to(DEV), None), reduce='per-batch',
                               return_optimizer=True, return_inequality=True, pass_through=True)
    # matrix-free evaluation vs the reference's dense 8450x8450 assembly: fp32 summation order only
    assert rel(out['residual'], gd['residual']) < 2e-5
    assert rel(out['optimizer'], gd['compliance']) < 2e-5
    assert torch.allclose(out['inequality'].cpu(), gd['inequality'], atol=1e-6)
    ((out['residual'] * gd['cotangent'].to(DEV)).sum() + 0.3 * out['optimizer'].sum()
     + 2.0 * out['inequality'].sum()).backward()
    assert rel(x.grad, gd['grad_x0_pred']) < 5e-5


WG_CASES = [
    # B, H, Cin, Cout, k
    (2, 64, 32, 32, 3),       # 64x64 C=32: 4 taps per M' tile (64B swizzle atoms), 3 M' tiles, last one padded
    (2, 32, 64, 64, 3),       # 128B atoms, 2 (tap,chunk) pairs per tile
    (2, 32, 32, 64, 3),
    (4, 16, 128, 128, 3),
    (3, 8, 256, 256, 3),      # odd batch with TN = 2
    (2, 64, 32, 768, 1),      # to_qkv
    (2, 64, 256, 32, 1),      # to_out
    (2, 16, 256, 64, 3),
    (2, 8, 512, 128, 3),
    (2, 16, 64, 96, 3),       # Cout % 64 != 0 -> N' = 32
]


@pytest.mark.parametrize('case', WG_CASES, ids=[f'B{c[0]}_H{c[1]}_C{c[2]}x{c[3]}_k{c[4]}' for c in WG_CASES])
def test_wgrad_tcgen05_matches_reference(pk, case):
    """wgmma wgrad (MN-major TMA operands, split over pixels, fp32 atomics) vs autograd of F.conv2d on
    bf16-representable operands: fp32 accumulation both sides -> 2e-3 (summation order over up to 131072 pixels)."""
    ops, packing = pk
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    B, H, Cin, Cout, k = case
    assert call('pidm_conv2d_wgrad_tc_supported', B, H, H, Cin, Cout, k, k, 1) == 1
    g = torch.Generator().manual_seed(31)
    x = torch.randn(B, Cin, H, H, generator=g).bfloat16().float()
    w = (torch.randn(Cout, Cin, 1, k, k, generator=g) / math.sqrt(Cin * k * k)).requires_grad_(True)
    b = torch.zeros(Cout, requires_grad=True)
    y = F.conv2d(x, w[:, :, 0], b, padding=k // 2)
    cot = torch.randn(y.shape, generator=g).bfloat16().float()
    (y * cot).sum().backward()
    xd, dyd = nhwc(x, torch.bfloat16).to(DEV), nhwc(cot, torch.bfloat16).to(DEV)
    dw = torch.zeros(Cout, Cin, 1, k, k, device=DEV)
    db = torch.zeros(Cout, device=DEV)
    args = (xd, dyd, dw, B, H, H, Cin, Cin, H, H, Cout, k, k, 1, k // 2, k * k, Cin * k * k, stream())
    call('pidm_conv2d_wgrad_tc', *args)
    call('pidm_colsum', dyd, db, B * H * H, Cout, 1, stream())
    torch.cuda.synchronize()
    assert rel(dw, w.grad) < 2e-3, rel(dw, w.grad)
    assert rel(db, b.grad) < 2e-3
    # accumulate semantics: a second call doubles the buffers
    call('pidm_conv2d_wgrad_tc', *args)
    assert rel(dw, 2 * w.grad) < 2e-3


TC_GENERAL_CASES = [
    # name, kind, Cin, Cout, k, stride, pad, H (input), B
    ('stem7x7_pad32', 'conv', 2, 32, 7, 1, 3, 64, 2),
    ('down4x4s2_c32', 'conv', 32, 32, 4, 2, 1, 64, 2),
    ('down4x4s2_c64', 'conv', 64, 64, 4, 2, 1, 32, 2),
    ('down4x4s2_c128', 'conv', 128, 128, 4, 2, 1, 16, 3),
    ('up4x4s2T_c128', 'convT', 128, 128, 4, 2, 1, 8, 3),
    ('up4x4s2T_c64', 'convT', 64, 64, 4, 2, 1, 16, 2),
    ('up4x4s2T_c32', 'convT', 32, 32, 4, 2, 1, 32, 2),
]


@pytest.mark.parametrize('case', TC_GENERAL_CASES, ids=[c[0] for c in TC_GENERAL_CASES])
def test_conv_tcgen05_strided_transposed_and_stem(pk, case):
    """Stride-2 conv (TMA elementStrides), stride-2 transposed conv (4 output-parity classes) and the channel-padded
    7x7 stem through the tensor-core (wgmma) kernels: forward, dgrad and wgrad vs autograd of torch conv ops on bf16-representable
    operands (1e-2: bf16 rounding of outputs)."""
    ops, packing = pk
    from physicsinformeddiffusionmodels_b200._lib import call
    name, kind, Cin, Cout, k, stride, pad, H, B = case
    ops.set_tensor_core_conv(True)
    g = torch.Generator().manual_seed(41)
    x = torch.randn(B, Cin, H, H, generator=g).bfloat16().float()
    wshape = (Cout, Cin, 1, k, k) if kind == 'conv' else (Cin, Cout, 1, k, k)
    w = (torch.randn(wshape, generator=g) / math.sqrt(Cin * k * k)).bfloat16().float()
    b = torch.randn(Cout, generator=g) * 0.1
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    if kind == 'conv':
        yr = F.conv2d(xr, wr[:, :, 0], br, stride=stride, padding=pad)
    else:
        yr = F.conv_transpose2d(xr, wr[:, :, 0], br, stride=stride, padding=pad)
    cot = torch.randn(yr.shape, generator=g).bfloat16().float()
    (yr * cot).sum().backward()
    cpad = (Cin + 31) // 32 * 32
    Ho = yr.shape[-1]
    assert call('pidm_conv2d_tc_general_supported', B, H, H, cpad, Ho, Ho, Cout, k, k, stride, pad,
                1 if kind == 'convT' else 0) == 1
    wd, bd = torch.nn.Parameter(w.to(DEV)), torch.nn.Parameter(b.to(DEV))
    spec = packing.ConvSpec(wd, kind, k, k, stride, pad, cin_pad=cpad, need_dgrad=(cpad == Cin))
    packer = packing.WeightPacker()
    packer.add(spec)
    packer.refresh(torch.bfloat16)
    xin = torch.zeros(B, H, H, cpad)
    xin[..., :Cin] = x.permute(0, 2, 3, 1)
    xd = xin.to(DEV).bfloat16().requires_grad_(cpad == Cin)
    y = ops.conv2d(xd, wd, bd, spec)
    assert rel(nchw(y), yr) < 1e-2, f'{name} fwd {rel(nchw(y), yr)}'
    y.backward(nhwc(cot, torch.bfloat16).to(DEV))
    assert rel(wd.grad, wr.grad) < 1e-2, f'{name} wgrad {rel(wd.grad, wr.grad)}'
    assert rel(bd.grad, br.grad) < 1e-2, f'{name} bgrad'
    if cpad == Cin:
        assert rel(nchw(xd.grad), xr.grad) < 1e-2, f'{name} dgrad {rel(nchw(xd.grad), xr.grad)}'
