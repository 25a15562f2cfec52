"""The linear-attention block at the 32-channel levels (pidm_linattn_block_{fwd,bwd,wgrad}): to_qkv, the linear
attention, to_out (1x1, 256 -> 32, with bias) and the residual add, without materialising the [B, N, 256] attention
output or its gradient.

Every launch is driven through the C ABI on seeded bf16-exact operands and checked per element against an fp64
reference, in the bound form of the launch census (tests/test_gpu_launch_census.py): 2^-7 |r| + b rms(slice).  The
residual and the bias are scaled to the rms of the attention term, so that each of the three terms of y is visible to
the bound.  Outputs sit between NaN guard regions; accumulated gradients are prefilled.  Edited references (a head's
partial missing from y, the bias or the residual missing, the last pixel chunk repeated, one head's dW_out block
transposed) must be rejected by the same predicates."""
import math

import pytest
import torch

from test_gpu_launch_census import (A_ATT, B_ATT, DEV, GUARD_BF16, _gen, _guarded, _guards_intact, _ratio, _randn,
                                    plan_laf)

pytestmark = pytest.mark.gpu

B_Y = 2.0 ** -3          # y: slice = sample
B_DX = B_ATT['bwd']      # dxn: slice = sample
B_GW = B_ATT['wgrad']    # dW_qkv: slice = (q | k | v, head); dW_out: slice = head's 32 columns; db: whole vector
PREFILL = 2.0 ** -14     # fp32 accumulation into a prefilled gradient: one rounding of the prefill


def _ref(xn, wq, wo, bo, res, dy, need_grad, chunk=8):
    """fp64: y = res + bo + attention(xn Wq^T) Wo^T, and with need_grad the gradients for the cotangent dy.
    Returns y, dxn, dWq [768,32], dWo [32,256], db [32], and the attention output out [B,N,256]."""
    B, N, _ = xn.shape
    ys, dxs, outs = [], [], []
    gq = torch.zeros(768, 32, dtype=torch.float64, device=DEV)
    go = torch.zeros(32, 256, dtype=torch.float64, device=DEV)
    for b0 in range(0, B, chunk):
        with torch.set_grad_enabled(need_grad):
            xr = xn[b0:b0 + chunk].double().requires_grad_(need_grad)
            wqr = wq.double().requires_grad_(need_grad)
            wor = wo.double().requires_grad_(need_grad)
            nb = xr.shape[0]
            q, k, v = (xr @ wqr.t()).view(nb, N, 3, 8, 32).permute(2, 0, 3, 4, 1)
            q = q.softmax(dim=-2) * 32 ** -0.5
            k = k.softmax(dim=-1)
            v = v / N
            ctx = torch.einsum('bhdn,bhen->bhde', k, v)
            out = torch.einsum('bhde,bhdn->bhen', ctx, q).permute(0, 3, 1, 2).reshape(nb, N, 256)
            y = res[b0:b0 + chunk].double() + bo.double() + out @ wor.t()
            if need_grad:
                (y * dy[b0:b0 + chunk].double()).sum().backward()
                dxs.append(xr.grad)
                gq += wqr.grad
                go += wor.grad
        ys.append(y.detach())
        outs.append(out.detach())
    db = dy.double().sum(dim=(0, 1)) if need_grad else None
    return (torch.cat(ys), torch.cat(dxs) if need_grad else None, gq, go, db, torch.cat(outs))


def y_bound(r):                       # [B, N, 32]: slice = sample
    rms = r.pow(2).mean(dim=(1, 2), keepdim=True).sqrt()
    return A_ATT * r.abs() + B_Y * rms


def dx_bound(r):
    rms = r.pow(2).mean(dim=(1, 2), keepdim=True).sqrt()
    return A_ATT * r.abs() + B_DX * rms


def gq_bound(r, prefill):             # [768, 32]
    rh = r.view(24, 32, 32)
    rms = rh.pow(2).mean(dim=(1, 2), keepdim=True).sqrt()
    return (A_ATT * rh.abs() + B_GW * rms).view(768, 32) + PREFILL * prefill.abs()


def go_bound(r, prefill):             # [32, 256]: slice = one head's 32 columns
    rh = r.view(32, 8, 32)
    rms = rh.pow(2).mean(dim=(0, 2), keepdim=True).sqrt()
    return (A_ATT * rh.abs() + B_GW * rms).view(32, 256) + PREFILL * prefill.abs()


def db_bound(r, prefill):
    return A_ATT * r.abs() + B_GW * r.pow(2).mean().sqrt() + PREFILL * prefill.abs()


class BlockCase:
    def __init__(self, B, N, need_grad=True):
        self.B, self.N = B, N
        g = _gen(('linattn-block', B, N))
        self.xn = _randn(g, B, N, 32)
        self.wq = _randn(g, 768, 32, scale=1.5 / math.sqrt(32))
        self.wo = _randn(g, 32, 256, scale=1.0 / math.sqrt(256))
        # the attention term of y is ~1/N of its inputs (v / N): residual and bias at its rms
        _, _, _, _, _, out = _ref(self.xn[:1], self.wq, self.wo, torch.zeros(32, device=DEV),
                                  torch.zeros(1, N, 32, device=DEV), None, False)
        s = (out @ self.wo.double().t()).pow(2).mean().sqrt().item()
        self.res = _randn(g, B, N, 32, scale=s)
        self.bo = _randn(g, 32, scale=s, dtype=torch.float32).bfloat16().float()
        self.dy = _randn(g, B, N, 32)
        self.y_r, self.dx_r, self.gq_r, self.go_r, self.db_r, self.out_r = _ref(
            self.xn, self.wq, self.wo, self.bo, self.res, self.dy, need_grad)

    def fwd(self):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, N = self.B, self.N
        self.ctx = torch.empty(B, 8, 32, 32, device=DEV)
        self.kmax, self.kzinv = torch.empty(B, 8, 32, device=DEV), torch.empty(B, 8, 32, device=DEV)
        ws = torch.empty(call('pidm_linattn_fused_workspace_floats', B, N), device=DEV)
        n = B * N * 32
        buf, y, guard = _guarded(n, GUARD_BF16)
        call('pidm_linattn_block_fwd', self.xn, self.wq, self.wo, self.bo, self.res, y, self.ctx, self.kmax, self.kzinv,
             ws, B, N, stream())
        torch.cuda.synchronize()
        return y.view(B, N, 32), _guards_intact(buf, guard, n, GUARD_BF16)

    def bwd(self):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, N = self.B, self.N
        n = B * N * 32
        buf, dx, guard = _guarded(n, GUARD_BF16)
        self.dctx = torch.empty_like(self.ctx)
        call('pidm_linattn_block_bwd', self.xn, self.wq, self.wo, self.dy, self.ctx, self.kmax, self.kzinv, dx, self.dctx,
             B, N, stream())
        torch.cuda.synchronize()
        return dx.view(B, N, 32), _guards_intact(buf, guard, n, GUARD_BF16)

    def wgrad(self):
        """both weight gradients accumulated into strided views of one prefilled flat buffer (as the engine's flat
        gradient buffer), and the bias gradient by pidm_colsum; returns (dWq, dWo, db) minus the prefill, guards ok"""
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, N = self.B, self.N
        g = _gen(('linattn-block-gw', B, N))
        guard = 1024
        nq, no = 768 * 32, 32 * 256
        gbuf = torch.randn(nq + no + 32 + 4 * guard, generator=g, device=DEV)
        keep = gbuf.clone()
        gq = gbuf[guard:guard + nq].view(768, 32)
        go = gbuf[2 * guard + nq:2 * guard + nq + no].view(32, 256)
        gb = gbuf[3 * guard + nq + no:3 * guard + nq + no + 32]
        call('pidm_linattn_block_wgrad', self.xn, self.wq, self.wo, self.dy, self.ctx, self.dctx, self.kmax, self.kzinv,
             gq, 32, 1, go, 256, 1, B, N, stream())
        call('pidm_colsum', self.dy, gb, B * N, 32, 1, stream())
        torch.cuda.synchronize()
        touched = torch.zeros_like(gbuf, dtype=torch.bool)
        for a, n in ((guard, nq), (2 * guard + nq, no), (3 * guard + nq + no, 32)):
            touched[a:a + n] = True
        ok = bool((gbuf[~touched] == keep[~touched]).all())
        kq = keep[guard:guard + nq].view(768, 32).double()
        ko = keep[2 * guard + nq:2 * guard + nq + no].view(32, 256).double()
        kb = keep[3 * guard + nq + no:3 * guard + nq + no + 32].double()
        self.prefill = (kq, ko, kb)
        return (gq.double() - kq, go.double() - ko, gb.double() - kb), ok

    def y_ratio(self, y):
        return _ratio((y.double() - self.y_r).abs(), y_bound(self.y_r))

    def go_ratio(self, go):
        return _ratio((go.double() - self.go_r).abs(), go_bound(self.go_r, self.prefill[1]))


# every shape the benchmark runs the block at (Darcy training at batch 32: 64x64 and 32x32; sampling forward at batch
# 16 / 64 / 256, 64x64 and 32x32), and shapes whose last pixel chunk is ragged in every kernel
TRAIN = [(32, 4096), (32, 1024), (5, 4096), (24, 4096)]
SAMPLE = [(b, n) for b in (16, 64, 256) for n in (4096, 1024)]


def _ragged(B, N, kind):
    p = plan_laf(B, N)
    px = {'fwd': p['ctx'], 'bwd': p['bwd'], 'wgrad': p['wgrad']}[kind]      # the block forward runs two CTAs per SM
    return N % px != 0


def test_shapes_reach_a_ragged_last_chunk():
    for kind in ('fwd', 'bwd', 'wgrad'):
        assert any(_ragged(B, N, kind) for B, N in TRAIN), kind


@pytest.mark.parametrize('B,N', SAMPLE, ids=[f'B{b}-N{n}' for b, n in SAMPLE])
def test_block_forward(B, N):
    c = BlockCase(B, N, need_grad=False)
    y, ok = c.fwd()
    assert ok, 'a store landed outside y'
    r = c.y_ratio(y)
    print(f'[block] fwd B={B} N={N} worst |err|/bound {r:.4g}')
    assert r <= 1.0, r


_CASES = {}


def _case(B, N):
    if (B, N) not in _CASES:
        _CASES.clear()
        _CASES[(B, N)] = BlockCase(B, N)
    return _CASES[(B, N)]


@pytest.mark.parametrize('B,N', TRAIN, ids=[f'B{b}-N{n}' for b, n in TRAIN])
def test_block_forward_backward_wgrad(B, N):
    c = _case(B, N)
    y, ok = c.fwd()
    assert ok, 'a store landed outside y'
    ry = c.y_ratio(y)
    dx, ok = c.bwd()
    assert ok, 'a store landed outside dxn'
    rx = _ratio((dx.double() - c.dx_r).abs(), dx_bound(c.dx_r))
    (gq, go, gb), ok = c.wgrad()
    assert ok, 'an element outside the weight and bias gradients changed'
    rq = _ratio((gq - c.gq_r).abs(), gq_bound(c.gq_r, c.prefill[0]))
    ro = _ratio((go - c.go_r).abs(), go_bound(c.go_r, c.prefill[1]))
    rb = _ratio((gb - c.db_r).abs(), db_bound(c.db_r, c.prefill[2]))
    print(f'[block] B={B} N={N} worst |err|/bound: y {ry:.4g} dxn {rx:.4g} dWqkv {rq:.4g} dWout {ro:.4g} db {rb:.4g}')
    assert max(ry, rx, rq, ro, rb) <= 1.0, (ry, rx, rq, ro, rb)


# ---- the predicates reject subtly wrong outputs (edits of the fp64 reference; no faulty code runs on the GPU) --------
def _bf16(t):
    return t.to(torch.bfloat16)


def test_mutants_rejected():
    B, N = next((b, n) for b, n in TRAIN if _ragged(b, n, 'fwd'))
    c = _case(B, N)
    assert c.y_ratio(_bf16(c.y_r)) <= 1.0
    head = c.out_r[..., 3 * 32:4 * 32] @ c.wo.double()[:, 3 * 32:4 * 32].t()
    assert c.y_ratio(_bf16(c.y_r - head)) > 1.0, 'one head partial missing'
    assert c.y_ratio(_bf16(c.y_r - c.bo.double())) > 1.0, 'bias missing'
    assert c.y_ratio(_bf16(c.y_r - c.res.double())) > 1.0, 'residual missing'
    px = plan_laf(B, N)['ctx']
    last = (N - 1) // px * px
    y = c.y_r.clone()
    y[:, last:] = c.y_r[:, last - px:last - px + (N - last)]
    assert c.y_ratio(_bf16(y)) > 1.0, 'last chunk repeated'
    c.prefill = (None, torch.zeros(32, 256, dtype=torch.float64, device=DEV), None)
    assert c.go_ratio(c.go_r.float()) <= 1.0
    go = c.go_r.clone()
    go[:, 32 * 5:32 * 6] = c.go_r[:, 32 * 5:32 * 6].t()
    assert c.go_ratio(go.float()) > 1.0, "one head's dW_out block transposed"


# ---- through autograd: the block op == linear_attention_fused followed by the to_out convolution ----------------------
@pytest.mark.parametrize('B,H', [(4, 64), (3, 32)])
def test_block_op_matches_unfused_composition(B, H):
    from physicsinformeddiffusionmodels_b200 import ops, packing
    ops.set_precision('bf16')
    ops.set_tensor_core_conv(True)
    g = _gen(('linattn-block-autograd', B, H))
    wq = torch.nn.Parameter(_randn(g, 768, 32, 1, 1, 1, scale=1.5 / math.sqrt(32), dtype=torch.float32).bfloat16().float())
    wo = torch.nn.Parameter(_randn(g, 32, 256, 1, 1, 1, scale=1.0 / math.sqrt(256), dtype=torch.float32).bfloat16().float())
    bo = torch.nn.Parameter(_randn(g, 32, scale=1e-3, dtype=torch.float32))
    sq, so = packing.ConvSpec(wq, 'conv', 1, 1, 1, 0), packing.ConvSpec(wo, 'conv', 1, 1, 1, 0)
    pk = packing.WeightPacker()
    pk.add(sq)
    pk.add(so)
    pk.refresh(torch.bfloat16)
    xn0 = _randn(g, B, H, H, 32)
    x0 = _randn(g, B, H, H, 32, scale=1e-3)
    dy = _randn(g, B, H, H, 32)

    def run(block):
        for p in (wq, wo, bo):
            p.grad = None
        xn = xn0.clone().requires_grad_(True)
        x = x0.clone().requires_grad_(True)
        if block:
            assert ops.linear_attention_block_supported(xn, sq, so, bo, 8)
            y = ops.linear_attention_block(xn, wq, sq, wo, bo, so, x, 8)
        else:
            y = ops.conv2d(ops.linear_attention_fused(xn, wq, sq, 8), wo, bo, so, residual=x)
        y.backward(dy)
        torch.cuda.synchronize()
        return [t.double() for t in (y, xn.grad, x.grad, wq.grad, wo.grad, bo.grad)]
    got, ref = run(True), run(False)
    names = ('y', 'dxn', 'dx', 'dWqkv', 'dWout', 'db')
    for name, a, r in zip(names, got, ref):
        # the two compositions sum in different orders and round dout / y to bf16 at different points
        tol = 2.0 ** -7 * r.abs() + 2.0 ** -7 * r.pow(2).mean().sqrt()
        q = _ratio((a - r).abs(), tol)
        print(f'[block] autograd {name}: worst |diff|/tol {q:.3g}')
        assert q <= 1.0, (name, q)
    assert torch.equal(got[2], dy.double()), 'the residual gradient is dy'
