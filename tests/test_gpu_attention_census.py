"""Every standalone linear-attention, mid softmax-attention and output-head launch of the benchmarked steps, and every
launch plan of attention.cu / attention_mid.cu and the head kernels, replayed element by element against an fp64
reference.

pidm_linattn_fwd takes one of three forward paths (one CTA per (sample, head) for bf16 at 32 <= N <= 64, mma.sync for
bf16 with 8 heads and N % 64 == 0, SIMT statistics -> context -> output otherwise) and one of two backward paths, and
sizes its pixel chunks from the batch and the SM count; pidm_attn_* take the 64-token mma.sync kernels or the CUDA-core
kernels with padded keys masked; pidm_head_bwd takes an octet kernel or a general one with a ragged last warp.  The
operator tests in test_gpu_ops.py compare whole tensors at batch 2 or 3 by a norm ratio, which a wrong last chunk, a
wrong head slice or a missing key mask at one shape cannot move.  Same four parts as the other census files:

  1. census: the distinct keys of the six entry points in one eager step of every workload bench.py times must equal
     the tables below (`python tests/census.py --print-table` regenerates them);
  2. replay: every table row plus synthetic rows, through the C ABI, with bf16 and with fp32 activations, on seeded
     operands exact in the activation type, against the fp64 evaluation of the contract in include/pidm.h.  With
     u = 2^-24, rnd = 2^-8 (bf16 output) or 2^-24 (fp32 output) and A the absolute-value evaluation of the same chain
     (p >= 0 and k~ >= 0, so A is the chain with |v|, |dout|, |ctx| and the absolute values of the other factors):
        every output            |o - r| <= rnd |r| + C eps A          (fp32 outputs: rnd = u)
        kmax                    exact (the fp32 column maximum)
        head y                  |o - r| <= C sqrt(C_in) u A   (+ the sigmoid's own error on the last channel)
        head dW, db             |o - r| <= C sqrt(M) u (|prefill| + A)
     eps states which intermediates each path rounds:
        SIMT kernels, la_small_fwd, the CUDA-core softmax attention, the statistics kernel: fp32 intermediates and the
          fast exponential (attention*.cu are built with --use_fast_math: about u (8 + 2|z|) relative, see
          test_gpu_norm_census._silu_terms): eps = u (16 + 2 z + 2 sqrt(N)), z = the largest |exponent argument|;
        mma.sync linear attention: exp(k - M), p, ctx and dctx are rounded to bf16 before mma.sync: eps += 2^-8 per
          rounding along the output's chain (MMA_ROUNDINGS);
        attention_mid.cu: P (and in the backward dS) is rounded to bf16: eps += 2^-8; the score error
          <= sqrt(32) u s sum_d |q| |k| is carried through the softmax (2 max_j e_S relative on P);
        head: __expf on the last channel although elementwise.cu is an exact unit: u (8 + 2|z|) on sigma.
     The linear-attention backward is checked twice: *given the statistics* (fp64 ctx / kmax / kzinv rounded to fp32
     and fed to the kernel; the reference uses those values) and *end to end* (the forward's own outputs; the bound
     is widened by the forward's ctx bound and the relative kzinv bound).  At bf16 and N = 64 the end-to-end check is
     the one-CTA forward -> mma.sync backward hand-off.  Overwritten outputs start as NaN between NaN guards; the
     head's dW / db are prefilled, because they accumulate; dctx is scratch, so only its guards are checked;
  3. mutants: the predicates reject the fp64 reference edited the way a subtle kernel bug would change it;
  4. plan coverage: pidm_linattn_plan (and the mid-attention choice and the head's grid / octet rule, restated here)
     show that the rows reach every path, every hand-off, ragged last chunks and tiles, and capped grids.
"""
import math

import pytest
import torch

from census import assert_census_in_tables, assert_tables_in_census
from checks import (CODE, DTYPES, NAME, RND, U, assert_ok, gen, guarded, guards_intact, note_all, ratios, rounded,
                    sms)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TAG = 'attention census'
BF = 2.0 ** -8
SCALE = float(torch.tensor(32 ** -0.5, dtype=torch.float32))       # the kernels' fp32 32^-1/2
# C_LA and C_ATT stayed at 1 after a run on an H100 80GB HBM3 (700 W).  C_HEAD is 2: at C = 8 over 570 k outputs the
# largest fp32 accumulation error of y reached 1.2 sqrt(C) u A.  The worst |err| / bound per kernel path is recorded in
# DESIGN.md section 2.
C_LA = 1.0
C_ATT = 1.0
C_HEAD = 2.0
# bf16 roundings before mma.sync along the chain of each linear-attention output: ctx <- exp(k - M); out <- exp(k - M),
# ctx, p; dq <- p, ctx; dk, dv <- p (in dctx), dctx, k~
MMA_ROUNDINGS = {'ctx': 1, 'out': 3, 'dq': 2, 'dk': 3, 'dv': 3}
FWD_PATHS = {0: 'small', 1: 'mma', 2: 'simt'}
BWD_PATHS = {0: 'mma', 1: 'simt'}

# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`)
# ----------------------------------------------------------------------------------------------------------------------
# pidm_linattn_fwd / _bwd: B, N, heads, dtype
LA_FWD_TABLE = [
    (16, 64, 8, 'bf16'),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 256, 8, 'bf16'),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 1024, 8, 'bf16'),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 64, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
    (32, 256, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
    (32, 1024, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
    (32, 4096, 8, 'bf16'),  # mech_train_b32
    (64, 64, 8, 'bf16'),  # darcy_sample_b64
    (64, 256, 8, 'bf16'),  # darcy_sample_b64
    (64, 1024, 8, 'bf16'),  # darcy_sample_b64
    (256, 64, 8, 'bf16'),  # darcy_sample_b256
    (256, 256, 8, 'bf16'),  # darcy_sample_b256
    (256, 1024, 8, 'bf16'),  # darcy_sample_b256
]
LA_BWD_TABLE = [
    (32, 64, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
    (32, 256, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
    (32, 1024, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
    (32, 4096, 8, 'bf16'),  # mech_train_b32
]
# pidm_attn_fwd / _bwd: B, n_tokens, heads, dtype
ATTN_FWD_TABLE = [
    (16, 64, 8, 'bf16'),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 64, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
    (64, 64, 8, 'bf16'),  # darcy_sample_b64
    (256, 64, 8, 'bf16'),  # darcy_sample_b256
]
ATTN_BWD_TABLE = [
    (32, 64, 8, 'bf16'),  # darcy_train_b32 mech_train_b32
]
# pidm_head_fwd / _bwd: B, HW, C, O, sigmoid_last, dtype
HEAD_FWD_TABLE = [
    (16, 4096, 32, 2, 0, 'bf16'),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 4096, 32, 2, 0, 'bf16'),  # darcy_train_b32
    (32, 4096, 128, 3, 1, 'bf16'),  # mech_train_b32
    (64, 4096, 32, 2, 0, 'bf16'),  # darcy_sample_b64
    (256, 4096, 32, 2, 0, 'bf16'),  # darcy_sample_b256
]
HEAD_BWD_TABLE = [
    (32, 4096, 32, 2, 0, 'bf16'),  # darcy_train_b32
    (32, 4096, 128, 3, 1, 'bf16'),  # mech_train_b32
]
TABLES = {'la_fwd': LA_FWD_TABLE, 'la_bwd': LA_BWD_TABLE, 'attn_fwd': ATTN_FWD_TABLE, 'attn_bwd': ATTN_BWD_TABLE,
          'head_fwd': HEAD_FWD_TABLE, 'head_bwd': HEAD_BWD_TABLE}

# Rows no benchmarked step produces, for the branches the workloads do not reach (see test_plan_coverage; the plan on
# the 132-SM H100 is in the comment as bf16 | fp32).
LA_SYNTHETIC = [
    (256, 128, 8),    # mma fwd and bwd, one chunk per sample, one statistics chunk | simt
    (2, 4096, 8),     # mma, chunks clamped to 64 pixels, 32 statistics chunks (the cap) | simt, 16 context chunks
    (5, 4096, 8),     # mma, 96-pixel chunks, the last one 64 (ctx, out and bwd) | simt
    (3, 96, 8),       # simt fwd and bwd (N % 64 != 0), one 128-row context chunk ragged in its second tile | same
    (2, 1056, 8),     # simt, 8 statistics chunks, 5 context chunks of 256 rows, the last 32 | same
    (3, 32, 8),       # one-CTA fwd -> simt bwd (N = 32) | simt
    (7, 64, 8),       # one-CTA fwd -> mma bwd, odd batch | simt
    (2, 64, 4),       # one-CTA fwd -> simt bwd (4 heads) | simt
    (2, 256, 4),      # simt fwd and bwd, 4 heads | same
    (1, 128, 12),     # simt, 12 heads, one statistics chunk | same
]
ATTN_SYNTHETIC = [(3, 1, 8), (3, 7, 8), (2, 16, 8), (2, 33, 8), (2, 63, 4), (2, 64, 4), (5, 64, 8)]
HEAD_SYNTHETIC = [
    (3, 401, 8, 1, 0),        # octet kernel, 1 lane per pixel
    (2, 300, 16, 2, 1),       # octet, 2 lanes
    (5, 123, 32, 3, 1),       # octet, 4 lanes
    (1, 1000, 64, 4, 0),      # octet, 8 lanes
    (2, 77, 128, 3, 1),       # octet, 16 lanes
    (3, 99, 256, 2, 0),       # octet, 32 lanes
    (3, 401, 24, 2, 1),       # general kernel, C / 8 = 3, M % 32 = 19
    (2, 333, 48, 4, 0),       # general, C / 8 = 6, M % 32 = 26
    (1, 261, 512, 1, 1),      # general, C / 8 = 64, M % 32 = 5
    (3, 190000, 8, 2, 1),     # forward grid capped: 2 grid-stride passes; octet backward capped: 5 passes
    (2, 40000, 24, 3, 0),     # general backward grid capped: 2 passes
]

LA_FWD_ROWS = [k[:3] for k in LA_FWD_TABLE] + LA_SYNTHETIC
LA_BWD_ROWS = [k[:3] for k in LA_BWD_TABLE] + [k for k in LA_SYNTHETIC if k[2] % 4 == 0]
ATTN_FWD_ROWS = [k[:3] for k in ATTN_FWD_TABLE] + ATTN_SYNTHETIC
ATTN_BWD_ROWS = [k[:3] for k in ATTN_BWD_TABLE] + ATTN_SYNTHETIC
HEAD_FWD_ROWS = [k[:5] for k in HEAD_FWD_TABLE] + HEAD_SYNTHETIC
HEAD_BWD_ROWS = [k[:5] for k in HEAD_BWD_TABLE] + HEAD_SYNTHETIC


def _id(k):
    return '_'.join(str(v) for v in k)


# ----------------------------------------------------------------------------------------------------------------------
# census
# ----------------------------------------------------------------------------------------------------------------------
def test_census_is_covered_by_the_table():
    assert_census_in_tables(TABLES)


def test_every_table_row_is_produced_by_the_census():
    assert_tables_in_census(TABLES)


# ----------------------------------------------------------------------------------------------------------------------
# plans
# ----------------------------------------------------------------------------------------------------------------------
def plan_la(B, N, heads, dtype):
    from physicsinformeddiffusionmodels_b200._lib import call
    out = torch.zeros(8, dtype=torch.int32)
    rc = call('pidm_linattn_plan', B, N, heads, CODE[dtype], out.data_ptr())
    assert rc == 0, f'linattn rejects B={B} N={N} heads={heads} {NAME[dtype]}'
    v = out.tolist()
    return dict(fwd=v[0], bwd=v[1], stat_chunks=v[2], stat_rows=v[3], ctx_rows=v[4], ctx_chunks=v[5], mma_px=v[6],
                mma_chunks=v[7])


def attn_kernel(n, dtype):
    """pidm_attn_* restated: attention_mid.cu for bf16 at exactly 64 tokens, the CUDA-core kernels otherwise"""
    return 'mid' if dtype == torch.bfloat16 and n == 64 else 'core'


def plan_head(B, HW, C, O, bwd):
    """pidm_head_{fwd,bwd} restated: grid_for(n, 256, cap) = min(ceil(n / 256), cap); the forward caps at 16 CTAs per
    SM, the octet backward (C / 8 lanes per pixel, a power of two <= 32) at 4 over M * C / 8 items, the general
    backward at 2 over M pixels; each loops grid-stride"""
    M, lpp = B * HW, C // 8
    octet = lpp <= 32 and lpp & (lpp - 1) == 0
    if not bwd:
        items, cap, kernel = M, sms() * 16, 'fwd'
    elif octet:
        items, cap, kernel = M * lpp, sms() * 4, 'octet'
    else:
        items, cap, kernel = M, sms() * 2, 'general'
    grid = max(1, min(-(-items // 256), cap))
    return dict(kernel=kernel, lpp=lpp, grid=grid, passes=-(-items // (grid * 256)), ragged_warp=M % 32 != 0)


# ----------------------------------------------------------------------------------------------------------------------
# operands, references, bounds
# ----------------------------------------------------------------------------------------------------------------------
def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device=DEV) * scale


def _ein(eq, *t):
    return torch.einsum(eq, *t)


def _sample_chunk(N, HID):
    return max(1, (1 << 21) // (N * HID))


def _eps32(z, N):
    return U * (16 + 2 * z + 2 * math.sqrt(N))


class LaCase:
    """operands of one standalone linear-attention shape; ref_* give the fp64 reference and bounds per sample slice"""

    def __init__(self, B, N, heads, dtype, edge=None):
        self.B, self.N, self.heads, self.dtype, self.HID = B, N, heads, dtype, heads * 32
        g = gen(('la', B, N, heads, edge))
        qkv = _randn(g, B, N, 3, heads, 32, scale=1.5)
        if edge == 'spike in the last statistics chunk':
            qkv[:, N - 1, 1] = 40.0
        elif edge == 'saturated q rows':
            d = torch.arange(N, device=DEV) % 32
            qkv[:, torch.arange(N, device=DEV), 0, :, d] += 30.0
        elif edge == 'constant k column':
            qkv[:, :, 1, :, 0] = 0.75
        self.qkv = qkv.reshape(B, N, 3 * self.HID).to(dtype)
        self.dout = _randn(g, B, N, self.HID).to(dtype)
        self.plan = plan_la(B, N, heads, dtype)
        x = self.qkv.view(B, N, 3, heads, 32).float()
        zk = (x[:, :, 1] - x[:, :, 1].amax(dim=1, keepdim=True)).abs().max().item()
        zq = (x[:, :, 0] - x[:, :, 0].amax(dim=3, keepdim=True)).abs().max().item()
        self.eps32 = _eps32(max(zk, zq), N)
        self.chunk = _sample_chunk(N, self.HID)

    def eps_fwd(self, o):
        return self.eps32 + (MMA_ROUNDINGS[o] * BF if self.plan['fwd'] == 1 else 0.0)

    def eps_bwd(self, o):
        return self.eps32 + (MMA_ROUNDINGS[o] * BF if self.plan['bwd'] == 0 else 0.0)

    def _qkv(self, sl):
        x = self.qkv[sl].double().view(-1, self.N, 3, self.heads, 32).permute(2, 0, 3, 1, 4)
        return x[0], x[1], x[2]                               # [b, h, N, 32]

    def _dout(self, sl):
        return self.dout[sl].double().view(-1, self.N, self.heads, 32).permute(0, 2, 1, 3)

    def slices(self):
        return [slice(b0, min(self.B, b0 + self.chunk)) for b0 in range(0, self.B, self.chunk)]

    def ref_fwd(self, sl, mut=()):
        """fp64 out [b,N,HID], ctx [b,h,32,32], kmax / kzinv [b,HID] of samples sl and their bounds"""
        N, rnd, eps = self.N, RND[self.dtype], self.eps_fwd
        q, k, v = self._qkv(sl)
        p = torch.softmax(q, dim=-1)
        M = k.amax(dim=2, keepdim=True)
        E = torch.exp(k - M)
        Z = E.sum(dim=2, keepdim=True)
        kt = E / Z
        if 'k-softmax per statistics chunk' in mut:
            rows = self.plan['stat_rows']
            kt = torch.cat([torch.softmax(k[:, :, n0:n0 + rows], dim=2) for n0 in range(0, N, rows)], dim=2)
        vn = v if 'v not divided by N' in mut else v / N
        ctx = _ein('bhnd,bhne->bhde', kt, vn)
        a_ctx = _ein('bhnd,bhne->bhde', kt, v.abs()) / N
        ctx_o = ctx
        if 'ctx of head 0 from head 1' in mut:
            ctx_o = ctx.clone()
            ctx_o[:, 0] = ctx[:, 1]
        out = SCALE * _ein('bhnd,bhde->bhne', p, ctx_o)
        a_out = SCALE * _ein('bhnd,bhde->bhne', p, a_ctx)
        if 'last mma chunk from its neighbour' in mut:
            px, last = self.plan['mma_px'], (self.plan['mma_chunks'] - 1) * self.plan['mma_px']
            n = N - last
            out = out.clone()
            out[:, :, last:] = out[:, :, last - px:last - px + n]
        flat = lambda t: t.permute(0, 2, 1, 3).reshape(t.shape[0], N, self.HID)
        zinv = (1 / Z).reshape(-1, self.HID)
        r = {'out': flat(out), 'ctx': ctx, 'kmax': M.reshape(-1, self.HID), 'kzinv': zinv}
        b = {'out': flat(rnd * out.abs() + C_LA * eps('out') * a_out), 'ctx': C_LA * eps('ctx') * a_ctx + U * ctx.abs(),
             'kmax': torch.zeros_like(r['kmax']), 'kzinv': (C_LA * self.eps32 + U) * zinv}
        return r, b

    def ref_bwd(self, sl, ctx, kmax, kzinv, e_ctx=None, eps_kz=0.0, mut=()):
        """fp64 dq | dk | dv [b,N,3,HID] of samples sl from the given ctx [b,h,32,32], kmax / kzinv [b,HID] and the
        bound; e_ctx / eps_kz: the given statistics are off by up to e_ctx (absolute) and eps_kz (relative, kzinv)"""
        N, rnd, eps, h = self.N, RND[self.dtype], self.eps_bwd, self.heads
        q, k, v = self._qkv(sl)
        g = self._dout(sl)
        ctx = ctx.double()
        M, zi = kmax.double().view(-1, h, 1, 32), kzinv.double().view(-1, h, 1, 32)
        p = torch.softmax(q, dim=-1)
        kt = torch.exp(k - M) * zi
        dp = SCALE * _ein('bhne,bhde->bhnd', g, ctx)
        a_dp = SCALE * _ein('bhne,bhde->bhnd', g.abs(), ctx.abs())
        dq = p * (dp - (p * dp).sum(-1, keepdim=True))
        a_dq = p * (a_dp + (p * a_dp).sum(-1, keepdim=True))
        dctx = _ein('bhnd,bhne->bhde', SCALE * p, g)
        a_dctx = _ein('bhnd,bhne->bhde', SCALE * p, g.abs())
        cd = 0.0 if 'dk without the dctx ctx term' in mut else (dctx * ctx).sum(-1).unsqueeze(2)
        dk = kt * (_ein('bhne,bhde->bhnd', v, dctx) / N - cd)
        a_dk = kt * (_ein('bhne,bhde->bhnd', v.abs(), a_dctx) / N + (a_dctx * ctx.abs()).sum(-1).unsqueeze(2))
        dv = _ein('bhnd,bhde->bhne', kt, dctx) / N
        a_dv = _ein('bhnd,bhde->bhne', kt, a_dctx) / N
        w_dq = w_dk = w_dv = 0.0
        if e_ctx is not None:
            D = SCALE * _ein('bhne,bhde->bhnd', g.abs(), e_ctx)
            w_dq = p * (D + (p * D).sum(-1, keepdim=True))
            w_dk = eps_kz * a_dk + kt * (a_dctx * e_ctx).sum(-1).unsqueeze(2)
            w_dv = eps_kz * a_dv
        flat = lambda t: t.permute(0, 2, 1, 3).reshape(t.shape[0], N, self.HID)
        r = {'dq': flat(dq), 'dk': flat(dk), 'dv': flat(dv)}
        b = {'dq': flat(rnd * dq.abs() + C_LA * (eps('dq') * a_dq + w_dq)),
             'dk': flat(rnd * dk.abs() + C_LA * (eps('dk') * a_dk + w_dk)),
             'dv': flat(rnd * dv.abs() + C_LA * (eps('dv') * a_dv + w_dv))}
        return r, b

    def stats(self):
        """fp64 ctx, kmax, kzinv of the whole batch and the ctx bound"""
        parts = [self.ref_fwd(sl) for sl in self.slices()]
        cat = lambda d, key: torch.cat([x[d][key] for x in parts])
        return {k: cat(0, k) for k in ('ctx', 'kmax', 'kzinv')}, cat(1, 'ctx')

    # ---- launches -----------------------------------------------------------------------------------------------------
    def run_fwd(self):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, N, h, HID = self.B, self.N, self.heads, self.HID
        bufs = {'out': guarded(B * N * HID, self.dtype), 'ctx': guarded(B * h * 1024), 'kmax': guarded(B * HID),
                'kzinv': guarded(B * HID)}
        ws = torch.empty(call('pidm_linattn_workspace_floats', B, N, h), device=DEV)
        v = {k: t[1] for k, t in bufs.items()}
        call('pidm_linattn_fwd', self.qkv, v['out'], v['ctx'], v['kmax'], v['kzinv'], ws, B, N, h, CODE[self.dtype],
             stream())
        torch.cuda.synchronize()
        out = {'out': v['out'].view(B, N, HID), 'ctx': v['ctx'].view(B, h, 32, 32), 'kmax': v['kmax'].view(B, HID),
               'kzinv': v['kzinv'].view(B, HID)}
        return out, all(guards_intact(t[0]) for t in bufs.values())

    def run_bwd(self, ctx, kmax, kzinv):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, N, h, HID = self.B, self.N, self.heads, self.HID
        dbuf, dqkv = guarded(B * N * 3 * HID, self.dtype)
        cbuf, dctx = guarded(B * h * 1024)
        call('pidm_linattn_bwd', self.qkv, self.dout, ctx.float().contiguous(), kmax.float().contiguous(),
             kzinv.float().contiguous(), dqkv, dctx, B, N, h, CODE[self.dtype], stream())
        torch.cuda.synchronize()
        d = dqkv.view(B, N, 3, HID)
        return {'dq': d[:, :, 0], 'dk': d[:, :, 1], 'dv': d[:, :, 2]}, guards_intact(dbuf) and guards_intact(cbuf)


def _merge(acc, rs):
    for k, v in rs.items():
        acc[k] = max(acc.get(k, 0.0), v)
    return acc


LA_ACT = ('out', 'dq', 'dk', 'dv')


class AttnCase:
    def __init__(self, B, n, heads, dtype, edge=None):
        self.B, self.n, self.heads, self.dtype, self.HID = B, n, heads, dtype, heads * 32
        g = gen(('attn', B, n, heads, edge))
        qkv = _randn(g, B, n, 3, heads, 32)
        if edge == 'dominant key':
            qkv[:, :, 0, :, 0] = 8.0
            qkv[:, n // 2, 1, :, 0] = 16.0
        self.qkv = qkv.reshape(B, n, 3 * self.HID).to(dtype)
        self.dout = _randn(g, B, n, self.HID).to(dtype)
        self.kernel = attn_kernel(n, dtype)

    def ref(self, backward, mut=()):
        B, n, h, rnd = self.B, self.n, self.heads, RND[self.dtype]
        x = self.qkv.double().view(B, n, 3, h, 32).permute(2, 0, 3, 1, 4)
        q, k, v = x[0], x[1], x[2]
        S = SCALE * q @ k.transpose(-1, -2)
        e_S = math.sqrt(32) * U * SCALE * (q.abs() @ k.abs().transpose(-1, -2)) + U * S.abs()
        if 'padded keys scored 0' in mut:
            S = torch.cat((S, torch.zeros(B, h, n, 64 - n, dtype=S.dtype, device=DEV)), dim=-1)
            v = torch.cat((v, torch.zeros(B, h, 64 - n, 32, dtype=v.dtype, device=DEV)), dim=2)
        P = torch.softmax(S, dim=-1)
        z = (S.amax(-1, keepdim=True) - S).max().item()
        mid = BF if self.kernel == 'mid' else 0.0
        rho = 2 * e_S.amax(-1, keepdim=True) + U * (16 + 2 * z) + mid          # relative error of P, per query row
        flat = lambda t: t.permute(0, 2, 1, 3).reshape(B, n, self.HID)
        out = P @ v
        if not backward:
            return {'out': flat(out)}, {'out': flat(rnd * out.abs() + C_ATT * (rho + 8 * U) * (P @ v.abs()))}
        g = self.dout.double().view(B, n, h, 32).permute(0, 2, 1, 3)
        dP = g @ v.transpose(-1, -2)
        a_dP = g.abs() @ v.abs().transpose(-1, -2)
        dS = P * dP if 'dS without the row-dot term' in mut else P * (dP - (P * dP).sum(-1, keepdim=True))
        a_dS = P * (a_dP + (P * a_dP).sum(-1, keepdim=True))
        eps = rho + math.sqrt(32) * U + mid + 8 * U                         # + dS rounded to bf16 (mid) + the sums
        epsk = eps.amax(dim=2, keepdim=True)                                # key-side products sum over all queries
        dq, a_dq = SCALE * dS @ k, SCALE * (eps * a_dS) @ k.abs()
        dk, a_dk = SCALE * dS.transpose(-1, -2) @ q, SCALE * epsk * (a_dS.transpose(-1, -2) @ q.abs())
        dv, a_dv = P.transpose(-1, -2) @ g, epsk * (P.transpose(-1, -2) @ g.abs())
        r = {'dq': flat(dq), 'dk': flat(dk), 'dv': flat(dv)}
        b = {'dq': flat(rnd * dq.abs() + C_ATT * a_dq), 'dk': flat(rnd * dk.abs() + C_ATT * a_dk),
             'dv': flat(rnd * dv.abs() + C_ATT * a_dv)}
        return r, b

    def run(self, backward):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, n, h, HID = self.B, self.n, self.heads, self.HID
        if not backward:
            buf, out = guarded(B * n * HID, self.dtype)
            call('pidm_attn_fwd', self.qkv, out, B, n, h, CODE[self.dtype], stream())
            torch.cuda.synchronize()
            return {'out': out.view(B, n, HID)}, guards_intact(buf)
        buf, d = guarded(B * n * 3 * HID, self.dtype)
        call('pidm_attn_bwd', self.qkv, self.dout, d, B, n, h, CODE[self.dtype], stream())
        torch.cuda.synchronize()
        d = d.view(B, n, 3, HID)
        return {'dq': d[:, :, 0], 'dk': d[:, :, 1], 'dv': d[:, :, 2]}, guards_intact(buf)


class HeadCase:
    def __init__(self, B, HW, C, O, sig, dtype, edge=None):
        self.shape, self.sig, self.dtype = (B, HW, C, O), sig, dtype
        g = gen(('head', B, HW, C, O, sig, edge))
        self.x = _randn(g, B * HW, C).to(dtype)
        self.w = _randn(g, O, C, scale=1 / math.sqrt(C))
        self.bias = _randn(g, O, scale=0.1)
        if edge == 'saturated sigmoid':
            self.w[-1] *= 0.1
            self.bias[-1] = 25.0
        self.dy = _randn(g, B, O, HW)
        self.pre = {'dW': _randn(g, O * C), 'db': _randn(g, O)}

    def ref_fwd(self):
        B, HW, C, O = self.shape
        x, w = self.x.double(), self.w.double()
        z = x @ w.T + self.bias.double()
        e_z = C_HEAD * math.sqrt(C) * U * (x.abs() @ w.abs().T + self.bias.double().abs())
        y, b = z.clone(), e_z.clone()
        if self.sig:
            s = torch.sigmoid(z[:, -1])
            y[:, -1] = s
            b[:, -1] = s * (1 - s) * (e_z[:, -1] + U * (8 + 2 * z[:, -1].abs())) + 3 * U * s
        nchw = lambda t: t.view(B, HW, O).permute(0, 2, 1)
        return {'y': nchw(y)}, {'y': nchw(b)}

    def ref_bwd(self, y, mut=()):
        """fp64 dx, dW, db from the forward output y (the kernel's, as the backward receives it)"""
        B, HW, C, O = self.shape
        M, rnd = B * HW, RND[self.dtype]
        x, w = self.x.double(), self.w.double()
        dz = self.dy.double().permute(0, 2, 1).reshape(M, O).clone()
        if self.sig and 'dz without sigma prime' not in mut:
            s = y.double().permute(0, 2, 1).reshape(M, O)[:, -1]
            dz[:, -1] = dz[:, -1] * s * (1 - s)
        dx = dz @ w
        a_dx = dz.abs() @ w.abs()
        xs, dzs = x, dz
        if 'ragged last warp missing from dW' in mut:
            xs, dzs = x[:M - M % 32], dz[:M - M % 32]
        dW = self.pre['dW'].double() + (dzs.T @ xs).reshape(-1)
        a_dW = (dz.abs().T @ x.abs()).reshape(-1)
        db = (0 if 'db overwritten' in mut else self.pre['db'].double()) + dz.sum(0)
        a_db = dz.abs().sum(0)
        acc = C_HEAD * math.sqrt(M) * U
        r = {'dx': dx, 'dW': dW, 'db': db}
        b = {'dx': rnd * dx.abs() + C_HEAD * (O + 3) * U * a_dx,
             'dW': acc * (self.pre['dW'].double().abs() + a_dW) + C_HEAD * 3 * U * a_dW,
             'db': acc * (self.pre['db'].double().abs() + a_db) + C_HEAD * 3 * U * a_db}
        return r, b

    def run_fwd(self):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, HW, C, O = self.shape
        buf, y = guarded(B * O * HW)
        call('pidm_head_fwd', self.x, self.w, self.bias, y, B, HW, C, O, self.sig, CODE[self.dtype], stream())
        torch.cuda.synchronize()
        return {'y': y.view(B, O, HW)}, guards_intact(buf)

    def run_bwd(self, y):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, HW, C, O = self.shape
        bufs = {'dx': guarded(B * HW * C, self.dtype), 'dW': guarded(O * C), 'db': guarded(O)}
        bufs['dW'][1].copy_(self.pre['dW'])
        bufs['db'][1].copy_(self.pre['db'])
        v = {k: t[1] for k, t in bufs.items()}
        call('pidm_head_bwd', self.x, self.w, y.contiguous(), self.dy, v['dx'], v['dW'], v['db'], B, HW, C, O, self.sig,
             CODE[self.dtype], stream())
        torch.cuda.synchronize()
        v['dx'] = v['dx'].view(B * HW, C)
        return v, all(guards_intact(t[0]) for t in bufs.values())


# ----------------------------------------------------------------------------------------------------------------------
# replay
# ----------------------------------------------------------------------------------------------------------------------
def replay_la_fwd(c, where):
    out, ok = c.run_fwd()
    assert ok, f'{where}: a store landed outside out, ctx, kmax or kzinv'
    rs = {}
    for sl in c.slices():
        _merge(rs, ratios(out, *c.ref_fwd(sl), sl))
    note_all(TAG, f'linattn_fwd {FWD_PATHS[c.plan["fwd"]]} {NAME[c.dtype]}', rs)
    assert_ok(rs, f'{where} (plan {c.plan})')
    return out


def replay_la_bwd(c, where, fwd_out=None):
    st, e_ctx = c.stats()
    path = f'linattn_bwd {BWD_PATHS[c.plan["bwd"]]} {NAME[c.dtype]}'
    given = {k: v.float() for k, v in st.items()}
    out, ok = c.run_bwd(given['ctx'], given['kmax'], given['kzinv'])
    assert ok, f'{where}: a store landed outside dqkv or dctx'
    rs = {}
    for sl in c.slices():
        _merge(rs, ratios(out, *c.ref_bwd(sl, given['ctx'][sl], given['kmax'][sl], given['kzinv'][sl]), sl))
    note_all(TAG, path + ' given statistics', rs)
    assert_ok(rs, f'{where} given the statistics (plan {c.plan})')
    fo = fwd_out if fwd_out is not None else replay_la_fwd(c, where)
    out, ok = c.run_bwd(fo['ctx'], fo['kmax'], fo['kzinv'])
    assert ok, f'{where}: a store landed outside dqkv or dctx'
    rs = {}
    for sl in c.slices():
        r, b = c.ref_bwd(sl, st['ctx'][sl], st['kmax'][sl], st['kzinv'][sl], e_ctx=e_ctx[sl], eps_kz=c.eps32 + U)
        _merge(rs, ratios(out, r, b, sl))
    hand = f'{FWD_PATHS[c.plan["fwd"]]}->{BWD_PATHS[c.plan["bwd"]]}'
    note_all(TAG, f'{path} end to end ({hand})', rs)
    assert_ok(rs, f'{where} end to end, {hand} (plan {c.plan})')
    return out


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', LA_FWD_ROWS, ids=_id)
def test_linattn_fwd_replay(k, dtype):
    replay_la_fwd(LaCase(*k, dtype), f'linattn_fwd {k} {NAME[dtype]}')


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', LA_BWD_ROWS, ids=_id)
def test_linattn_bwd_replay(k, dtype):
    replay_la_bwd(LaCase(*k, dtype), f'linattn_bwd {k} {NAME[dtype]}')


def replay_attn(c, backward, where):
    out, ok = c.run(backward)
    assert ok, f'{where}: a store landed outside the output (padded query rows must not be written)'
    rs = ratios(out, *c.ref(backward))
    note_all(TAG, f'attn_{"bwd" if backward else "fwd"} {c.kernel} {NAME[c.dtype]}', rs)
    assert_ok(rs, where)
    return out


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', ATTN_FWD_ROWS, ids=_id)
def test_attn_fwd_replay(k, dtype):
    replay_attn(AttnCase(*k, dtype), False, f'attn_fwd {k} {NAME[dtype]}')


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', ATTN_BWD_ROWS, ids=_id)
def test_attn_bwd_replay(k, dtype):
    replay_attn(AttnCase(*k, dtype), True, f'attn_bwd {k} {NAME[dtype]}')


def replay_head(c, backward, where):
    out, ok = c.run_fwd()
    assert ok, f'{where}: a store landed outside y'
    rs = ratios(out, *c.ref_fwd())
    note_all(TAG, f'head_fwd {NAME[c.dtype]}', rs)
    assert_ok(rs, where)
    if not backward:
        return out, None
    dout, ok = c.run_bwd(out['y'])
    assert ok, f'{where}: a store landed outside dx, dW or db'
    rs = ratios(dout, *c.ref_bwd(out['y']))
    note_all(TAG, f'head_bwd {plan_head(*c.shape, True)["kernel"]} {NAME[c.dtype]}', rs)
    assert_ok(rs, f'{where} (plan {plan_head(*c.shape, True)})')
    return out, dout


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', HEAD_FWD_ROWS, ids=_id)
def test_head_fwd_replay(k, dtype):
    replay_head(HeadCase(*k, dtype), False, f'head_fwd {k} {NAME[dtype]}')


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', HEAD_BWD_ROWS, ids=_id)
def test_head_bwd_replay(k, dtype):
    replay_head(HeadCase(*k, dtype), True, f'head_bwd {k} {NAME[dtype]}')


# ----------------------------------------------------------------------------------------------------------------------
# edges
# ----------------------------------------------------------------------------------------------------------------------
EDGE_LA_SHAPES = [(2, 4096, 8), (3, 1056, 8), (2, 64, 8)]       # bf16: mma | simt | one CTA -> mma;  fp32: simt


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', EDGE_LA_SHAPES, ids=_id)
def test_linattn_spike_in_the_last_statistics_chunk(k, dtype):
    """k = +40 at the last pixel only: every other statistics chunk's partial sum is rescaled by exp(-40...) when the
    chunks are merged, and ctx is that pixel's v / N"""
    c = LaCase(*k, dtype, edge='spike in the last statistics chunk')
    assert c.plan['fwd'] == 0 or (k[1] - 1) // c.plan['stat_rows'] == c.plan['stat_chunks'] - 1
    out = replay_la_fwd(c, f'spike {k} {NAME[dtype]}')
    assert (out['kmax'] == 40.0).all()
    replay_la_bwd(c, f'spike {k} {NAME[dtype]}', out)


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', EDGE_LA_SHAPES, ids=_id)
def test_linattn_saturated_q_rows(k, dtype):
    """q rows with one channel 30 above the others: the row softmax is one-hot to fp32 precision"""
    c = LaCase(*k, dtype, edge='saturated q rows')
    replay_la_bwd(c, f'saturated q {k} {NAME[dtype]}', replay_la_fwd(c, f'saturated q {k} {NAME[dtype]}'))


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', EDGE_LA_SHAPES, ids=_id)
def test_linattn_constant_k_column(k, dtype):
    """a constant k column: exp(0) = 1 at every pixel, Z = N and kzinv = 1 / N exactly"""
    c = LaCase(*k, dtype, edge='constant k column')
    out = replay_la_fwd(c, f'constant k {k} {NAME[dtype]}')
    col0 = out['kzinv'].view(k[0], k[2], 32)[:, :, 0].double()
    assert (out['kmax'].view(k[0], k[2], 32)[:, :, 0] == 0.75).all()
    assert ((col0 * k[1] - 1).abs() <= 2 * U).all(), col0          # Z = N exactly; one rounding of 1 / Z
    replay_la_bwd(c, f'constant k {k} {NAME[dtype]}', out)


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('n', [1, 7, 33, 63, 64])
def test_mid_attention_dominant_key_and_padding(n, dtype):
    """one key (n // 2) scores about 22 above the rest for every query: P is one-hot; with n < 64 the padded keys must
    get no weight and the padded query rows must not be written"""
    c = AttnCase(3, n, 8, dtype, edge='dominant key')
    out = replay_attn(c, False, f'dominant key n={n} {NAME[dtype]}')
    replay_attn(c, True, f'dominant key n={n} {NAME[dtype]}')
    assert torch.isfinite(out['out']).all()


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_head_saturated_sigmoid(dtype):
    """z > 20 on the sigmoid channel: y = 1 exactly, sigma' = 0, so that channel adds nothing to dx, dW, db"""
    c = HeadCase(2, 300, 32, 3, 1, dtype, edge='saturated sigmoid')
    out, dout = replay_head(c, True, f'saturated sigmoid {NAME[dtype]}')
    assert (out['y'][:, -1] == 1.0).all()
    assert torch.isfinite(dout['dx']).all()
    assert torch.equal(dout['db'][-1], c.pre['db'][-1]) and torch.equal(dout['dW'][-32:], c.pre['dW'][-32:])


# ----------------------------------------------------------------------------------------------------------------------
# the predicates reject subtly wrong outputs (edits of the fp64 reference; no faulty code runs on the GPU)
# ----------------------------------------------------------------------------------------------------------------------
def _la_mutant(k, dtype, mutation, output, backward=False):
    c = LaCase(*k, dtype)
    sl = slice(0, c.chunk)
    if backward:
        st, _ = c.stats()
        args = (st['ctx'][sl].float(), st['kmax'][sl].float(), st['kzinv'][sl].float())
        r, b = c.ref_bwd(sl, *args)
        m, _ = c.ref_bwd(sl, *args, mut=(mutation,))
    else:
        r, b = c.ref_fwd(sl)
        m, _ = c.ref_fwd(sl, mut=(mutation,))
    assert max(ratios(rounded(r, dtype, LA_ACT), r, b).values()) <= 1.0
    return ratios(rounded(m, dtype, LA_ACT), r, b)[output]


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_mutant_k_softmax_per_statistics_chunk(dtype):
    assert _la_mutant((2, 1024, 8), dtype, 'k-softmax per statistics chunk', 'ctx') > 1.0
    assert _la_mutant((2, 1024, 8), dtype, 'k-softmax per statistics chunk', 'out') > 1.0


def test_mutant_last_mma_chunk_from_its_neighbour():
    p = plan_la(5, 4096, 8, torch.bfloat16)
    assert p['fwd'] == 1 and 4096 % p['mma_px'] != 0
    assert _la_mutant((5, 4096, 8), torch.bfloat16, 'last mma chunk from its neighbour', 'out') > 1.0


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_mutant_linattn_terms(dtype):
    assert _la_mutant((2, 256, 8), dtype, 'v not divided by N', 'ctx') > 1.0
    assert _la_mutant((2, 256, 8), dtype, 'ctx of head 0 from head 1', 'out') > 1.0
    assert _la_mutant((2, 256, 8), dtype, 'dk without the dctx ctx term', 'dk', backward=True) > 1.0


def _attn_mutant(k, dtype, mutation, output, backward):
    c = AttnCase(*k, dtype)
    r, b = c.ref(backward)
    assert max(ratios(rounded(r, dtype, LA_ACT), r, b).values()) <= 1.0
    m, _ = c.ref(backward, mut=(mutation,))
    return ratios(rounded(m, dtype, LA_ACT), r, b)[output]


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_mutant_mid_attention(dtype):
    for n in (7, 33, 63):
        assert _attn_mutant((2, n, 8), dtype, 'padded keys scored 0', 'out', False) > 1.0
    for n in (33, 64):
        assert _attn_mutant((2, n, 8), dtype, 'dS without the row-dot term', 'dq', True) > 1.0
        assert _attn_mutant((2, n, 8), dtype, 'dS without the row-dot term', 'dk', True) > 1.0


def _head_mutant(k, dtype, mutation, output):
    c = HeadCase(*k, dtype)
    y = rounded(c.ref_fwd()[0], dtype, ())['y']
    r, b = c.ref_bwd(y)
    assert max(ratios(rounded(r, dtype, ('dx',)), r, b).values()) <= 1.0
    m, _ = c.ref_bwd(y, mut=(mutation,))
    return ratios(rounded(m, dtype, ('dx',)), r, b)[output]


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_mutant_head(dtype):
    for k in ((5, 123, 32, 3, 1), (3, 401, 24, 2, 1)):
        assert _head_mutant(k, dtype, 'dz without sigma prime', 'dx') > 1.0
        assert _head_mutant(k, dtype, 'dz without sigma prime', 'dW') > 1.0
    for k in ((3, 401, 24, 2, 1), (1, 261, 512, 1, 1)):
        assert plan_head(*k[:4], True)['kernel'] == 'general' and plan_head(*k[:4], True)['ragged_warp']
        assert _head_mutant(k, dtype, 'ragged last warp missing from dW', 'dW') > 1.0
    assert _head_mutant((2, 300, 16, 2, 1), dtype, 'db overwritten', 'db') > 1.0


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
def la_coverage():
    fwd = [(k, dt, plan_la(*k, dt)) for k in LA_FWD_ROWS + EDGE_LA_SHAPES for dt in DTYPES]
    bwd = [(k, dt, plan_la(*k, dt)) for k in LA_BWD_ROWS + EDGE_LA_SHAPES for dt in DTYPES]
    mma_fwd = [(k, p) for k, dt, p in fwd if p['fwd'] == 1]
    simt = [(k, p) for k, dt, p in fwd + bwd if p['fwd'] == 2 or p['bwd'] == 1]
    return {
        'fwd paths': {(p['fwd'], NAME[dt]) for _, dt, p in fwd},
        'bwd paths': {(p['bwd'], NAME[dt]) for _, dt, p in bwd},
        'hand-offs (bf16)': {(p['fwd'], p['bwd']) for _, dt, p in bwd if dt == torch.bfloat16},
        'mma one chunk per sample': any(p['mma_chunks'] == 1 and k[0] == 256 for k, p in mma_fwd),
        'mma clamped to 64 pixels': any(p['mma_px'] == 64 and -(-k[1] // (sms() * 2 // k[0])) < 64
                                        for k, p in mma_fwd),
        'mma ragged last chunk': any(k[1] % p['mma_px'] for k, p in mma_fwd
                                     if any(kb == k and pb['bwd'] == 0 for kb, _, pb in bwd)),
        'statistics chunks': {min(p['stat_chunks'], 2) for _, _, p in fwd if p['fwd']}
                             | ({32} if any(p['stat_chunks'] == 32 for _, _, p in fwd if p['fwd']) else set()),
        'simt ctx chunk ragged in its tile': {k[1] for k, p in simt
                                              if (k[1] - (p['ctx_chunks'] - 1) * p['ctx_rows']) % 64},
        'heads': {k[2] for k, _, _ in fwd + bwd},
    }


def head_coverage():
    fwd = [(k, plan_head(*k[:4], False)) for k in HEAD_FWD_ROWS]
    bwd = [(k, plan_head(*k[:4], True)) for k in HEAD_BWD_ROWS]
    return {
        'octet lanes per pixel': {p['lpp'] for _, p in bwd if p['kernel'] == 'octet'},
        'general C, ragged last warp': {k[2] for k, p in bwd if p['kernel'] == 'general' and p['ragged_warp']},
        'O': {k[3] for k in HEAD_FWD_ROWS} & {k[3] for k in HEAD_BWD_ROWS},
        'sigmoid': {k[4] for k in HEAD_FWD_ROWS} & {k[4] for k in HEAD_BWD_ROWS},
        'capped grid, several passes': {p['kernel'] for _, p in fwd + bwd if p['passes'] > 1},
    }


def test_plan_coverage():
    assert sms() == 132, 'the synthetic rows are chosen for the 132-SM H100'
    cv = la_coverage()
    print(f'[attention census] linear attention coverage {cv}')
    assert cv['fwd paths'] == {(0, 'bf16'), (1, 'bf16'), (2, 'bf16'), (2, 'fp32')}, cv
    assert cv['bwd paths'] == {(0, 'bf16'), (1, 'bf16'), (1, 'fp32')}, cv
    assert cv['hand-offs (bf16)'] >= {(0, 0), (0, 1), (1, 0), (2, 1)}, cv
    assert cv['mma one chunk per sample'] and cv['mma clamped to 64 pixels'] and cv['mma ragged last chunk'], cv
    assert cv['statistics chunks'] == {1, 2, 32}, cv
    assert {96, 1056} <= cv['simt ctx chunk ragged in its tile'], cv
    assert cv['heads'] - {8}, cv
    modes = {(attn_kernel(k[1], dt), NAME[dt]) for k in ATTN_FWD_ROWS + ATTN_BWD_ROWS for dt in DTYPES}
    assert modes == {('mid', 'bf16'), ('core', 'bf16'), ('core', 'fp32')}, modes
    hv = head_coverage()
    print(f'[attention census] head coverage {hv}')
    assert hv['octet lanes per pixel'] == {1, 2, 4, 8, 16, 32}, hv
    assert {24, 48, 512} <= hv['general C, ragged last warp'], hv
    assert hv['O'] == {1, 2, 3, 4} and hv['sigmoid'] == {0, 1}, hv
    assert hv['capped grid, several passes'] == {'fwd', 'octet', 'general'}, hv


def test_rejected_shapes_are_refused_before_any_launch():
    """shapes the kernels do not support return an error and leave every output untouched"""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    out = torch.zeros(8, dtype=torch.int32)
    assert call('pidm_linattn_plan', 2, 256, 2, 1, out.data_ptr()) == 0 and out[1].item() == -1
    for B, N, heads in ((2, 48, 8), (2, 256, 33)):
        assert call('pidm_linattn_plan', B, N, heads, 1, out.data_ptr()) != 0, (B, N, heads)
    bf = torch.bfloat16
    qkv = torch.zeros(2 * 256 * 192, dtype=bf, device=DEV)
    dbuf, d = guarded(2 * 256 * 192, bf)
    cbuf, dctx = guarded(2 * 2 * 1024)
    st = torch.zeros(2 * 2 * 1024, device=DEV)
    with pytest.raises(RuntimeError):
        call('pidm_linattn_bwd', qkv, qkv[:2 * 256 * 64], st, st, st, d, dctx, 2, 256, 2, 1, stream())
    qkv = torch.zeros(2 * 65 * 768, dtype=bf, device=DEV)
    obuf, o = guarded(2 * 65 * 768, bf)
    with pytest.raises(RuntimeError):
        call('pidm_attn_fwd', qkv, o[:2 * 65 * 256], 2, 65, 8, 1, stream())
    with pytest.raises(RuntimeError):
        call('pidm_attn_bwd', qkv, qkv[:2 * 65 * 256], o, 2, 65, 8, 1, stream())
    x = torch.zeros(2 * 16 * 64, dtype=bf, device=DEV)
    w = torch.zeros(5 * 64, device=DEV)
    ybuf, y = guarded(2 * 5 * 16)
    for C, O in ((64, 5), (12, 2)):
        with pytest.raises(RuntimeError):
            call('pidm_head_fwd', x, w, w[:O], y, 2, 16, C, O, 0, 1, stream())
        with pytest.raises(RuntimeError):
            call('pidm_head_bwd', x, w, y, y, x, w, w[:O], 2, 16, C, O, 0, 1, stream())
    torch.cuda.synchronize()
    for buf in (dbuf, cbuf, obuf, ybuf):
        assert torch.isnan(buf.float()).all()
    assert not x.any() and not w.any()

