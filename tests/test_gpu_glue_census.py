"""Every time-conditioning, optimizer, weight-packing and element-wise glue launch of the benchmarked steps, replayed
element by element against an fp64 reference.

These entry points run on every training or sampling step, but the per-op tests compared them by a norm ratio at a few
small shapes: a time embedding at B = 5, t <= 99; block MLPs whose backward only ever saw one 32-sample chunk; an Adam
step with a host step count, no gradient scale and no zeroing; a weight packer whose output only the end-to-end
tolerances looked at.  Here, in the four parts of the other census files:

  1. census: one eager step of every workload bench.py times is recorded at the C ABI, and the distinct keys of the
     glue entry points must equal the tables below (`python tests/census.py --print-table` regenerates them).  Keys
     are the integer and flag arguments and the geometry decoded from the device tables (packing._PACK_DT, _PAIR_DT,
     _MLP_DT), never pointers;
  2. replay: every table row and synthetic row runs through the C ABI on seeded operands, outputs between NaN guards,
     accumulating outputs prefilled, against fp64 references of the semantics in oracle/pidm_oracle.py:
        packing, concat, split, nchw_to_nhwc, scale    bitwise (packing: the torch permutation of fp32 weights that are
                                                       not bf16-exact, rounded to nearest even; gaps between packed
                                                       matrices untouched)
        qsample, axpby                                 |y - r| <= C_EW u A           u = 2^-24, A = |terms|
        time MLP, block MLPs and their gradients       |y - r| <= C_GEMV sqrt(K) u A + propagated input error
        sinusoid                                       |y - r| <= C_SIN u (1 + |t f|)   (what fp32 PyTorch achieves)
        Adam / EMA                                     |y - r| <= C_ADAM u A         A = the chain on absolute values
        sumsq                                          |y - r| <= (C_SUM + depth) u A
  3. mutants: the same predicates reject the fp64 reference edited the way a subtle kernel bug would change it;
  4. plan coverage: the launch arithmetic, restated below, shows that the rows reach every grid and chunking case.
Two tests run without a GPU: the fp64 references against the oracle (test_references_follow_the_oracle), and the
reciprocal division of pack_pair_kernel, exhaustively (test_pack_pair_reciprocal_division).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from census import assert_census_in_tables, assert_tables_in_census, census
from checks import DTYPE, U, call_sync, check, gen, guarded, guards_intact, note, sms
from oracle import pidm_oracle as O

gpu = pytest.mark.gpu                            # per test: the two CPU tests run without a GPU
DEV = 'cuda'
TAG = 'glue census'

# Bound constants, each the smallest power of two that passes on an H100; the worst |err| / bound per output is
# recorded in DESIGN.md section 2.
C_SIN = 8          # fp32 PyTorch's own SinusoidalPosEmb reaches 7.4 u (1 + |t f|) at dim = 1024, t < 1000
C_GEMV = 2         # fp32 dot products: c sqrt(K) u A
C_ACT = 16         # activations: u (C_ACT + 2|z|) relative for the fast exponential and division of --use_fast_math
C_EW = 4           # element-wise fp32 chains of at most three terms
C_ADAM = 16        # roundings along the clip / Adam / EMA chain
C_SUM = 4          # sumsq: roundings beside the accumulation depth
GELU_LIP, SILU_LIP = 1.13, 1.10        # max |gelu'|, max |silu'|

# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`)
# ----------------------------------------------------------------------------------------------------------------------
# time_fwd: B, dim, td;  time_bwd: B, dim, td, parts
# mlp_fwd: B, td, max_rows, rows of every entry;  mlp_bwd: B, td, max_rows, rows of every entry, parts
# sumsq: n;  adam: n, device step, grad_scale, max_norm, ema_first_step, zero_grad
# pack: dtype, N, C, Cpad, taps, flip, s_n, s_c  (one row per entry)
# pair: dtype, Cout, Cin, taps, flip, ci_inner (conv layout), has dgrad  (one row per entry)
# pair_launch: dtype, tile_base, n_tiles, max_taps
# qsample / axpby: B, per_sample;  scale: n;  concat / split: rows, Ca, Cb, dtype;  nchw: B, C, HW, Cpad, dtype
TIME_FWD_TABLE = [
    (16, 32, 128),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 32, 128),  # darcy_train_b32
    (32, 128, 512),  # mech_train_b32
    (64, 32, 128),  # darcy_sample_b64
    (256, 32, 128),  # darcy_sample_b256
]
TIME_BWD_TABLE = [
    (32, 32, 128, 1),  # darcy_train_b32
    (32, 32, 128, 2),  # darcy_train_b32
    (32, 128, 512, 1),  # mech_train_b32
    (32, 128, 512, 2),  # mech_train_b32
]
MLP_FWD_TABLE = [
    (16, 128, 512, (64, 64, 128, 128, 256, 256, 512, 512, 512, 512, 256, 256, 128, 128, 64, 64, 64, 64)),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 128, 512, (64, 64, 128, 128, 256, 256, 512, 512, 512, 512, 256, 256, 128, 128, 64, 64, 64, 64)),  # darcy_train_b32
    (32, 512, 2048, (256, 256, 512, 512, 1024, 1024, 2048, 2048, 2048, 2048, 1024, 1024, 512, 512, 256, 256, 256, 256)),  # mech_train_b32
    (64, 128, 512, (64, 64, 128, 128, 256, 256, 512, 512, 512, 512, 256, 256, 128, 128, 64, 64, 64, 64)),  # darcy_sample_b64
    (256, 128, 512, (64, 64, 128, 128, 256, 256, 512, 512, 512, 512, 256, 256, 128, 128, 64, 64, 64, 64)),  # darcy_sample_b256
]
MLP_BWD_TABLE = [
    (32, 128, 512, (64, 64, 128, 128, 256, 256, 512, 512, 512, 512, 256, 256, 128, 128, 64, 64, 64, 64), 1),  # darcy_train_b32
    (32, 128, 512, (64, 64, 128, 128, 256, 256, 512, 512, 512, 512, 256, 256, 128, 128, 64, 64, 64, 64), 2),  # darcy_train_b32
    (32, 512, 2048, (256, 256, 512, 512, 1024, 1024, 2048, 2048, 2048, 2048, 1024, 1024, 512, 512, 256, 256, 256, 256), 1),  # mech_train_b32
    (32, 512, 2048, (256, 256, 512, 512, 1024, 1024, 2048, 2048, 2048, 2048, 1024, 1024, 512, 512, 256, 256, 256, 256), 2),  # mech_train_b32
]
SUMSQ_TABLE = [
    (10388480,),  # darcy_train_b32
    (136207168,),  # mech_train_b32
]
ADAM_TABLE = [
    (10388480, 1, 1.0, 1.0, 1, 1),  # darcy_train_b32
    (136207168, 1, 1.0, 1.0, 1, 1),  # mech_train_b32
]
PACK_TABLE = [
    (1, 32, 2, 32, 49, 0, 98, 49),  # darcy_train_b32
    (1, 128, 10, 32, 49, 0, 490, 49),  # mech_train_b32
]
PAIR_TABLE = [
    (1, 32, 32, 9, 1, 1, 1),  # darcy_train_b32
    (1, 32, 32, 16, 0, 0, 1),  # darcy_train_b32
    (1, 32, 32, 16, 0, 1, 1),  # darcy_train_b32
    (1, 32, 64, 1, 1, 1, 1),  # darcy_train_b32
    (1, 32, 64, 9, 1, 1, 1),  # darcy_train_b32
    (1, 32, 128, 1, 1, 1, 1),  # darcy_train_b32
    (1, 32, 128, 9, 1, 1, 1),  # darcy_train_b32
    (1, 32, 256, 1, 1, 1, 1),  # darcy_train_b32
    (1, 64, 32, 1, 1, 1, 1),  # darcy_train_b32
    (1, 64, 32, 9, 1, 1, 1),  # darcy_train_b32
    (1, 64, 64, 9, 1, 1, 1),  # darcy_train_b32
    (1, 64, 64, 16, 0, 0, 1),  # darcy_train_b32
    (1, 64, 64, 16, 0, 1, 1),  # darcy_train_b32
    (1, 64, 256, 1, 1, 1, 1),  # darcy_train_b32
    (1, 64, 256, 9, 1, 1, 1),  # darcy_train_b32
    (1, 128, 64, 1, 1, 1, 1),  # darcy_train_b32
    (1, 128, 64, 9, 1, 1, 1),  # darcy_train_b32
    (1, 128, 128, 9, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 128, 128, 16, 0, 0, 1),  # darcy_train_b32 mech_train_b32
    (1, 128, 128, 16, 0, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 128, 256, 1, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 128, 256, 9, 1, 1, 1),  # mech_train_b32
    (1, 128, 512, 1, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 128, 512, 9, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 256, 128, 1, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 256, 128, 9, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 256, 256, 1, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 256, 256, 9, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 256, 256, 16, 0, 0, 1),  # mech_train_b32
    (1, 256, 256, 16, 0, 1, 1),  # mech_train_b32
    (1, 256, 1024, 1, 1, 1, 1),  # mech_train_b32
    (1, 256, 1024, 9, 1, 1, 1),  # mech_train_b32
    (1, 512, 256, 1, 1, 1, 1),  # mech_train_b32
    (1, 512, 256, 9, 1, 1, 1),  # mech_train_b32
    (1, 512, 512, 9, 1, 1, 1),  # mech_train_b32
    (1, 512, 512, 16, 0, 0, 1),  # mech_train_b32
    (1, 512, 512, 16, 0, 1, 1),  # mech_train_b32
    (1, 512, 2048, 1, 1, 1, 1),  # mech_train_b32
    (1, 512, 2048, 9, 1, 1, 1),  # mech_train_b32
    (1, 768, 32, 1, 1, 1, 1),  # darcy_train_b32
    (1, 768, 64, 1, 1, 1, 1),  # darcy_train_b32
    (1, 768, 128, 1, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 768, 256, 1, 1, 1, 1),  # darcy_train_b32 mech_train_b32
    (1, 768, 512, 1, 1, 1, 1),  # mech_train_b32
    (1, 768, 1024, 1, 1, 1, 1),  # mech_train_b32
    (1, 1024, 256, 1, 1, 1, 1),  # mech_train_b32
    (1, 1024, 512, 1, 1, 1, 1),  # mech_train_b32
    (1, 1024, 512, 9, 1, 1, 1),  # mech_train_b32
    (1, 1024, 1024, 9, 1, 1, 1),  # mech_train_b32
]
PAIR_LAUNCH_TABLE = [
    (1, 0, 36, 16),  # darcy_train_b32
    (1, 0, 192, 16),  # mech_train_b32
    (1, 36, 1840, 16),  # darcy_train_b32
    (1, 192, 17920, 16),  # mech_train_b32
]
QSAMPLE_TABLE = [
    (32, 8192),  # darcy_train_b32
    (32, 12675),  # mech_train_b32
]
AXPBY_TABLE = [
    (16, 8192),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (64, 8192),  # darcy_sample_b64
    (256, 8192),  # darcy_sample_b256
]
SCALE_TABLE = [
    (32,),  # mech_train_b32
    (131072,),  # mech_train_b32
    (262144,),  # darcy_train_b32
    (270400,),  # mech_train_b32
]
CONCAT_TABLE = [
    (1024, 256, 256, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (2048, 256, 256, 1),  # darcy_train_b32
    (2048, 1024, 1024, 1),  # mech_train_b32
    (4096, 128, 128, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (4096, 256, 256, 1),  # darcy_sample_b64
    (8192, 128, 128, 1),  # darcy_train_b32
    (8192, 512, 512, 1),  # mech_train_b32
    (16384, 64, 64, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16384, 128, 128, 1),  # darcy_sample_b64
    (16384, 256, 256, 1),  # darcy_sample_b256
    (32768, 64, 64, 1),  # darcy_train_b32
    (32768, 256, 256, 1),  # mech_train_b32
    (65536, 32, 32, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (65536, 64, 64, 1),  # darcy_sample_b64
    (65536, 128, 128, 1),  # darcy_sample_b256
    (131072, 32, 32, 1),  # darcy_train_b32
    (131072, 128, 128, 1),  # mech_train_b32
    (262144, 32, 32, 1),  # darcy_sample_b64
    (262144, 64, 64, 1),  # darcy_sample_b256
    (1048576, 32, 32, 1),  # darcy_sample_b256
]
SPLIT_TABLE = [
    (2048, 256, 256, 1),  # darcy_train_b32
    (2048, 1024, 1024, 1),  # mech_train_b32
    (8192, 128, 128, 1),  # darcy_train_b32
    (8192, 512, 512, 1),  # mech_train_b32
    (32768, 64, 64, 1),  # darcy_train_b32
    (32768, 256, 256, 1),  # mech_train_b32
    (131072, 32, 32, 1),  # darcy_train_b32
    (131072, 128, 128, 1),  # mech_train_b32
]
NCHW_TABLE = [
    (16, 2, 4096, 32, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 2, 4096, 32, 1),  # darcy_train_b32
    (32, 10, 4096, 32, 1),  # mech_train_b32
    (64, 2, 4096, 32, 1),  # darcy_sample_b64
    (256, 2, 4096, 32, 1),  # darcy_sample_b256
]
TABLES = {'time_fwd': TIME_FWD_TABLE, 'time_bwd': TIME_BWD_TABLE, 'mlp_fwd': MLP_FWD_TABLE, 'mlp_bwd': MLP_BWD_TABLE,
          'sumsq': SUMSQ_TABLE, 'adam': ADAM_TABLE, 'pack': PACK_TABLE, 'pair': PAIR_TABLE,
          'pair_launch': PAIR_LAUNCH_TABLE, 'qsample': QSAMPLE_TABLE, 'axpby': AXPBY_TABLE, 'scale': SCALE_TABLE,
          'concat': CONCAT_TABLE, 'split': SPLIT_TABLE, 'nchw': NCHW_TABLE}
# the entry points this file replays per element
GLUE_NAMES = {'pidm_time_embed_fwd', 'pidm_time_embed_bwd', 'pidm_block_mlps_fwd', 'pidm_block_mlps_bwd', 'pidm_sumsq',
              'pidm_adam_ema_step', 'pidm_pack_weights', 'pidm_pack_weights_pairs', 'pidm_qsample',
              'pidm_axpby_per_sample', 'pidm_scale', 'pidm_concat_channels', 'pidm_split_channels', 'pidm_nchw_to_nhwc'}


# ----------------------------------------------------------------------------------------------------------------------
# census
# ----------------------------------------------------------------------------------------------------------------------
@gpu
def test_census_is_covered_by_the_table():
    assert_census_in_tables(TABLES)


@gpu
def test_every_table_row_is_produced_by_the_census():
    assert_tables_in_census(TABLES)


@gpu
def test_every_glue_entry_point_is_recorded():
    _, names = census()
    assert GLUE_NAMES <= names, f'entry points no benchmarked step calls any more: {sorted(GLUE_NAMES - names)}'


# ----------------------------------------------------------------------------------------------------------------------
# launch arithmetic (restated from the launches)
# ----------------------------------------------------------------------------------------------------------------------
MLP_BCHUNK, MLP_ROWS, MLP_DG_ROWS = 32, 16, 32          # linear.cu
SUMSQ_CAP = 148 * 8                                     # optim.cu pidm_sumsq (and its workspace: 1 + SUMSQ_CAP floats)


def sumsq_grid(n):                   # pidm_sumsq: 256 threads, ceil(n/4 / 256) CTAs, capped at 148 * 8
    return min(max(-(-(n // 4) // 256), 1), SUMSQ_CAP)


def adam_grid(n, n_sms):             # pidm_adam_ema_step: 256 threads, ceil(n/4 / 256) CTAs, capped at 8 per SM
    return min(max(-(-(n // 4) // 256), 1), 8 * n_sms)


def grid_for(n, block, n_sms):       # elementwise.cu grid_for: 16 CTAs per SM
    return min(max(-(-n // block), 1), 16 * n_sms)


def ew_passes(B, per_sample, n_sms):  # qsample / axpby: float4 path when per_sample % 4 == 0, else scalar
    n = B * per_sample // 4 if per_sample % 4 == 0 else B * per_sample
    return -(-n // (grid_for(n, 256, n_sms) * 256))


def pair_smem(max_taps, esz):        # pidm_pack_weights_pairs
    return 32 * (32 * (max_taps | 1) + 2) * esz


def mlp_smem(td):                    # pidm_block_mlps_fwd / _bwd: [32][td + 1] floats
    return MLP_BCHUNK * (td + 1) * 4


# ----------------------------------------------------------------------------------------------------------------------
# shared helpers
# ----------------------------------------------------------------------------------------------------------------------
def _within(y, r, bound):
    d = (y.double() - r).abs()
    return bool((d <= bound).all())


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _exact(what, y, r):
    bad = int((_bits(y.contiguous()) != _bits(r.contiguous())).sum())
    note(TAG, what + ' (elements differing)', float(bad))
    assert bad == 0, f'{what}: {bad} elements differ bitwise'


def _upload(rows, dt):
    arr = np.array(rows, dtype=dt)
    return torch.from_numpy(arr.view(np.uint8).copy()).to(DEV)


# ----------------------------------------------------------------------------------------------------------------------
# time embedding (linear.cu): SinusoidalPosEmb -> Linear -> GELU(erf) -> Linear (-> SiLU)
# ----------------------------------------------------------------------------------------------------------------------
def sinusoid(t, dim, edit=None):
    """fp64 emb [B, dim] and |t f| per element; edit: 'halves_swapped', 'exponent_over_half'"""
    half = dim // 2
    k = torch.arange(half, dtype=torch.float64, device=t.device)
    f = torch.exp(k * -(math.log(10000) / (half if edit == 'exponent_over_half' else half - 1)))
    arg = t.double()[:, None] * f[None]
    e = (arg.cos(), arg.sin()) if edit == 'halves_swapped' else (arg.sin(), arg.cos())
    return torch.cat(e, dim=1), arg.abs().repeat(1, 2)


def gelu64(x, edit=None):
    return F.gelu(x, approximate='tanh' if edit == 'tanh_gelu' else 'none')


def time_fwd_ref(t, W1, b1, W2, b2, edit=None):
    """fp64 (value, bound) of emb, h1, temb, silu_t.  The bound of each stage adds its own rounding
    (C_GEMV sqrt(K) u A, the activations' C_ACT terms) to the error of its input carried through |W| or the Lipschitz
    constant of the activation."""
    dim = W1.shape[1]
    W1, b1, W2, b2 = (v.double() for v in (W1, b1, W2, b2))
    e, tf = sinusoid(t, dim, edit)
    E_e = C_SIN * U * (1 + tf)
    h1 = e @ W1.T + b1
    E_h1 = C_GEMV * math.sqrt(dim + 1) * U * (e.abs() @ W1.abs().T + b1.abs()) + E_e @ W1.abs().T
    a1 = gelu64(h1, edit)
    E_a1 = GELU_LIP * E_h1 + C_ACT * U * h1.abs()
    temb = a1 @ W2.T + b2
    td = W2.shape[0]
    E_t = C_GEMV * math.sqrt(td + 1) * U * (a1.abs() @ W2.abs().T + b2.abs()) + E_a1 @ W2.abs().T
    s = F.silu(temb)
    E_s = SILU_LIP * E_t + U * (C_ACT + 2 * temb.abs()) * s.abs()
    return {'emb': (e, E_e), 'h1': (h1, E_h1), 'temb': (temb, E_t), 'silu_t': (s, E_s)}


def time_operands(B, dim, td, t_spec, seed):
    g = gen(seed)
    W1 = torch.randn(td, dim, generator=g, device=DEV) / math.sqrt(dim)
    b1 = torch.randn(td, generator=g, device=DEV) * 0.1
    W2 = torch.randn(td, td, generator=g, device=DEV) / math.sqrt(td)
    b2 = torch.randn(td, generator=g, device=DEV) * 0.1
    if isinstance(t_spec, int):
        t = torch.full((B,), t_spec, dtype=torch.long, device=DEV)
    else:                                      # 'mix': 0, 1, 99, 249 and draws below 250
        t = torch.randint(0, 250, (B,), generator=g, device=DEV)
        t[:min(B, 4)] = torch.tensor([0, 1, 99, 249], device=DEV)[:min(B, 4)]
    return t, W1, b1, W2, b2


def time_fwd_launch(t, W1, b1, W2, b2):
    B, (td, dim) = t.shape[0], W1.shape
    bufs = [guarded(B * dim)] + [guarded(B * td) for _ in range(3)]
    call_sync('pidm_time_embed_fwd', t, W1, b1, W2, b2, *(o for _, o in bufs), B, dim, td)
    assert all(guards_intact(b) for b, _ in bufs)
    emb, h1, temb, s = (o.view(B, -1) for _, o in bufs)
    return {'emb': emb, 'h1': h1, 'temb': temb, 'silu_t': s}


# (B, dim, td, t): table rows at t = 249 (the sampling step) and a mix; synthetic: the largest block (td = 1024),
# dim = td and dim = 4, B = 1, t in {0, 1, 99, 249}
TIME_SYNTH = ([(3, 1024, 1024, 'mix'), (2, 4, 64, 'mix'), (1, 32, 128, 249), (1, 128, 512, 'mix'), (7, 64, 64, 'mix')]
              + [(4, 128, 512, t) for t in (0, 1, 99, 249)])
# t = 999 is outside the +-100 pi range in which sin.approx keeps its stated accuracy: the bound must still hold
TIME_FAR = [(4, 128, 512, 999), (2, 1024, 1024, 999)]


def _time_rows():
    return ([k + (249,) for k in TIME_FWD_TABLE] + [k + ('mix',) for k in TIME_FWD_TABLE] + TIME_SYNTH + TIME_FAR)


@gpu
@pytest.mark.parametrize('row', _time_rows(), ids=lambda r: f'B{r[0]}_dim{r[1]}_td{r[2]}_t{r[3]}')
def test_time_embed_fwd_replay(row):
    B, dim, td, ts = row
    ops = time_operands(B, dim, td, ts, 100 + dim)
    y = time_fwd_launch(*ops)
    ref = time_fwd_ref(*ops)
    tag = ' (t = 999, outside sin.approx range)' if ts == 999 else ''
    print(f'[glue census] time_fwd emb max |err| {(y["emb"].double() - ref["emb"][0]).abs().max().item():.3g}{tag}')
    for k in ('emb', 'h1', 'temb', 'silu_t'):
        check(TAG, f'time_fwd {k}{tag}', y[k], *ref[k])


def time_bwd_ref(d_silu, emb, h1, temb, W2, ws_dt, ws_dh, prefill, edit=None):
    """fp64 stage 1 (dt, dh, from the kernel's fp32 inputs) and stage 2 (dW1, db1, dW2, db2 from the kernel's own
    workspace dt, dh, accumulated onto the prefill), each (value, bound)"""
    d, e, h, z, W2 = (v.double() for v in (d_silu, emb, h1, temb, W2))
    B, td = h.shape
    sg = torch.sigmoid(z)
    sp = sg * (1 + z * (1 - sg))
    dt = d * sp
    E_dt = U * (C_ACT + 2 * z.abs()) * d.abs() * (sg + z.abs() * sg * (1 - sg))
    da = dt @ W2
    E_da = C_GEMV * math.sqrt(td) * U * (dt.abs() @ W2.abs()) + E_dt @ W2.abs()
    phi = torch.exp(-0.5 * h * h) / math.sqrt(2 * math.pi)
    cdf = 0.5 * (1 + torch.erf(h / math.sqrt(2)))
    gp = cdf + h * phi
    dh = da * gp
    E_dh = gp.abs() * E_da + da.abs() * U * (C_ACT * (cdf + (h * phi).abs()) + h * h * (h * phi).abs())
    wdt, wdh = ws_dt.double(), ws_dh.double()
    gh = gelu64(h, edit)
    k = math.sqrt(B + 1)
    pW1, pb1, pW2, pb2 = (v.double() for v in prefill)
    dW2 = pW2 + wdt.T @ gh
    E_dW2 = C_GEMV * k * U * (pW2.abs() + wdt.abs().T @ gh.abs()) + wdt.abs().T @ (C_ACT * U * h.abs())
    db2 = pb2 + wdt.sum(0)
    E_db2 = C_GEMV * k * U * (pb2.abs() + wdt.abs().sum(0))
    dW1 = pW1 + wdh.T @ e
    E_dW1 = C_GEMV * k * U * (pW1.abs() + wdh.abs().T @ e.abs())
    db1 = pb1 + wdh.sum(0)
    E_db1 = C_GEMV * k * U * (pb1.abs() + wdh.abs().sum(0))
    return {'dt': (dt, E_dt), 'dh': (dh, E_dh), 'dW1': (dW1, E_dW1), 'db1': (db1, E_db1), 'dW2': (dW2, E_dW2),
            'db2': (db2, E_db2)}


def time_bwd_launch(B, dim, td, ts, parts, seed):
    t, W1, b1, W2, b2 = time_operands(B, dim, td, ts, seed)
    fw = time_fwd_launch(t, W1, b1, W2, b2)
    g = gen(seed + 1)
    d_silu = torch.randn(B, td, generator=g, device=DEV)
    prefill = [torch.randn(*s, generator=g, device=DEV) * 0.01 for s in ((td, dim), (td,), (td, td), (td,))]
    outs = [guarded(p.numel()) for p in prefill]
    for (_, o), p in zip(outs, prefill):
        o.copy_(p.reshape(-1))
    bw, ws = guarded(2 * B * td)
    for p in (2, 1):                           # stage 1 then stage 2, as ops._TimeEmbed.backward issues them; a
        if p == 2 or parts & 1:                # parts = 1 row reads the workspace a stage-1 call left
            call_sync('pidm_time_embed_bwd', d_silu, fw['emb'], fw['h1'], fw['temb'], W2, *(o for _, o in outs), ws, B,
                      dim, td, p)
    assert guards_intact(bw) and all(guards_intact(b) for b, _ in outs)
    grads = [o.view(p.shape) for (_, o), p in zip(outs, prefill)]
    return (d_silu, fw, W2, prefill), ws.view(2, B, td), grads


@gpu
@pytest.mark.parametrize('row', [k for k in TIME_BWD_TABLE] + [(r[0], r[1], r[2], 3) for r in TIME_SYNTH[:5]]
                         + [(33, 128, 512, 3), (64, 32, 128, 1)], ids=lambda r: f'B{r[0]}_dim{r[1]}_td{r[2]}_parts{r[3]}')
def test_time_embed_bwd_replay(row):
    B, dim, td, parts = row
    (d_silu, fw, W2, prefill), ws, grads = time_bwd_launch(B, dim, td, 'mix', parts, 200 + dim)
    ref = time_bwd_ref(d_silu, fw['emb'], fw['h1'], fw['temb'], W2, ws[0], ws[1], prefill)
    check(TAG, 'time_bwd dt', ws[0], *ref['dt'])           # stage 1 runs in every row
    check(TAG, 'time_bwd dh', ws[1], *ref['dh'])
    for name, y, p in zip(('dW1', 'db1', 'dW2', 'db2'), grads, prefill):
        if parts & 1:
            check(TAG, f'time_bwd {name}', y, *ref[name])
        else:
            _exact(f'time_bwd {name} untouched by stage 1', y, p)


# ----------------------------------------------------------------------------------------------------------------------
# block MLPs (linear.cu): out_e = silu_t W_e^T + b_e for every ResnetBlock in one launch
# ----------------------------------------------------------------------------------------------------------------------
class MlpCase:
    """operands, device table and guarded outputs of one block-MLP launch"""

    def __init__(self, B, td, ns, seed, with_grad=False):
        g = gen(seed)
        self.B, self.td, self.ns = B, td, list(ns)
        self.s = torch.randn(B, td, generator=g, device=DEV)
        self.W = [torch.randn(n, td, generator=g, device=DEV) / math.sqrt(td) for n in ns]
        self.b = [torch.randn(n, generator=g, device=DEV) * 0.1 for n in ns]
        self.out = [guarded(B * n) for n in ns]
        self.dout = [torch.randn(B, n, generator=g, device=DEV) for n in ns]
        self.pW = [torch.randn(n, td, generator=g, device=DEV) for n in ns]
        self.pb = [torch.randn(n, generator=g, device=DEV) for n in ns]
        self.dW = [guarded(n * td) for n in ns]
        self.db = [guarded(n) for n in ns]
        for (_, o), p in zip(self.dW + self.db, self.pW + self.pb):
            o.copy_(p.reshape(-1))
        self.ds = guarded(B * td)
        rows = [(W.data_ptr(), b.data_ptr(), dW.data_ptr() if with_grad else 0, db.data_ptr() if with_grad else 0,
                 o.data_ptr(), do.data_ptr(), n, 0)
                for W, b, (_, dW), (_, db), (_, o), do, n in zip(self.W, self.b, self.dW, self.db, self.out, self.dout, ns)]
        from physicsinformeddiffusionmodels_b200 import packing
        self.table = _upload(rows, packing._MLP_DT)

    def guards(self):
        return all(guards_intact(b) for b, _ in self.out + self.dW + self.db + [self.ds])

    def fwd(self):
        call_sync('pidm_block_mlps_fwd', self.table, len(self.ns), max(self.ns), self.s, self.B, self.td)
        assert self.guards()
        return [o.view(self.B, n) for (_, o), n in zip(self.out, self.ns)]

    def bwd(self, parts):
        call_sync('pidm_block_mlps_bwd', self.table, len(self.ns), max(self.ns), self.s, self.ds[1], self.B, self.td,
                  parts)
        assert self.guards()
        return ([o.view(n, self.td) for (_, o), n in zip(self.dW, self.ns)], [o for _, o in self.db],
                self.ds[1].view(self.B, self.td))


def mlp_fwd_ref(c, edit=None):
    """fp64 (out_e, bound_e); edit 'ragged_last_row_dropped': the last row of every ragged row chunk left at 0"""
    s = c.s.double()
    res = []
    for W, b, n in zip(c.W, c.b, c.ns):
        W, b = W.double(), b.double()
        r = s @ W.T + b
        if edit == 'ragged_last_row_dropped' and n % MLP_ROWS:
            r[:, n - 1] = 0
        res.append((r, C_GEMV * math.sqrt(c.td + 1) * U * (s.abs() @ W.abs().T + b.abs())))
    return res


def mlp_wgrad_ref(c, edit=None):
    """fp64 [(dW_e, bound), (db_e, bound)] accumulated onto the prefill; edits: 'second_chunk_dropped' (samples 32..63
    missing), 'dW_overwritten' (no prefill)"""
    s = c.s.double()
    keep = torch.ones(c.B, 1, dtype=torch.float64, device=DEV)
    if edit == 'second_chunk_dropped':
        keep[MLP_BCHUNK:2 * MLP_BCHUNK] = 0
    depth = math.sqrt(c.B + -(-c.B // MLP_BCHUNK) + 1)
    res = []
    for d, pW, pb in zip(c.dout, c.pW, c.pb):
        d = d.double() * keep
        pW, pb = (torch.zeros_like(pW.double()), pb.double()) if edit == 'dW_overwritten' else (pW.double(), pb.double())
        res.append(((pW + d.T @ s, C_GEMV * depth * U * (pW.abs() + d.abs().T @ s.abs())),
                    (pb + d.sum(0), C_GEMV * depth * U * (pb.abs() + d.abs().sum(0)))))
    return res


def mlp_dgrad_ref(c, edit=None):
    """fp64 (ds, bound) = sum_e dout_e W_e; edit 'entry_missing': the last entry's term missing"""
    terms = [(d.double() @ W.double(), d.double().abs() @ W.double().abs()) for d, W in zip(c.dout, c.W)]
    K = sum(c.ns)
    r = sum(t for t, _ in (terms[:-1] if edit == 'entry_missing' else terms))
    return r, C_GEMV * math.sqrt(K) * U * sum(a for _, a in terms)


# (B, td, entry rows): B in {1, 5, 32, 33, 64, 256}; rows % 16 and % 32 != 0, entries shorter than max_rows;
# td = 96, 160 ((td/32) % 4 != 0, (td/4) % 16 != 0) and 704 (> 48 KB of shared memory)
MLP_NS = (40, 24, 64, 7)
MLP_SYNTH = ([(B, 128, MLP_NS) for B in (1, 5, 32, 33, 64, 256)] + [(33, 96, MLP_NS), (37, 160, (48, 17)),
                                                                      (65, 704, (96, 40, 1))])


def _mlp_id(r):
    return f'B{r[0]}_td{r[1]}_max{max(r[2])}_n{len(r[2])}'


@gpu
@pytest.mark.parametrize('row', [(k[0], k[1], k[3]) for k in MLP_FWD_TABLE] + MLP_SYNTH, ids=_mlp_id)
def test_block_mlps_fwd_replay(row):
    c = MlpCase(*row, seed=300 + row[0])
    for y, (r, bound) in zip(c.fwd(), mlp_fwd_ref(c)):
        check(TAG, 'mlp_fwd out', y, r, bound)


@gpu
@pytest.mark.parametrize('row', [(k[0], k[1], k[3], k[4]) for k in MLP_BWD_TABLE] + [r + (3,) for r in MLP_SYNTH]
                         + [(33, 128, MLP_NS, 1), (33, 128, MLP_NS, 2)], ids=lambda r: _mlp_id(r) + f'_parts{r[3]}')
def test_block_mlps_bwd_replay(row):
    B, td, ns, parts = row
    c = MlpCase(B, td, ns, seed=400 + B, with_grad=True)
    dWs, dbs, ds = c.bwd(parts)
    if parts & 1:
        for y, yb, ((r, bd), (rb, bdb)) in zip(dWs, dbs, mlp_wgrad_ref(c)):
            check(TAG, 'mlp_bwd dW', y, r, bd)
            check(TAG, 'mlp_bwd db', yb, rb, bdb)
    else:
        for y, yb, pW, pb in zip(dWs, dbs, c.pW, c.pb):
            _exact('mlp_bwd dW untouched', y, pW)
            _exact('mlp_bwd db untouched', yb, pb)
    if parts & 2:
        check(TAG, 'mlp_bwd d_silu', ds, *mlp_dgrad_ref(c))
    else:
        assert torch.isnan(ds).all(), 'd_silu was written without parts & 2'


# ----------------------------------------------------------------------------------------------------------------------
# sumsq and the Adam / EMA step (optim.cu)
# ----------------------------------------------------------------------------------------------------------------------
def sumsq_depth(n):
    """fp32 chain of pidm_sumsq: 4 squares per float4 and grid-stride pass, the tail, a warp, 8 warps, the last CTA's
    strided pass over the partials, a warp, 8 warps, the add onto out"""
    G = sumsq_grid(n)
    iters = -(-(n // 4) // (G * 256))
    return 4 * iters + 1 + 5 + 5 + -(-G // 256) + 5 + 8 + 1


def sumsq_launch(x, prefill, ws=None):
    n = x.numel()
    bo, out = guarded(1)
    out.fill_(prefill)
    if ws is None:
        bw, ws = guarded(1 + SUMSQ_CAP)
        ws.zero_()
    call_sync('pidm_sumsq', x, n, out, ws)
    assert guards_intact(bo)
    assert int(ws[:1].view(torch.int32).item()) == 0, 'the ticket counter was not reset'
    return out


def sumsq_ref(x, prefill, edit=None):
    xd = x.double()
    if edit == 'tail_dropped':
        xd = xd[:x.numel() // 4 * 4]
    r = prefill + (xd * xd).sum()
    return r, (C_SUM + sumsq_depth(x.numel())) * U * r


def _sumsq_x(n, seed):
    x = torch.randn(n, generator=gen(seed), device=DEV)
    x[-(n % 4 or 1):] *= 8                     # a tail that weighs: dropping it must be visible
    return x


# n < 4, n % 4 in {1, 2, 3}, below one CTA (n/4 < 256), the n = 100003 tail, past the 148 * 8 and 8 * SM grid caps
SUMSQ_SYNTH = [1, 2, 3, 5, 6, 7, 1023, 100003, 3 * 4 * 256 * SUMSQ_CAP + 2]


@gpu
@pytest.mark.parametrize('n', [k[0] for k in SUMSQ_TABLE] + SUMSQ_SYNTH)
def test_sumsq_replay(n):
    x = _sumsq_x(n, 500 + n % 97)
    bw, ws = guarded(1 + SUMSQ_CAP)
    ws.zero_()
    a = sumsq_launch(x, 0.375, ws).clone()
    b = sumsq_launch(x, 0.375, ws)                 # the same workspace: the ticket reset that graph replay relies on
    assert guards_intact(bw)
    _exact('sumsq twice on one workspace', b, a)
    check(TAG, 'sumsq', a, *sumsq_ref(x, 0.375))


F32 = lambda v: float(np.float32(v))           # the fp32 ABI arguments, as the kernel receives them
LR, EPS, MU, B1, B2 = F32(1e-4), F32(1e-8), F32(0.99), 0.9, 0.999


def adam_state(n, seed, fresh):
    """p with a block of exact zeros (and ema = 0 there), g ~ 1e-2, m, v zero at a fresh start, else drawn"""
    g_ = gen(seed)
    p = torch.randn(n, generator=g_, device=DEV)
    gr = torch.randn(n, generator=g_, device=DEV) * 0.01
    if fresh:
        m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    else:
        m = torch.randn(n, generator=g_, device=DEV) * 0.01
        v = torch.rand(n, generator=g_, device=DEV) * 1e-4
    ema = p + torch.randn(n, generator=g_, device=DEV) * 1e-3
    zero = torch.arange(n, device=DEV) % 5 == 0
    p[zero], ema[zero] = 0., 0.
    return [p, gr, m, v, ema]


def adam_ref(state, st, gnorm_sq, grad_scale, max_norm, ema_first, edit=None):
    """fp64 reference of clip -> Adam -> EMA (oracle adam_ema_step, with the kernel's grad_scale and EMA switch) on the
    fp32 state, and its bounds: {name: (value, C_ADAM u A)}.  Edits: 'clip_not_clamped', 'scale_after_norm',
    'ema_one_step_early', 'ema_from_pre_update_p', 'fp32_bias_corrections'."""
    p, g, m, v, e = (x.double() for x in state)
    coef = grad_scale
    if gnorm_sq is not None and max_norm > 0:
        total = math.sqrt(gnorm_sq) * (1.0 if edit == 'scale_after_norm' else grad_scale)
        c = max_norm / (total + 1e-6)
        coef *= c if edit == 'clip_not_clamped' else min(c, 1.0)
    if edit == 'fp32_bias_corrections':
        b1, b2 = np.float32(B1), np.float32(B2)
        bc1, bc2 = float(np.float32(1) - b1 ** np.float32(st)), float(np.float32(1) - b2 ** np.float32(st))
    else:
        bc1, bc2 = 1 - B1 ** st, 1 - B2 ** st
    step, rs = LR / bc1, 1 / math.sqrt(bc2)
    gi = g * coef
    m1 = B1 * m + (1 - B1) * gi
    Am = B1 * m.abs() + (1 - B1) * gi.abs()
    v1 = B2 * v + (1 - B2) * gi * gi
    D = v1.sqrt() * rs + EPS
    q = step * m1 / D
    p1 = p - q
    Ap = p.abs() + step * Am / D + q.abs()
    on = ema_first > 0 and st >= ema_first - (1 if edit == 'ema_one_step_early' else 0)
    if on:
        e1 = MU * e + (1 - MU) * (p if edit == 'ema_from_pre_update_p' else p1)
        Ae = MU * e.abs() + (1 - MU) * Ap
    else:
        e1, Ae = e, torch.zeros_like(e)
    k = C_ADAM * U
    return {'m': (m1, k * Am), 'v': (v1, k * v1), 'p': (p1, k * Ap), 'ema': (e1, k * Ae)}


def adam_launch(state, st, device_step, gnorm_sq, grad_scale, max_norm, ema_first, zero_grad):
    """one pidm_adam_ema_step on guarded copies of state; returns {'p','g','m','v','ema'} after the call"""
    n = state[0].numel()
    bufs = [guarded(n) for _ in range(5)]
    for (_, o), x in zip(bufs, state):
        o.copy_(x)
    bg, gn = guarded(1)
    gn.fill_(gnorm_sq if gnorm_sq is not None else 0.)
    bc = None
    if device_step:
        bc = torch.full((3,), -7, dtype=torch.int32, device=DEV)
        bc[1] = st - 1                                   # the counter holds the steps done so far
    p, g, m, v, e = (o for _, o in bufs)
    call_sync('pidm_adam_ema_step', p, g, m, v, e, n, LR, B1, B2, EPS, 0 if device_step else st,
              bc[1:2] if device_step else None, gn if gnorm_sq is not None else None, grad_scale, max_norm, MU, ema_first,
              zero_grad)
    assert all(guards_intact(b) for b, _ in bufs) and guards_intact(bg)
    if device_step:
        assert bc.tolist() == [-7, st, -7], 'the device step counter must advance by exactly one'
    return dict(zip(('p', 'g', 'm', 'v', 'ema'), (p, g, m, v, e)))


def check_adam(y, state, st, gnorm_sq, grad_scale, max_norm, ema_first, zero_grad, edit=None):
    ref = adam_ref(state, st, gnorm_sq, grad_scale, max_norm, ema_first, edit)
    ok = True
    for k in ('m', 'v', 'p', 'ema'):
        if edit is None:
            check(TAG, f'adam {k}', y[k], *ref[k])
        ok &= _within(y[k], *ref[k])
    if edit is None:
        if zero_grad:
            assert bool((_bits(y['g']) == 0).all()), 'zero_grad left a gradient element that is not +0'
        else:
            _exact('adam grad untouched', y['g'], state[1])
        if not (ema_first > 0 and st >= ema_first):
            _exact('adam ema untouched', y['ema'], state[4])
    return ok


# (n, device step, step, grad_scale, max_norm, clip, ema_first_step, zero_grad); clip: 'active' / 'inactive'
# (the gradient norm is given, so the clip state does not depend on the draw); max_norm = 0 switches the clip off
ADAM_SYNTH = ([(n, 1, 1, 1.0, 1.0, 'active', 1, 1) for n in (1, 2, 3, 5, 6, 7, 1023, 100003)]
              + [(3 * 4 * 256 * SUMSQ_CAP + 2, 1, 1, 0.125, 1.0, 'active', 1, 1)]
              + [(4099, ds, st, gs, mn, clip, ef, zg) for ds in (0, 1) for st in (1, 2, 1000)
                 for gs, mn, clip in ((1.0, 1.0, 'active'), (0.125, 1.0, 'inactive'), (0.125, 1.0, 'active'),
                                      (1.0, 0.0, 'off'))
                 for ef, zg in ((0, 0), (1, 1))]
              + [(4099, 1, st, 1.0, 1.0, 'active', 3, 1) for st in (2, 3)])        # the EMA switch-on boundary


def _gnorm(clip, grad_scale, max_norm):
    if clip == 'off':
        return 9.0
    return (4 * max_norm / grad_scale) ** 2 if clip == 'active' else (0.25 * max_norm / grad_scale) ** 2


def _adam_rows():
    rows = []
    for k in ADAM_TABLE:
        n, ds, gs, mn, ef, zg = k
        rows += [(n, ds, st, gs, mn, clip, ef, zg) for st in (1, 1000) for clip in ('active', 'inactive')]
    return rows + ADAM_SYNTH


@gpu
@pytest.mark.parametrize('row', _adam_rows(), ids=lambda r: 'n{}_{}_step{}_gs{}_mn{}_{}_ema{}_zg{}'.format(
    r[0], 'dev' if r[1] else 'host', *r[2:]))
def test_adam_replay(row):
    n, ds, st, gs, mn, clip, ef, zg = row
    state = adam_state(n, 600 + st, fresh=st == 1)
    gnsq = F32(_gnorm(clip, gs, mn))
    y = adam_launch(state, st, ds, gnsq, gs, mn, ef, zg)
    assert check_adam(y, state, st, gnsq, gs, mn, ef, zg)


@gpu
@pytest.mark.parametrize('device_step', [0, 1])
def test_adam_three_chained_steps(device_step):
    """three steps as TrainEngine runs them (sumsq of the gradient, then the step; n = 100003 has a tail of three), each
    checked against the fp64 reference on the state the previous step left; the last one also against the CPU oracle"""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    n = 100003
    p, gr, m, v, ema = adam_state(n, 700, fresh=True)
    bw, ws = guarded(1 + SUMSQ_CAP)
    ws.zero_()
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    pr, mr, vr, er = (x.double().cpu() for x in (p, m, v, ema))
    for st in (1, 2, 3):
        gr = torch.randn(n, generator=gen(710 + st), device=DEV) * 0.01
        state = [x.clone() for x in (p, gr, m, v, ema)]
        nsq = torch.zeros(1, device=DEV)
        call('pidm_sumsq', gr, n, nsq, ws, stream())
        call('pidm_adam_ema_step', p, gr, m, v, ema, n, LR, B1, B2, EPS, 0 if device_step else st,
             counter if device_step else None, nsq, 1.0, 1.0, MU, 1, 0, stream())
        torch.cuda.synchronize()
        check(TAG, 'sumsq (chained)', nsq[0], *sumsq_ref(state[1], 0.0))
        assert check_adam({'p': p, 'g': gr, 'm': m, 'v': v, 'ema': ema}, state, st, nsq.item(), 1.0, 1.0, 1, 0)
        O.adam_ema_step([pr], [state[1].double().cpu()], [mr], [vr], [er], st, lr=LR, eps=EPS, ema_mu=MU)
    if device_step:
        assert counter.item() == 3
    assert torch.allclose(p.double().cpu(), pr, rtol=1e-6, atol=1e-9)
    assert torch.allclose(ema.double().cpu(), er, rtol=1e-6, atol=1e-9)


# ----------------------------------------------------------------------------------------------------------------------
# weight packing (conv_simt.cu)
# ----------------------------------------------------------------------------------------------------------------------
class Arena:
    """every packed matrix of a replay at a 128-element boundary of one NaN-filled buffer, a gap of at least 128
    elements after each: what the packer writes outside its matrices stays NaN"""

    def __init__(self, sizes, dtype):
        self.offs, off = [], 128
        for s in sizes:
            self.offs.append(off)
            off += -(-s // 128) * 128 + 128
        self.buf = torch.full((off,), float('nan'), dtype=dtype, device=DEV)
        self.sizes = sizes

    def view(self, i):
        return self.buf[self.offs[i]:self.offs[i] + self.sizes[i]]

    def gaps_intact(self):
        mask = torch.ones(self.buf.numel(), dtype=torch.bool, device=DEV)
        for o, s in zip(self.offs, self.sizes):
            mask[o:o + s] = False
        return bool(torch.isnan(self.buf[mask]).all())


def _rne(x, dtype, edit=None):
    """fp32 -> the activation dtype, rounded to nearest even (edit 'truncated': the low 16 bits dropped)"""
    if dtype == torch.float32:
        return x.clone()
    if edit == 'truncated':
        return (x.view(torch.int32) & -65536).view(torch.float32).to(dtype)
    return x.to(dtype)


def pack_ref(src, N, C, Cpad, taps, flip, s_n, s_c, dtype, edit=None):
    """Wp[n][tap * Cpad + c] = W[n * s_n + c * s_c + tap_src], tap_src = taps - 1 - tap under flip, zero for c >= C"""
    n = torch.arange(N, device=DEV)[:, None, None]
    tap = torch.arange(taps, device=DEV)[None, :, None]
    c = torch.arange(C, device=DEV)[None, None, :]
    ts = taps - 1 - tap if flip else tap
    out = torch.zeros(N, taps, Cpad, dtype=torch.float32, device=DEV)
    out[..., :C] = src[n * s_n + c * s_c + ts]
    return _rne(out.reshape(-1), dtype, edit)


def pack_src(N, C, taps, s_n, s_c, seed):
    """fp32 weights that are not bf16-exact (a truncating conversion differs from rounding on about half of them)"""
    size = (N - 1) * s_n + (C - 1) * s_c + taps
    return torch.randn(size, generator=gen(seed), device=DEV) * (1 + 2.0 ** -12)


def replay_pack(rows, seed, edit=None):
    """one pidm_pack_weights launch over rows (dtype, N, C, Cpad, taps, flip, s_n, s_c) of one dtype"""
    dtype = DTYPE[rows[0][0]]
    srcs = [pack_src(k[1], k[2], k[4], k[6], k[7], seed + i) for i, k in enumerate(rows)]
    arena = Arena([k[1] * k[4] * k[3] for k in rows], dtype)
    from physicsinformeddiffusionmodels_b200 import packing
    table = _upload([(s.data_ptr(), arena.view(i).data_ptr(), k[6], k[7], k[1], k[2], k[3], k[4], k[5], 0)
                     for i, (s, k) in enumerate(zip(srcs, rows))], packing._PACK_DT)
    call_sync('pidm_pack_weights', table, len(rows), rows[0][0])
    assert arena.gaps_intact(), 'pidm_pack_weights wrote outside its matrices'
    return [(arena.view(i), pack_ref(s, *k[1:], dtype=dtype, edit=edit)) for i, (s, k) in enumerate(zip(srcs, rows))]


# the generic packer: C < Cpad with C odd (the stem at 3 and 1 channels), the dgrad entry of a conv with swapped strides
# (s_n = taps, s_c = Cin * taps) and flip, both dtypes
PACK_SYNTH = [(d, 32, 3, 8, 49, 0, 3 * 49, 49) for d in (0, 1)] + [(d, 16, 1, 8, 9, 0, 9, 9) for d in (0, 1)] \
    + [(d, 24, 32, 32, 9, 1, 9, 24 * 9) for d in (0, 1)]


@gpu
@pytest.mark.parametrize('dtype', [0, 1], ids=['fp32', 'bf16'])
def test_pack_weights_replay(dtype):
    """the census entries (recorded with bf16 activations) in both activation dtypes, and the synthetic ones"""
    rows = sorted({(dtype,) + k[1:] for k in PACK_TABLE}) + [k for k in PACK_SYNTH if k[0] == dtype]
    for y, r in replay_pack(rows, 800):
        _exact(f'pack {"fp32" if dtype == 0 else "bf16"}', y, r)


def pair_ref(src, Cout, Cin, taps, flip, ci_inner, dtype, edit=None):
    """(Wp_f [Cout][taps * Cin], Wp_d [Cin][taps * Cout]) of fp32 weights in the conv ([co][ci][tap]) or convT
    ([ci][co][tap]) layout.  Edits: 'flip_on_convT' (the dgrad flip applied to a transposed layer), 'block_transposed'
    (co and ci swapped inside the first 32 x 32 block), 'truncated'."""
    W = src.view(Cout, Cin, taps) if ci_inner else src.view(Cin, Cout, taps).permute(1, 0, 2)
    if edit == 'block_transposed':
        W = W.clone()
        W[:32, :32] = W[:32, :32].transpose(0, 1).clone()
    f = W.permute(0, 2, 1).reshape(-1)
    Wd = W.flip(2) if (flip or (edit == 'flip_on_convT' and not ci_inner)) else W
    d = Wd.permute(1, 2, 0).reshape(-1)
    return _rne(f.contiguous(), dtype, edit), _rne(d.contiguous(), dtype, edit)


def _tiles(k):
    return (k[1] // 32) * (k[2] // 32)


def replay_pairs(entries, dtype_code, seed, splits=(0,), max_taps=None, edit=None):
    """pidm_pack_weights_pairs over entries (Cout, Cin, taps, flip, ci_inner, has_dgrad), the tile list cut into launches
    at `splits` (tile_base > 0 for all but the first); -> [(y_f, r_f, y_d or None, r_d)] and the arena"""
    from physicsinformeddiffusionmodels_b200 import packing
    dtype = DTYPE[dtype_code]
    srcs = [torch.randn(co * ci * t, generator=gen(seed + i), device=DEV) * (1 + 2.0 ** -12)
            for i, (co, ci, t, *_) in enumerate(entries)]
    sizes = []
    for co, ci, t, _, _, hd in entries:
        sizes += [co * ci * t] + ([co * ci * t] if hd else [])
    arena = Arena(sizes, dtype)
    rows, tmap, views, j = [], [], [], 0
    for i, ((co, ci, t, fl, inner, hd), s) in enumerate(zip(entries, srcs)):
        vf = arena.view(j)
        vd = arena.view(j + 1) if hd else None
        j += 2 if hd else 1
        s_co, s_ci = (ci * t, t) if inner else (t, co * t)
        rows.append((s.data_ptr(), vf.data_ptr(), vd.data_ptr() if hd else 0, s_co, s_ci, co, ci, t, fl, len(tmap), 0))
        tmap += [i] * ((co // 32) * (ci // 32))
        views.append((vf, vd))
    table = _upload(rows, packing._PAIR_DT)
    tm = torch.tensor(tmap, dtype=torch.int32, device=DEV)
    mt = max_taps or max(e[2] for e in entries)
    cuts = list(splits) + [len(tmap)]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        call_sync('pidm_pack_weights_pairs', table, tm, lo, hi - lo, mt, dtype_code)
    out = []
    for (co, ci, t, fl, inner, hd), s, (vf, vd) in zip(entries, srcs, views):
        rf, rd = pair_ref(s, co, ci, t, fl, inner, dtype, edit)
        out.append((vf, rf, vd, rd))
    return out, arena


def _check_pairs(what, out, arena):
    assert arena.gaps_intact(), f'{what}: pidm_pack_weights_pairs wrote outside its matrices'
    bad = {'forward': 0, 'dgrad': 0}
    for vf, rf, vd, rd in out:
        bad['forward'] += int((_bits(vf) != _bits(rf)).sum())
        if vd is not None:
            bad['dgrad'] += int((_bits(vd) != _bits(rd)).sum())
    for k, v in bad.items():
        note(TAG, f'{what} {k} operand (elements differing)', float(v))
    assert not any(bad.values()), f'{what}: packed operands differ bitwise from the permutation: {bad}'


# synthetic entries (Cout, Cin, taps, flip, ci_inner, has_dgrad): taps 1 / 4 / 9 / 16, both layouts, flip 0 / 1, dgrad
# operand absent, fewer taps than max_taps in one launch
PAIR_SYNTH = [(64, 32, 9, 1, 1, 1), (32, 64, 1, 1, 1, 0), (64, 64, 16, 0, 1, 1), (32, 96, 4, 0, 0, 1),
              (96, 32, 16, 0, 0, 1), (32, 32, 9, 0, 0, 0), (64, 32, 1, 1, 1, 1)]
SYNTH_SPLIT = 7                    # the second launch starts at tile 7, inside the (64, 64, 16) entry


@gpu
@pytest.mark.parametrize('dtype', [0, 1], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('split', ['one_launch', 'split'])
def test_pack_pairs_table_replay(dtype, split):
    """every census entry (recorded with bf16 activations) in one table, in both activation dtypes, packed in one
    launch or in two (tile_base > 0, cut inside an entry)"""
    entries = sorted({k[1:] for k in PAIR_TABLE})
    total = sum((e[0] // 32) * (e[1] // 32) for e in entries)
    out, arena = replay_pairs(entries, dtype, 900, splits=(0,) if split == 'one_launch' else (0, total // 2 + 1))
    _check_pairs(f'pair {"fp32" if dtype == 0 else "bf16"}', out, arena)


@gpu
@pytest.mark.parametrize('dtype', [0, 1], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('split', ['one_launch', 'split'])
def test_pack_pairs_synthetic_replay(dtype, split):
    out, arena = replay_pairs(PAIR_SYNTH, dtype, 950, splits=(0,) if split == 'one_launch' else (0, SYNTH_SPLIT))
    _check_pairs(f'pair {"fp32" if dtype == 0 else "bf16"} synthetic', out, arena)


def _launch_entries(k):
    """entries for a census launch row (dtype, tile_base, n_tiles, max_taps): the census entries of the dtype with at
    most max_taps taps, in table order and repeated, then single-tile 32 x 32 entries up to tile_base + n_tiles tiles"""
    dtype, base, n, mt = k
    pool = [e[1:] for e in PAIR_TABLE if e[0] == dtype and e[3] <= mt]
    pool = [e for e in pool if e[2] == mt] + [e for e in pool if e[2] != mt]
    out, tiles = [], 0
    for e in pool * (1 + (base + n) // max(1, sum(_tiles((0,) + e) for e in pool))):
        if tiles + _tiles((0,) + e) > base + n:
            break
        out.append(e)
        tiles += _tiles((0,) + e)
    out += [(32, 32, mt if tiles == 0 and i == 0 else 1, 0, 1, 1) for i in range(base + n - tiles)]
    return out


@gpu
@pytest.mark.parametrize('row', PAIR_LAUNCH_TABLE, ids=lambda k: 'dt{}_base{}_tiles{}_taps{}'.format(*k))
def test_pack_pairs_launch_replay(row):
    dtype, base, n, mt = row
    entries = _launch_entries(row)
    out, arena = replay_pairs(entries, dtype, 990, splits=(0, base) if base else (0,), max_taps=mt)
    _check_pairs('pair launch', out, arena)


def test_references_follow_the_oracle():
    """the fp64 references above against oracle/pidm_oracle.py on the CPU: time_embedding (whose fp32 sinusoid stays
    inside the emb bound, so its temb inside the temb bound) and adam_ema_step evaluated in float64"""
    g = torch.Generator().manual_seed(3)
    dim, td = 32, 128
    sd = {'time_mlp.1.weight': torch.randn(td, dim, generator=g, dtype=torch.float64) / 6,
          'time_mlp.1.bias': torch.randn(td, generator=g, dtype=torch.float64) * .1,
          'time_mlp.3.weight': torch.randn(td, td, generator=g, dtype=torch.float64) / 11,
          'time_mlp.3.bias': torch.randn(td, generator=g, dtype=torch.float64) * .1}
    t = torch.tensor([0, 3, 50, 99, 249, 999])
    ref = time_fwd_ref(t, sd['time_mlp.1.weight'], sd['time_mlp.1.bias'], sd['time_mlp.3.weight'], sd['time_mlp.3.bias'])
    temb, bound = ref['temb']
    assert bool(((O.time_embedding(sd, t, dim) - temb).abs() <= bound).all())
    n = 1001
    p, gr, ema = (torch.randn(n, generator=g, dtype=torch.float64) for _ in range(3))
    gr *= 0.1
    m, v = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    state = [p.clone(), gr, m.clone(), v.clone(), ema.clone()]
    for st in (1, 2, 3):
        nsq = float((state[1] ** 2).sum())
        r = adam_ref(state, st, nsq, 1.0, 1.0, 1)
        O.adam_ema_step([p], [gr], [m], [v], [ema], st, lr=LR, eps=EPS, ema_mu=MU)
        for k, x in (('p', p), ('m', m), ('v', v), ('ema', ema)):
            assert torch.allclose(r[k][0], x, rtol=1e-6, atol=1e-12), (st, k)
        state = [r['p'][0], gr, r['m'][0], r['v'][0], r['ema'][0]]


def _umulhi(x, inv):
    return (x.astype(np.uint64) * np.uint64(inv)) >> np.uint64(32)


def test_pack_pair_reciprocal_division():
    """pack_pair_kernel divides by taps and by run = 32 taps with __umulhi(x, ceil(2^32 / d)), exact for x d < 2^32:
    checked for every index below total = 32 run (div_run) and below run (div_taps) at taps 1..16"""
    for taps in range(1, 17):
        run = 32 * taps
        total = 32 * run
        x = np.arange(total + 8 * 256, dtype=np.uint64)       # the load loop divides indices up to base + 7 * 256
        inv_run = ((1 << 32) + run - 1) // run
        assert (_umulhi(x, inv_run) == x // run).all(), f'div_run wrong at taps = {taps}'
        if taps > 1:
            inv_taps = ((1 << 32) + taps - 1) // taps
            y = np.arange(total, dtype=np.uint64)
            assert (_umulhi(y, inv_taps) == y // taps).all(), f'div_taps wrong at taps = {taps}'


# ----------------------------------------------------------------------------------------------------------------------
# element-wise (elementwise.cu)
# ----------------------------------------------------------------------------------------------------------------------
def _multi_B(per_sample):
    """a batch whose grid_for-capped grid (16 CTAs per SM) takes at least three grid-stride passes"""
    vec = 4 if per_sample % 4 == 0 else 1
    return -(-3 * 16 * sms() * 256 * vec // per_sample) + 1


def _ew_B(spec, per_sample):
    return _multi_B(per_sample) if spec == 'multi' else spec


def qsample_ref(x0, eps, t, sa, sb, edit=None):
    """fp64 x_t = sa[t_b] x0 + sb[t_b] eps (oracle q_sample); edit 'indexed_by_element': t[i mod B] for element i"""
    B = x0.shape[0]
    if edit == 'indexed_by_element':
        idx = t[torch.arange(x0.numel(), device=DEV) % B].view(x0.shape)
    else:
        idx = t[:, None].expand_as(x0)
    a, s = sa.double()[idx], sb.double()[idx]
    r = a * x0.double() + s * eps.double()
    return r, C_EW * U * ((a * x0.double()).abs() + (s * eps.double()).abs())


def qsample_launch(B, per, seed):
    g = gen(seed)
    tab = O.diffusion_tables(250)
    sa, sb = tab['alphas_bar_sqrt'].float().to(DEV), tab['one_minus_alphas_bar_sqrt'].float().to(DEV)
    x0, eps = torch.randn(B, per, generator=g, device=DEV), torch.randn(B, per, generator=g, device=DEV)
    t = torch.randint(0, 250, (B,), generator=g, device=DEV)
    t[0] = 249
    bo, xt = guarded(B * per)
    call_sync('pidm_qsample', x0, eps, t, sa, sb, xt, B, per)
    assert guards_intact(bo)
    return (x0, eps, t, sa, sb), xt.view(B, per)


# (B or 'multi', per_sample): per_sample % 4 == 0 (float4) and != 0 (scalar: 65 x 65 fields), capped grids, B = 1
EW_SYNTH = [(1, 8192), (3, 4225), (5, 3 * 4225), ('multi', 8192), ('multi', 4225), (1, 3), (7, 12)]


@gpu
@pytest.mark.parametrize('row', [k for k in QSAMPLE_TABLE] + EW_SYNTH, ids=lambda k: f'B{k[0]}_per{k[1]}')
def test_qsample_replay(row):
    ops, y = qsample_launch(_ew_B(row[0], row[1]), row[1], 1000 + row[1] % 89)
    check(TAG, 'qsample', y, *qsample_ref(*ops))
    if row == (5, 3 * 4225):                   # the oracle's own q_sample (fp32) on the same operands
        x0, eps, t, sa, sb = ops
        tab = {'alphas_bar_sqrt': sa.cpu(), 'one_minus_alphas_bar_sqrt': sb.cpu()}
        assert torch.allclose(y.cpu(), O.q_sample(x0.cpu(), t.cpu(), eps.cpu(), tab), rtol=1e-6, atol=1e-6)


def axpby_ref(a, x, b, y, c, z):
    t = [v[:, None].double() * w.double() for v, w in ((a, x), (b, y), (c, z))]
    return sum(t), C_EW * U * sum(v.abs() for v in t)


@gpu
@pytest.mark.parametrize('row', [k for k in AXPBY_TABLE] + EW_SYNTH, ids=lambda k: f'B{k[0]}_per{k[1]}')
def test_axpby_replay(row):
    B, per = _ew_B(row[0], row[1]), row[1]
    g = gen(1100 + per % 89)
    a, b, c = (torch.randn(B, generator=g, device=DEV) for _ in range(3))
    x, y, z = (torch.randn(B, per, generator=g, device=DEV) for _ in range(3))
    bo, out = guarded(B * per)
    call_sync('pidm_axpby_per_sample', a, x, b, y, c, z, out, B, per)
    assert guards_intact(bo)
    check(TAG, 'axpby', out.view(B, per), *axpby_ref(a, x, b, y, c, z))


@gpu
@pytest.mark.parametrize('n', [k[0] for k in SCALE_TABLE] + [1, 7, 4225, 3 * 16 * 256 * 132 * 3 + 5])
def test_scale_replay(n):
    g = gen(1200 + n % 89)
    x, alpha = torch.randn(n, generator=g, device=DEV), torch.randn(1, generator=g, device=DEV)
    bo, out = guarded(n)
    call_sync('pidm_scale', x, alpha, out, n)
    assert guards_intact(bo)
    _exact('scale', out, x * alpha)


def _rows_spec(spec, C):
    return -(-3 * 16 * sms() * 256 * 8 // C) + 1 if spec == 'multi' else spec


CONCAT_SYNTH = [(1, 8, 8, 1), (1, 8, 8, 0), (37, 32, 64, 1), (37, 64, 8, 0), ('multi', 64, 32, 1), ('multi', 16, 8, 0)]


@gpu
@pytest.mark.parametrize('row', [k for k in CONCAT_TABLE] + CONCAT_SYNTH, ids=lambda k: 'rows{}_Ca{}_Cb{}_dt{}'.format(*k))
def test_concat_replay(row):
    rows, Ca, Cb, code = _rows_spec(row[0], row[1] + row[2]), *row[1:]
    dtype = DTYPE[code]
    g = gen(1300 + Ca)
    a = torch.randn(rows, Ca, generator=g, device=DEV).to(dtype)
    b = torch.randn(rows, Cb, generator=g, device=DEV).to(dtype)
    bo, out = guarded(rows * (Ca + Cb), dtype)
    call_sync('pidm_concat_channels', a, b, out, rows, Ca, Cb, code)
    assert guards_intact(bo)
    _exact('concat', out.view(rows, Ca + Cb), concat_ref(a, b))


def concat_ref(a, b, edit=None):
    return torch.cat((b, a) if edit == 'halves_swapped' else (a, b), dim=1)


@gpu
@pytest.mark.parametrize('row', [k for k in SPLIT_TABLE] + CONCAT_SYNTH, ids=lambda k: 'rows{}_Ca{}_Cb{}_dt{}'.format(*k))
def test_split_replay(row):
    rows, Ca, Cb, code = _rows_spec(row[0], row[1] + row[2]), *row[1:]
    dtype = DTYPE[code]
    gsrc = torch.randn(rows, Ca + Cb, generator=gen(1400 + Ca), device=DEV).to(dtype)
    ba, ga = guarded(rows * Ca, dtype)
    bb, gb = guarded(rows * Cb, dtype)
    call_sync('pidm_split_channels', gsrc, ga, gb, rows, Ca, Cb, code)
    assert guards_intact(ba) and guards_intact(bb)
    _exact('split a', ga.view(rows, Ca), gsrc[:, :Ca])
    _exact('split b', gb.view(rows, Cb), gsrc[:, Ca:])


def nchw_ref(x, Cpad, dtype):
    B, C, HW = x.shape
    r = torch.zeros(B, HW, Cpad, dtype=torch.float32, device=DEV)
    r[..., :C] = x.permute(0, 2, 1)
    return r.to(dtype)


NCHW_SYNTH = [(1, 2, 4096, 8, 1), (3, 10, 4225, 16, 1), (2, 3, 17, 8, 0), (1, 8, 64, 8, 0), ('multi', 2, 4096, 8, 1)]


@gpu
@pytest.mark.parametrize('row', [k for k in NCHW_TABLE] + NCHW_SYNTH, ids=lambda k: 'B{}_C{}_HW{}_Cpad{}_dt{}'.format(*k))
def test_nchw_to_nhwc_replay(row):
    B, C, HW, Cpad, code = row
    if B == 'multi':                           # grid_for(B * HW, 128) capped, three or more passes
        B = -(-3 * 16 * sms() * 128 // HW) + 1
    dtype = DTYPE[code]
    x = torch.randn(B, C, HW, generator=gen(1500 + C), device=DEV)
    bo, out = guarded(B * HW * Cpad, dtype)    # NaN: a padding lane left unwritten would stay NaN
    call_sync('pidm_nchw_to_nhwc', x, out, B, C, HW, Cpad, code)
    assert guards_intact(bo)
    _exact('nchw_to_nhwc (padding included)', out.view(B, HW, Cpad), nchw_ref(x, Cpad, dtype))


# ----------------------------------------------------------------------------------------------------------------------
# mutants: the predicates above reject edited references
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('edit', ['halves_swapped', 'exponent_over_half', 'tanh_gelu'])
def test_mutant_time_embed(edit):
    ops = time_operands(16, 128, 512, 'mix', 77)
    y = time_fwd_launch(*ops)
    ref, mut = time_fwd_ref(*ops), time_fwd_ref(*ops, edit=edit)
    assert all(_within(y[k], *ref[k]) for k in ref)
    assert not all(_within(y[k], *mut[k]) for k in mut), edit


@gpu
def test_mutant_time_embed_bwd_tanh_gelu():
    (d_silu, fw, W2, prefill), ws, grads = time_bwd_launch(16, 128, 512, 'mix', 3, 78)
    ref = time_bwd_ref(d_silu, fw['emb'], fw['h1'], fw['temb'], W2, ws[0], ws[1], prefill)
    mut = time_bwd_ref(d_silu, fw['emb'], fw['h1'], fw['temb'], W2, ws[0], ws[1], prefill, edit='tanh_gelu')
    assert _within(grads[2], *ref['dW2']) and not _within(grads[2], *mut['dW2'])


@gpu
def test_mutant_block_mlps_fwd_ragged_last_row_dropped():
    c = MlpCase(33, 128, MLP_NS, seed=81)
    ys = c.fwd()
    assert all(_within(y, r, b) for y, (r, b) in zip(ys, mlp_fwd_ref(c)))
    assert not all(_within(y, r, b) for y, (r, b) in zip(ys, mlp_fwd_ref(c, 'ragged_last_row_dropped')))


@gpu
@pytest.mark.parametrize('edit', ['second_chunk_dropped', 'dW_overwritten'])
def test_mutant_block_mlps_wgrad(edit):
    c = MlpCase(64, 128, MLP_NS, seed=82, with_grad=True)
    dWs, dbs, _ = c.bwd(1)
    ok = lambda ref: all(_within(y, r, b) and _within(yb, rb, bb) for y, yb, ((r, b), (rb, bb)) in zip(dWs, dbs, ref))
    assert ok(mlp_wgrad_ref(c))
    assert not ok(mlp_wgrad_ref(c, edit)), edit


@gpu
def test_mutant_block_mlps_dgrad_entry_missing():
    c = MlpCase(33, 128, MLP_NS, seed=83, with_grad=True)
    _, _, ds = c.bwd(2)
    assert _within(ds, *mlp_dgrad_ref(c))
    assert not _within(ds, *mlp_dgrad_ref(c, 'entry_missing'))


ADAM_MUTANTS = {                 # edit: (n, device step, step, grad_scale, max_norm, clip, ema_first_step, zero_grad)
    'clip_not_clamped': (4099, 1, 2, 1.0, 1.0, 'inactive', 1, 1),
    'scale_after_norm': (4099, 1, 2, 0.125, 1.0, 'active', 1, 1),
    'ema_one_step_early': (4099, 1, 2, 1.0, 1.0, 'active', 3, 1),
    'ema_from_pre_update_p': (4099, 1, 2, 1.0, 1.0, 'active', 1, 1),
    'fp32_bias_corrections': (4099, 1, 1, 1.0, 1.0, 'active', 1, 1),
}


@gpu
@pytest.mark.parametrize('edit', list(ADAM_MUTANTS))
def test_mutant_adam(edit):
    n, ds, st, gs, mn, clip, ef, zg = ADAM_MUTANTS[edit]
    state = adam_state(n, 88, fresh=st == 1)
    gnsq = F32(_gnorm(clip, gs, mn))
    y = adam_launch(state, st, ds, gnsq, gs, mn, ef, zg)
    assert check_adam(y, state, st, gnsq, gs, mn, ef, zg, edit='none')
    assert not check_adam(y, state, st, gnsq, gs, mn, ef, zg, edit=edit), edit


@gpu
@pytest.mark.parametrize('n', [5, 100003])
def test_mutant_sumsq_tail_dropped(n):
    x = _sumsq_x(n, 89)
    y = sumsq_launch(x, 0.0)
    assert _within(y, *sumsq_ref(x, 0.0))
    assert not _within(y, *sumsq_ref(x, 0.0, 'tail_dropped'))


@gpu
@pytest.mark.parametrize('edit', ['flip_on_convT', 'block_transposed', 'truncated'])
def test_mutant_pack_pairs(edit):
    entries = [(64, 64, 9, 1, 1, 1), (64, 32, 16, 0, 0, 1)]
    out, _ = replay_pairs(entries, 1, 91)
    mut, _ = replay_pairs(entries, 1, 91, edit=edit)
    same = lambda a, b: bool((_bits(a) == _bits(b)).all())
    assert all(same(vf, rf) and same(vd, rd) for vf, rf, vd, rd in out)
    assert not all(same(vf, rf) and same(vd, rd) for (vf, _, vd, _), (_, rf, _, rd) in zip(out, mut)), edit


@gpu
def test_mutant_pack_truncated():
    rows = [(1, 32, 3, 8, 49, 0, 3 * 49, 49)]
    (y, r), = replay_pack(rows, 92)
    (_, m), = replay_pack(rows, 92, edit='truncated')
    assert bool((_bits(y) == _bits(r)).all()) and not bool((_bits(y) == _bits(m)).all())


@gpu
def test_mutant_qsample_indexed_by_element():
    ops, y = qsample_launch(5, 4225, 93)
    assert _within(y, *qsample_ref(*ops))
    assert not _within(y, *qsample_ref(*ops, edit='indexed_by_element'))


@gpu
def test_mutant_concat_halves_swapped():
    a = torch.randn(9, 32, generator=gen(94), device=DEV).bfloat16()
    b = torch.randn(9, 32, generator=gen(95), device=DEV).bfloat16()
    out = torch.empty(9, 64, dtype=torch.bfloat16, device=DEV)
    call_sync('pidm_concat_channels', a, b, out, 9, 32, 32, 1)
    assert torch.equal(_bits(out), _bits(concat_ref(a, b)))
    assert not torch.equal(_bits(out), _bits(concat_ref(a, b, 'halves_swapped')))


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
@gpu
def test_plan_coverage():
    n_sms = sms()
    # block MLPs
    mlp = [(k[0], k[1], k[3]) for k in MLP_FWD_TABLE] + MLP_SYNTH
    Bs = {r[0] for r in mlp}
    assert {1, 5, 32, 33, 64, 256} <= Bs, f'block MLP batches missing: {sorted({1, 5, 32, 33, 64, 256} - Bs)}'
    ns = [n for r in mlp for n in r[2]]
    tds = {r[1] for r in mlp}
    cases = {'rows % 16 != 0': any(n % MLP_ROWS for n in ns), 'rows % 32 != 0': any(n % MLP_DG_ROWS for n in ns),
             'entries shorter than max_rows': any(len(set(r[2])) > 1 for r in mlp),
             '(td/32) % 4 != 0': any((td // 32) % 4 for td in tds), '(td/4) % 16 != 0': any((td // 4) % 16 for td in tds),
             '> 48 KB shared memory': any(mlp_smem(td) > 48 * 1024 for td in tds), 'td = 704': 704 in tds,
             'a partial sample chunk': any(B % MLP_BCHUNK for B in Bs), 'several sample chunks': any(B > 2 * MLP_BCHUNK for B in Bs)}
    bwd = [(k[0], k[1], k[3]) for k in MLP_BWD_TABLE] + MLP_SYNTH
    cases['backward: a partial chunk after full ones'] = any(B > MLP_BCHUNK and B % MLP_BCHUNK for B, _, _ in bwd)
    cases['backward: ragged row chunks'] = any(n % MLP_ROWS for _, _, r in bwd for n in r)
    missing = [c for c, ok in cases.items() if not ok]
    assert not missing, f'block MLP rows miss {missing}'
    # time embedding
    rows = _time_rows()
    cases = {'td = 1024': any(r[2] == 1024 for r in rows), 'dim = td': any(r[1] == r[2] for r in rows),
             'dim = 4': any(r[1] == 4 for r in rows), 'B = 1': any(r[0] == 1 for r in rows),
             't = 999 (outside sin.approx range)': any(r[3] == 999 for r in rows)}
    for t in (0, 1, 99, 249):
        cases[f't = {t}'] = any(r[3] in (t, 'mix') for r in rows)
    missing = [c for c, ok in cases.items() if not ok]
    assert not missing, f'time embedding rows miss {missing}'
    # sumsq / Adam
    sn = [k[0] for k in SUMSQ_TABLE] + SUMSQ_SYNTH
    an = _adam_rows()
    for name, nset in (('sumsq', sn), ('adam', [r[0] for r in an])):
        cases = {'n < 4': any(n < 4 for n in nset), 'n % 4 = 1, 2, 3': {1, 2, 3} <= {n % 4 for n in nset},
                 'below one CTA': any(n // 4 < 256 for n in nset),
                 'past the sumsq grid cap': any(sumsq_grid(n) == SUMSQ_CAP and n // 4 > 2 * 256 * SUMSQ_CAP for n in nset),
                 'past the Adam grid cap': any(n // 4 > 2 * 256 * adam_grid(n, n_sms) for n in nset)}
        missing = [c for c, ok in cases.items() if not ok]
        assert not missing, f'{name} rows miss {missing}'
    cases = {'host step': any(not r[1] for r in an), 'device step': any(r[1] for r in an)}
    for clip in ('active', 'inactive', 'off'):
        cases[f'clip {clip}'] = any(r[5] == clip for r in an)
    for gs in (1.0, 0.125):
        cases[f'grad_scale {gs}'] = any(r[3] == gs for r in an)
    cases.update({'ema_first_step 0': any(r[6] == 0 for r in an), 'ema_first_step 1': any(r[6] == 1 for r in an),
                  'EMA switch-on boundary': any(r[6] > 1 and r[2] == r[6] - 1 for r in an)
                  and any(r[6] > 1 and r[2] == r[6] for r in an),
                  'zero_grad 0': any(r[7] == 0 for r in an), 'zero_grad 1': any(r[7] == 1 for r in an)})
    missing = [c for c, ok in cases.items() if not ok]
    assert not missing, f'Adam rows miss {missing}'
    # pair packing
    pe = [k[1:] for k in PAIR_TABLE] + PAIR_SYNTH
    cases = {f'taps {t}': any(e[2] == t for e in pe) for t in (1, 4, 9, 16)}
    cases.update({'conv layout': any(e[4] for e in pe), 'convT layout': any(not e[4] for e in pe),
                  'flip 0': any(not e[3] for e in pe), 'flip 1': any(e[3] for e in pe),
                  'dst_d null': any(not e[5] for e in pe),
                  'tile_base > 0 inside an entry': 0 < SYNTH_SPLIT - 4 < 4,
                  'fewer taps than max_taps in one launch': len({e[2] for e in PAIR_SYNTH}) > 1,
                  'fp32, max_taps 16 (> 48 KB)': pair_smem(max(e[2] for e in PAIR_SYNTH), 4) > 48 * 1024})
    missing = [c for c, ok in cases.items() if not ok]
    assert not missing, f'pair packing rows miss {missing}'
    pk = PACK_TABLE + PACK_SYNTH
    assert any(k[2] < k[3] and k[2] % 2 for k in pk), 'generic packer: no C < Cpad with C odd'
    assert any(k[5] and k[6] < k[7] for k in pk), 'generic packer: no dgrad entry (swapped strides, flip)'
    # element-wise
    ew = [(_ew_B(b, p), p) for b, p in [k for k in QSAMPLE_TABLE] + EW_SYNTH]
    cases = {'per_sample % 4 == 0': any(p % 4 == 0 for _, p in ew), 'per_sample % 4 != 0': any(p % 4 for _, p in ew),
             'capped float4 grid, >= 3 passes': any(p % 4 == 0 and ew_passes(B, p, n_sms) >= 3 for B, p in ew),
             'capped scalar grid, >= 3 passes': any(p % 4 and ew_passes(B, p, n_sms) >= 3 for B, p in ew),
             'B = 1': any(B == 1 for B, _ in ew)}
    cc = [k for k in CONCAT_TABLE] + CONCAT_SYNTH
    cases.update({'concat rows = 1': any(k[0] == 1 for k in cc), 'concat bf16 and fp32': {k[3] for k in cc} == {0, 1},
                  'concat capped grid': any(k[0] == 'multi' for k in cc),
                  'nchw padding channels': any(k[1] < k[3] for k in NCHW_TABLE + NCHW_SYNTH),
                  'nchw bf16 and fp32': {k[4] for k in NCHW_TABLE + NCHW_SYNTH} == {0, 1}})
    missing = [c for c, ok in cases.items() if not ok]
    assert not missing, f'element-wise rows miss {missing}'

