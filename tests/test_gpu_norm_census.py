"""Every GroupNorm, LayerNorm and column-sum launch of the benchmarked steps, and every launch plan of norm.cu, replayed
element by element against an fp64 reference.

pidm_groupnorm_silu_bwd picks a channel slab, a thread count, a cluster size 1..8 and one of five code paths from the
shape, the batch and the SM count; the forward sizes its apply grid by three rules; the LayerNorm kernels cap their grid
and loop.  The operator tests in test_gpu_ops.py compare whole tensors by a norm ratio against an fp32 reference, which a
bug confined to one cluster rank, one channel slab or the last pixel rows cannot move.  Same four parts as the other
census files:

  1. census: the distinct keys of the five entry points in one eager step of every workload bench.py times must equal the
     tables below (`python tests/census.py --print-table` regenerates them);
  2. replay: every table row plus synthetic rows, through the C ABI, with bf16 and with fp32 activations, on seeded
     inputs, against the fp64 evaluation of the contract in include/pidm.h.  With u = 2^-24, rnd = 2^-8 (bf16 output) or
     2^-24 (fp32 output) and A(.) the absolute-value evaluation of the same expression:
        statistics            |sums - r| <= C_ACC sqrt(n) u A,   n = HW C/G
        y, dx                 |o - r|    <= rnd |r| + C_EL e(o)
        parameter / FiLM / producer-bias gradients, column sums
                              |o - r|    <= C_EL e(o) + C_ACC sqrt(K) u (|prefill| + A),   K = summed pixels
     e(o) propagates, to first order, a few fp32 roundings per operation, the error of the fast exponential (norm.cu is
     built with --use_fast_math: exp2 of a rounded product, about u (8 + 2|z|) relative, see _silu_terms) and the error
     of mean and variance.  The variance is var = max(ss/n - mean^2, 0) evaluated in fp32, so even from exact sums it
     carries 3 u (ss/n + mean^2), i.e. u (1 + mean^2/var) relative: that term is part of e(o) in every check.
     Each GroupNorm row is checked twice: *given the statistics* (forward with stats_precomputed = 1, backward with the
     fp64 sums rounded to fp32; the reference uses those same fp32 sums) and *end to end* (the kernel's own sums; the
     reference uses the fp64 sums and e(o) is widened by the statistics bound).  The streaming backward with bf16
     activations uses tanh.approx for SiLU' (2^-12 (1 + |z|) absolute) and parks dz in bf16 between its passes: its bound
     carries those two terms and no other path's does.
     Overwritten outputs start as NaN between NaN guard regions; accumulating outputs are prefilled;
  3. mutants: the predicates reject the fp64 reference edited the way a subtle kernel bug would change it;
  4. plan coverage: pidm_groupnorm_plan (and the LayerNorm grid formula, restated here) show that the rows reach every
     backward path, every cluster size, a ragged last cluster rank on every path, every thread count and grid rule.
"""
import math

import pytest
import torch

from census import assert_census_in_tables, assert_tables_in_census
from checks import (CODE, DTYPES, NAME, RND, U, assert_ok, gen, guarded, guards_intact, note_all, ratio, ratios,
                    rounded, sms)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TAG = 'norm census'
ACT = ('y', 'dx')            # the outputs in the activation type
EPS = float(torch.tensor(1e-5, dtype=torch.float32))      # the entry points take eps as a float
# Both stayed at 1 after a run on an H100 80GB HBM3 (700 W); the worst |err| / bound per kernel path is recorded in
# DESIGN.md section 2.
C_ACC = 1.0
C_EL = 1.0
PATHS = {0: 'fallback', 1: 'piece1', 2: 'piece2', 3: 'packed4', 4: 'stream'}

# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`)
# ----------------------------------------------------------------------------------------------------------------------
# pidm_groupnorm_silu_fwd: B, HW, C, G, scale_shift, residual, stats_precomputed
GN_FWD_TABLE = [
    (16, 64, 128, 8, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 128, 8, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 128, 8, 1, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 256, 8, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 256, 8, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 256, 8, 1, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 256, 64, 8, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 256, 64, 8, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 256, 64, 8, 1, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 256, 128, 8, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 256, 128, 8, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 256, 128, 8, 1, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 1024, 32, 8, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 1024, 32, 8, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 1024, 32, 8, 1, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 1024, 64, 8, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 1024, 64, 8, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 1024, 64, 8, 1, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 4096, 32, 8, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 4096, 32, 8, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 4096, 32, 8, 1, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 64, 128, 8, 0, 0, 1),  # darcy_train_b32
    (32, 64, 128, 8, 0, 1, 1),  # darcy_train_b32
    (32, 64, 128, 8, 1, 0, 1),  # darcy_train_b32
    (32, 64, 256, 8, 0, 0, 1),  # darcy_train_b32
    (32, 64, 256, 8, 0, 1, 1),  # darcy_train_b32
    (32, 64, 256, 8, 1, 0, 1),  # darcy_train_b32
    (32, 64, 512, 8, 0, 0, 1),  # mech_train_b32
    (32, 64, 512, 8, 0, 1, 1),  # mech_train_b32
    (32, 64, 512, 8, 1, 0, 1),  # mech_train_b32
    (32, 64, 1024, 8, 0, 0, 1),  # mech_train_b32
    (32, 64, 1024, 8, 0, 1, 1),  # mech_train_b32
    (32, 64, 1024, 8, 1, 0, 1),  # mech_train_b32
    (32, 256, 64, 8, 0, 0, 1),  # darcy_train_b32
    (32, 256, 64, 8, 0, 1, 1),  # darcy_train_b32
    (32, 256, 64, 8, 1, 0, 1),  # darcy_train_b32
    (32, 256, 128, 8, 0, 0, 1),  # darcy_train_b32
    (32, 256, 128, 8, 0, 1, 1),  # darcy_train_b32
    (32, 256, 128, 8, 1, 0, 1),  # darcy_train_b32
    (32, 256, 256, 8, 0, 0, 1),  # mech_train_b32
    (32, 256, 256, 8, 0, 1, 1),  # mech_train_b32
    (32, 256, 256, 8, 1, 0, 1),  # mech_train_b32
    (32, 256, 512, 8, 0, 0, 1),  # mech_train_b32
    (32, 256, 512, 8, 0, 1, 1),  # mech_train_b32
    (32, 256, 512, 8, 1, 0, 1),  # mech_train_b32
    (32, 1024, 32, 8, 0, 0, 1),  # darcy_train_b32
    (32, 1024, 32, 8, 0, 1, 1),  # darcy_train_b32
    (32, 1024, 32, 8, 1, 0, 1),  # darcy_train_b32
    (32, 1024, 64, 8, 0, 0, 1),  # darcy_train_b32
    (32, 1024, 64, 8, 0, 1, 1),  # darcy_train_b32
    (32, 1024, 64, 8, 1, 0, 1),  # darcy_train_b32
    (32, 1024, 128, 8, 0, 0, 1),  # mech_train_b32
    (32, 1024, 128, 8, 0, 1, 1),  # mech_train_b32
    (32, 1024, 128, 8, 1, 0, 1),  # mech_train_b32
    (32, 1024, 256, 8, 0, 0, 1),  # mech_train_b32
    (32, 1024, 256, 8, 0, 1, 1),  # mech_train_b32
    (32, 1024, 256, 8, 1, 0, 1),  # mech_train_b32
    (32, 4096, 32, 8, 0, 0, 1),  # darcy_train_b32
    (32, 4096, 32, 8, 0, 1, 1),  # darcy_train_b32
    (32, 4096, 32, 8, 1, 0, 1),  # darcy_train_b32
    (32, 4096, 128, 8, 0, 0, 1),  # mech_train_b32
    (32, 4096, 128, 8, 0, 1, 1),  # mech_train_b32
    (32, 4096, 128, 8, 1, 0, 1),  # mech_train_b32
    (64, 64, 128, 8, 0, 0, 1),  # darcy_sample_b64
    (64, 64, 128, 8, 0, 1, 1),  # darcy_sample_b64
    (64, 64, 128, 8, 1, 0, 1),  # darcy_sample_b64
    (64, 64, 256, 8, 0, 0, 1),  # darcy_sample_b64
    (64, 64, 256, 8, 0, 1, 1),  # darcy_sample_b64
    (64, 64, 256, 8, 1, 0, 1),  # darcy_sample_b64
    (64, 256, 64, 8, 0, 0, 1),  # darcy_sample_b64
    (64, 256, 64, 8, 0, 1, 1),  # darcy_sample_b64
    (64, 256, 64, 8, 1, 0, 1),  # darcy_sample_b64
    (64, 256, 128, 8, 0, 0, 1),  # darcy_sample_b64
    (64, 256, 128, 8, 0, 1, 1),  # darcy_sample_b64
    (64, 256, 128, 8, 1, 0, 1),  # darcy_sample_b64
    (64, 1024, 32, 8, 0, 0, 1),  # darcy_sample_b64
    (64, 1024, 32, 8, 0, 1, 1),  # darcy_sample_b64
    (64, 1024, 32, 8, 1, 0, 1),  # darcy_sample_b64
    (64, 1024, 64, 8, 0, 0, 1),  # darcy_sample_b64
    (64, 1024, 64, 8, 0, 1, 1),  # darcy_sample_b64
    (64, 1024, 64, 8, 1, 0, 1),  # darcy_sample_b64
    (64, 4096, 32, 8, 0, 0, 1),  # darcy_sample_b64
    (64, 4096, 32, 8, 0, 1, 1),  # darcy_sample_b64
    (64, 4096, 32, 8, 1, 0, 1),  # darcy_sample_b64
    (256, 64, 128, 8, 0, 0, 1),  # darcy_sample_b256
    (256, 64, 128, 8, 0, 1, 1),  # darcy_sample_b256
    (256, 64, 128, 8, 1, 0, 1),  # darcy_sample_b256
    (256, 64, 256, 8, 0, 0, 1),  # darcy_sample_b256
    (256, 64, 256, 8, 0, 1, 1),  # darcy_sample_b256
    (256, 64, 256, 8, 1, 0, 1),  # darcy_sample_b256
    (256, 256, 64, 8, 0, 0, 1),  # darcy_sample_b256
    (256, 256, 64, 8, 0, 1, 1),  # darcy_sample_b256
    (256, 256, 64, 8, 1, 0, 1),  # darcy_sample_b256
    (256, 256, 128, 8, 0, 0, 1),  # darcy_sample_b256
    (256, 256, 128, 8, 0, 1, 1),  # darcy_sample_b256
    (256, 256, 128, 8, 1, 0, 1),  # darcy_sample_b256
    (256, 1024, 32, 8, 0, 0, 1),  # darcy_sample_b256
    (256, 1024, 32, 8, 0, 1, 1),  # darcy_sample_b256
    (256, 1024, 32, 8, 1, 0, 1),  # darcy_sample_b256
    (256, 1024, 64, 8, 0, 0, 1),  # darcy_sample_b256
    (256, 1024, 64, 8, 0, 1, 1),  # darcy_sample_b256
    (256, 1024, 64, 8, 1, 0, 1),  # darcy_sample_b256
    (256, 4096, 32, 8, 0, 0, 1),  # darcy_sample_b256
    (256, 4096, 32, 8, 0, 1, 1),  # darcy_sample_b256
    (256, 4096, 32, 8, 1, 0, 1),  # darcy_sample_b256
]
# pidm_groupnorm_silu_bwd: B, HW, C, G, scale_shift, d_scale_shift, dbias_of_producer
GN_BWD_TABLE = [
    (32, 64, 128, 8, 0, 0, 1),  # darcy_train_b32
    (32, 64, 128, 8, 1, 1, 1),  # darcy_train_b32
    (32, 64, 256, 8, 0, 0, 1),  # darcy_train_b32
    (32, 64, 256, 8, 1, 1, 1),  # darcy_train_b32
    (32, 64, 512, 8, 0, 0, 1),  # mech_train_b32
    (32, 64, 512, 8, 1, 1, 1),  # mech_train_b32
    (32, 64, 1024, 8, 0, 0, 1),  # mech_train_b32
    (32, 64, 1024, 8, 1, 1, 1),  # mech_train_b32
    (32, 256, 64, 8, 0, 0, 1),  # darcy_train_b32
    (32, 256, 64, 8, 1, 1, 1),  # darcy_train_b32
    (32, 256, 128, 8, 0, 0, 1),  # darcy_train_b32
    (32, 256, 128, 8, 1, 1, 1),  # darcy_train_b32
    (32, 256, 256, 8, 0, 0, 1),  # mech_train_b32
    (32, 256, 256, 8, 1, 1, 1),  # mech_train_b32
    (32, 256, 512, 8, 0, 0, 1),  # mech_train_b32
    (32, 256, 512, 8, 1, 1, 1),  # mech_train_b32
    (32, 1024, 32, 8, 0, 0, 1),  # darcy_train_b32
    (32, 1024, 32, 8, 1, 1, 1),  # darcy_train_b32
    (32, 1024, 64, 8, 0, 0, 1),  # darcy_train_b32
    (32, 1024, 64, 8, 1, 1, 1),  # darcy_train_b32
    (32, 1024, 128, 8, 0, 0, 1),  # mech_train_b32
    (32, 1024, 128, 8, 1, 1, 1),  # mech_train_b32
    (32, 1024, 256, 8, 0, 0, 1),  # mech_train_b32
    (32, 1024, 256, 8, 1, 1, 1),  # mech_train_b32
    (32, 4096, 32, 8, 0, 0, 1),  # darcy_train_b32
    (32, 4096, 32, 8, 1, 1, 1),  # darcy_train_b32
    (32, 4096, 128, 8, 0, 0, 1),  # mech_train_b32
    (32, 4096, 128, 8, 1, 1, 1),  # mech_train_b32
]
# pidm_layernorm_c_fwd: M, C
LN_FWD_TABLE = [
    (1024, 128),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (1024, 256),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (2048, 128),  # darcy_train_b32
    (2048, 256),  # darcy_train_b32
    (2048, 512),  # mech_train_b32
    (2048, 1024),  # mech_train_b32
    (4096, 64),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (4096, 128),  # darcy_sample_b16 darcy_sample_b64 darcy_sample_ddim0_b16
    (4096, 256),  # darcy_sample_b64
    (8192, 64),  # darcy_train_b32
    (8192, 128),  # darcy_train_b32
    (8192, 256),  # mech_train_b32
    (8192, 512),  # mech_train_b32
    (16384, 32),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16384, 64),  # darcy_sample_b16 darcy_sample_b64 darcy_sample_ddim0_b16
    (16384, 128),  # darcy_sample_b256 darcy_sample_b64
    (16384, 256),  # darcy_sample_b256
    (32768, 32),  # darcy_train_b32
    (32768, 64),  # darcy_train_b32
    (32768, 128),  # mech_train_b32
    (32768, 256),  # mech_train_b32
    (65536, 32),  # darcy_sample_b16 darcy_sample_b64 darcy_sample_ddim0_b16
    (65536, 64),  # darcy_sample_b256 darcy_sample_b64
    (65536, 128),  # darcy_sample_b256
    (131072, 32),  # darcy_train_b32
    (131072, 128),  # mech_train_b32
    (262144, 32),  # darcy_sample_b256 darcy_sample_b64
    (262144, 64),  # darcy_sample_b256
    (1048576, 32),  # darcy_sample_b256
]
# pidm_layernorm_c_bwd: M, C, dx_residual
LN_BWD_TABLE = [
    (2048, 128, 1),  # darcy_train_b32
    (2048, 256, 1),  # darcy_train_b32
    (2048, 512, 1),  # mech_train_b32
    (2048, 1024, 1),  # mech_train_b32
    (8192, 64, 1),  # darcy_train_b32
    (8192, 128, 1),  # darcy_train_b32
    (8192, 256, 1),  # mech_train_b32
    (8192, 512, 1),  # mech_train_b32
    (32768, 32, 1),  # darcy_train_b32
    (32768, 64, 1),  # darcy_train_b32
    (32768, 128, 1),  # mech_train_b32
    (32768, 256, 1),  # mech_train_b32
    (131072, 32, 1),  # darcy_train_b32
    (131072, 128, 1),  # mech_train_b32
]
# pidm_colsum: M, C
COLSUM_TABLE = [
    (2048, 128),  # darcy_train_b32
    (2048, 256),  # darcy_train_b32
    (2048, 512),  # mech_train_b32
    (2048, 1024),  # mech_train_b32
    (8192, 64),  # darcy_train_b32
    (8192, 128),  # darcy_train_b32
    (8192, 256),  # mech_train_b32
    (8192, 512),  # mech_train_b32
    (32768, 32),  # darcy_train_b32
    (32768, 64),  # darcy_train_b32
    (32768, 128),  # mech_train_b32
    (32768, 256),  # mech_train_b32
    (131072, 32),  # darcy_train_b32
    (131072, 128),  # mech_train_b32
]
TABLES = {'gn_fwd': GN_FWD_TABLE, 'gn_bwd': GN_BWD_TABLE, 'ln_fwd': LN_FWD_TABLE, 'ln_bwd': LN_BWD_TABLE,
          'colsum': COLSUM_TABLE}

# Rows no benchmarked step produces, for the planner branches the workloads do not reach (see test_plan_coverage; the
# plan of each is in the comment as bf16 | fp32, cl = cluster size, ragged = the last cluster rank owns fewer rows).
GN_SHAPES_SYNTHETIC = [
    (1, 63, 256, 1),      # piece1 cl 8 ragged | fallback (64 vectors per pixel row)
    (1, 144, 32, 8),      # piece1 cl 2 ragged (12 x 12), C/G = 4 | same
    (3, 400, 32, 8),      # piece1 cl 4 ragged (20 x 20), odd batch | same
    (1, 900, 256, 8),     # piece2 cl 8 ragged (30 x 30) | packed4 cl 8 ragged
    (5, 400, 256, 8),     # piece2 cl 4 ragged | packed4 cl 4 ragged
    (32, 900, 64, 8),     # packed4 cl 2 ragged | stream cl 1
    (5, 400, 1024, 8),    # stream cl 4 ragged, odd vector count | stream cl 8 ragged
    (1, 400, 256, 1),     # stream cl 8 ragged, G = 1 | fallback
    (2, 64, 512, 1),      # fallback: 64 (128) vectors per pixel row of the slab
    (1, 33, 256, 1),      # fallback: with cl = 8 a cluster rank would own no pixel
    (1, 16, 32, 8),       # 32 threads, 4 x 4, C/G = 4
    (1, 16, 256, 8),      # 64 threads | 128 threads
    (1, 63, 32, 8),       # 128 threads, HW odd
    (3, 144, 64, 16),     # G = 16, C/G = 4
]
# flag combinations of the pointer arguments on the synthetic shapes: (scale_shift, residual) and
# (scale_shift, d_scale_shift, dbias_of_producer); a shape takes combination number (its index mod the count)
FWD_FLAGS = [(1, 1), (0, 0), (1, 0), (0, 1)]
BWD_FLAGS = [(1, 1, 1), (0, 0, 0), (1, 0, 1), (1, 1, 0), (0, 0, 1)]
GN_FWD_SYNTHETIC = [s + FWD_FLAGS[i % 4] + (0,) for i, s in enumerate(GN_SHAPES_SYNTHETIC)]
GN_BWD_SYNTHETIC = [s + BWD_FLAGS[i % 5] for i, s in enumerate(GN_SHAPES_SYNTHETIC)]
# LayerNorm: M = 1, one short of, equal to and one past a row group, and a capped grid with a ragged tail, for the
# register kernel (C = 32, 128, 256) and the looping one (C = 512, 1024)
LN_SHAPES_SYNTHETIC = [(1, 32), (255, 32), (256, 32), (257, 32), (300001, 32), (1, 128), (63, 128), (65, 128),
                       (70001, 128), (1, 256), (31, 256), (33, 256), (40001, 256), (1, 512), (7, 512), (8, 512),
                       (9, 512), (9001, 512), (1, 1024), (7, 1024), (9, 1024), (9001, 1024)]
LN_FWD_SYNTHETIC = list(LN_SHAPES_SYNTHETIC)
LN_BWD_SYNTHETIC = [s + (i % 2,) for i, s in enumerate(LN_SHAPES_SYNTHETIC)]
COLSUM_SYNTHETIC = [(1, 32), (4099, 32), (1, 256), (70001, 128)]

GN_FWD_ROWS = GN_FWD_TABLE + GN_FWD_SYNTHETIC
GN_BWD_ROWS = GN_BWD_TABLE + GN_BWD_SYNTHETIC
LN_FWD_ROWS = LN_FWD_TABLE + LN_FWD_SYNTHETIC
LN_BWD_ROWS = LN_BWD_TABLE + LN_BWD_SYNTHETIC
COLSUM_ROWS = COLSUM_TABLE + COLSUM_SYNTHETIC


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
def plan_gn(B, HW, C, G, dtype):
    from physicsinformeddiffusionmodels_b200._lib import call
    out = torch.zeros(10, dtype=torch.int32)
    rc = call('pidm_groupnorm_plan', B, HW, C, G, CODE[dtype], out.data_ptr())
    assert rc == 0, f'groupnorm rejects B={B} HW={HW} C={C} G={G} {NAME[dtype]}'
    v = out.tolist()
    return dict(stats_chunks=v[0], stats_block=v[1], apply_chunks=v[2], rules=v[3], path=v[4], S=v[5], threads=v[6],
                cl=v[7], rows_per_cta=v[8], v=v[9])


def plan_ln(M, C, bwd):
    """pidm_layernorm_c_{fwd,bwd} restated: a group of L lanes owns a row, a CTA has 8 warps; the register kernel
    (C/8 a power of two <= 32) keeps 4 rows per group in flight; the grid is capped at 8 (4) CTAs per SM and loops"""
    oct_, L = C // 8, 1
    while L < 32 and L < oct_:
        L *= 2
    reg = L == oct_
    rows = (32 // L) * 8 * (4 if reg else 1)            # rows per CTA and iteration
    want, cap = max(1, -(-M // rows)), sms() * (4 if bwd else 8)
    grid = min(want, cap)
    return dict(kernel='ln1' if reg else 'ln', capped=want > cap, ragged=M % (grid * rows) != 0, grid=grid, rows=rows)


# ----------------------------------------------------------------------------------------------------------------------
# operands, references, bounds
# ----------------------------------------------------------------------------------------------------------------------
def _randn(g, *shape, dtype=torch.float32):
    return torch.randn(*shape, generator=g, device=DEV).to(dtype)


def _silu_terms(z, e_z):
    """sigmoid, SiLU', and the error bounds of SiLU and SiLU' as the kernels evaluate them in fp32 from a z that is off by
    e_z: Taylor in e_z (|SiLU''| <= 1/2) plus the fast exponential.  With --use_fast_math exp(-z) is
    ex2.approx of the rounded product -z log2(e): relative error (2 + 1.5 |z|) u, which moves sigmoid by at most
    s (1 - s) times that, and the division is approximate (2 ulp).  u (8 + 2 |z|) relative covers SiLU, and
    u (8 + 3 |z|) times the absolute-value evaluation s (1 + |z| (1 - s)) covers SiLU'."""
    s = torch.sigmoid(z)
    d = s * (1 + z * (1 - s))
    e_silu = (d.abs() + 0.25 * e_z) * e_z + U * (8 + 2 * z.abs()) * (z * s).abs()     # second order: SiLU' has a zero
    e_d = 0.5 * e_z + U * (8 + 3 * z.abs()) * s * (1 + z.abs() * (1 - s))
    return s, d, e_silu, e_d


def _moments_err(mean, E2, var, e_s_n, e_ss_n):
    """relative error bound of rstd = 1/sqrt(var + eps) when mean = s/n and var = max(ss/n - mean^2, 0) are evaluated in
    fp32 from sums that are off by e_s_n * n and e_ss_n * n (worst case over the interval, not first order: a constant
    group has var = 0 and an error of the order of eps)"""
    e_var = e_ss_n + 2 * mean.abs() * e_s_n + 3 * U * (E2 + mean * mean)
    up = ((var + EPS) / ((var - e_var).clamp_min(0) + EPS)).sqrt() - 1
    down = 1 - ((var + EPS) / (var + e_var + EPS)).sqrt()
    return torch.maximum(up, down) + 4 * U


class GnCase:
    """operands of one GroupNorm shape and activation type; eval() gives the fp64 reference and the bounds"""

    def __init__(self, B, HW, C, G, dtype, ss=1, res=0, m_over_sigma=None, constant_group=False):
        self.shape, self.dtype = (B, HW, C, G), dtype
        g = gen(('gn', B, HW, C, G, m_over_sigma))
        if m_over_sigma is None:
            x = torch.randn(B, HW, C, generator=g, device=DEV) * 1.5 + 0.3
        else:
            x = torch.randn(B, HW, C, generator=g, device=DEV) + float(m_over_sigma)
        if constant_group:
            x[0, :, :C // G] = 2.0
        self.x = x.to(dtype)
        self.dy = _randn(g, B, HW, C, dtype=dtype)
        self.gamma = 1 + 0.2 * _randn(g, C)
        self.beta = 0.1 * _randn(g, C)
        self.ss = 0.3 * _randn(g, B, 2 * C) if ss else None
        self.res = _randn(g, B, HW, C, dtype=dtype) if res else None
        self.pre = {k: _randn(g, C) for k in ('dgamma', 'dbeta', 'dbias')}
        cpg = C // G
        xg = self.x.double().view(B, HW, G, cpg)
        self.n = HW * cpg
        self.sums = torch.stack((xg.sum(dim=(1, 3)), (xg * xg).sum(dim=(1, 3))), dim=-1)          # fp64 [B, G, 2]
        acc = C_ACC * math.sqrt(self.n) * U
        self.e_sums = torch.stack((acc * xg.abs().sum(dim=(1, 3)), (acc + U) * self.sums[..., 1]), dim=-1)

    def plan(self):
        return plan_gn(*self.shape, self.dtype)

    def eval(self, sums, end_to_end, backward=True, dss=1, dbias=1, mut=()):
        """(reference, bound) dictionaries of y (and dx, dgamma, dbeta, dss, dbias) from the statistics `sums` [B,G,2].
        end_to_end: the kernels start from their own sums, which are within e_sums of `sums`.  mut: edits of the
        reference (see the mutant tests)."""
        B, HW, C, G = self.shape
        cpg, n, rnd = C // G, self.n, RND[self.dtype]
        per_c = lambda t: t.double().view(1, 1, G, cpg)
        per_bc = lambda t: t.double().view(B, 1, G, cpg)
        x = self.x.double().view(B, HW, G, cpg)
        s, q = (sums[..., i].double().view(B, 1, G, 1) for i in (0, 1))
        e_s_n, e_ss_n = ((self.e_sums[..., i].view(B, 1, G, 1) / n if end_to_end else 0.0) for i in (0, 1))
        mean, E2 = s / n, q / n
        if 'variance over n - 1' in mut:
            var = ((q - n * mean * mean) / (n - 1)).clamp_min(0)
        else:
            var = (E2 - mean * mean).clamp_min(0)
        rstd = (var + EPS).rsqrt()
        gam, bet = per_c(self.gamma), per_c(self.beta)
        one = torch.ones(1, 1, 1, 1, dtype=torch.float64, device=x.device)
        f = per_bc(self.ss[:, :C]) + (0 if 'scale + 1 applied as scale' in mut else 1) if self.ss is not None else one
        sh = per_bc(self.ss[:, C:]) if self.ss is not None else 0 * one
        res = self.res.double().view(B, HW, G, cpg) if self.res is not None else 0 * one
        xh = (x - mean) * rstd
        z = (xh * gam + bet) * f + sh
        r_rel = _moments_err(mean, E2, var, e_s_n, e_ss_n)
        e_xh = rstd * e_s_n + 3 * U * (x.abs() + mean.abs()) * rstd + xh.abs() * r_rel
        gf = (gam * f).abs()
        e_z = e_xh * gf + 3 * U * ((xh * gam * f).abs() + (bet * f).abs() + sh.abs())
        sg, dsilu, e_silu, e_dsilu = _silu_terms(z, e_z)
        y0 = z * sg
        r = {'y': (y0 + (0 if 'residual missing' in mut else res)).reshape(B, HW, C)}
        b = {'y': (rnd * (y0 + res).abs() + C_EL * (e_silu + U * (y0.abs() + res.abs()))).reshape(B, HW, C)}
        if not backward:
            return r, b
        pl = self.plan()
        tanh_path = self.dtype == torch.bfloat16 and pl['path'] == 4
        if tanh_path:
            e_dsilu = e_dsilu + 2.0 ** -12 * (1 + z.abs())
        dy = self.dy.double().view(B, HW, G, cpg)
        dz = dy * dsilu
        e_dz = dy.abs() * e_dsilu + U * dz.abs()
        acc, accB = C_ACC * math.sqrt(HW) * U, C_ACC * math.sqrt(B * HW) * U
        psum = lambda t: t.sum(dim=1, keepdim=True)
        s1, s2, a1, a2 = psum(dz), psum(dz * xh), psum(dz.abs()), psum((dz * xh).abs())
        e_s1 = psum(e_dz) + acc * a1
        e_s2 = psum(e_dz * xh.abs() + dz.abs() * e_xh + U * (dz * xh).abs()) + acc * a2
        pre = {k: v.double() for k, v in self.pre.items()}
        chan = lambda t: t.sum(dim=0).reshape(C)
        r['dgamma'] = pre['dgamma'] + chan(f * s2)
        r['dbeta'] = (0 if 'dbeta overwritten' in mut else pre['dbeta']) + chan(f * s1)
        if 'one channel slab missing from dgamma' in mut:
            S = pl['S']
            r['dgamma'][S:2 * S] = pre['dgamma'][S:2 * S]
        b['dgamma'] = C_EL * chan(f.abs() * e_s2) + accB * (pre['dgamma'].abs() + chan(f.abs() * a2))
        b['dbeta'] = C_EL * chan(f.abs() * e_s1) + accB * (pre['dbeta'].abs() + chan(f.abs() * a1))
        if self.ss is not None and dss:
            r['dss'] = torch.cat(((gam * s2 + bet * s1).reshape(B, C), (s1 + 0 * gam).reshape(B, C)), dim=1)
            e_dsc = gam.abs() * e_s2 + bet.abs() * e_s1 + 2 * U * ((gam * s2).abs() + (bet * s1).abs())
            b['dss'] = C_EL * torch.cat((e_dsc.reshape(B, C), (e_s1 + 0 * gam).reshape(B, C)), dim=1)
        # group means of gamma (1 + scale) dz and of gamma (1 + scale) dz xhat
        s1m, s2m = s1, s2
        if 'last cluster rank missing from the group sums' in mut:
            rows = (pl['cl'] - 1) * pl['rows_per_cta']
            s1m, s2m = psum(dz[:, :rows]), psum((dz * xh)[:, :rows])
        gsum = lambda t: t.sum(dim=3, keepdim=True)
        m1, m2 = gsum(gam * f * s1m) / n, gsum(gam * f * s2m) / n
        cacc = (math.sqrt(cpg) + 4) * U
        e_m1 = gsum(gf * e_s1) / n + cacc * gsum(gf * a1) / n
        e_m2 = gsum(gf * e_s2) / n + cacc * gsum(gf * a2) / n
        dx = rstd * (gam * f * dz - m1 - xh * m2)
        e_core = (gf * e_dz + e_m1 + xh.abs() * e_m2 + m2.abs() * e_xh
                  + 3 * U * (gf * dz.abs() + m1.abs() + (xh * m2).abs()))
        e_dx = rstd * e_core + (r_rel + 2 * U) * dx.abs()
        e_park = rstd * gf * 2.0 ** -8 * dz.abs() if tanh_path else 0 * one      # dz parked in bf16 between the passes
        r['dx'] = dx.reshape(B, HW, C)
        b['dx'] = (rnd * dx.abs() + C_EL * (e_dx + e_park)).reshape(B, HW, C)
        if dbias:
            bsum = lambda t: (t + 0 * dx).sum(dim=(0, 1)).reshape(C)
            r['dbias'] = pre['dbias'] + bsum(dx)
            if 'one sample missing from dbias' in mut:
                r['dbias'] = r['dbias'] - dx[-1].sum(dim=0).reshape(C)
            # the column sums are taken before the output rounding; the parking roundings are independent: root sum square
            b['dbias'] = (C_EL * (bsum(e_dx) + 4 * bsum(e_park * e_park).sqrt())
                          + accB * (pre['dbias'].abs() + bsum(dx.abs())))
        return r, b

    # ---- launches -----------------------------------------------------------------------------------------------------
    def run_fwd(self, sums_in):
        """forward through the C ABI; sums_in (fp32 [B,G,2]) = stats_precomputed, None = the kernel's own statistics"""
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, HW, C, G = self.shape
        ybuf, y = guarded(B * HW * C, self.dtype)
        sbuf, sums = guarded(B * G * 2)
        if sums_in is not None:
            sums.copy_(sums_in.reshape(-1))
        call('pidm_groupnorm_silu_fwd', self.x, self.gamma, self.beta, self.ss, self.res, y, sums,
             0 if sums_in is None else 1, B, HW, C, G, EPS, CODE[self.dtype], stream())
        torch.cuda.synchronize()
        return {'y': y.view(B, HW, C)}, sums.view(B, G, 2), guards_intact(ybuf) and guards_intact(sbuf)

    def run_bwd(self, sums, dss=1, dbias=1):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, HW, C, G = self.shape
        bufs = {'dx': guarded(B * HW * C, self.dtype), 'ws': guarded(B * C * 2)}
        if self.ss is not None and dss:
            bufs['dss'] = guarded(B * 2 * C)
        for k in ('dgamma', 'dbeta') + (('dbias',) if dbias else ()):
            bufs[k] = guarded(C)
            bufs[k][1].copy_(self.pre[k])
        v = lambda k: bufs[k][1] if k in bufs else None
        call('pidm_groupnorm_silu_bwd', self.x, self.dy, sums.contiguous(), self.gamma, self.beta, self.ss, v('dx'),
             v('dgamma'), v('dbeta'), v('dss'), v('dbias'), v('ws'), B, HW, C, G, EPS, CODE[self.dtype], stream())
        torch.cuda.synchronize()
        out = {k: t[1] for k, t in bufs.items() if k != 'ws'}
        out['dx'] = out['dx'].view(B, HW, C)
        if 'dss' in out:
            out['dss'] = out['dss'].view(B, 2 * C)
        return out, all(guards_intact(t[0]) for t in bufs.values())


class LnCase:
    def __init__(self, M, C, dtype, res=0):
        self.M, self.C, self.dtype = M, C, dtype
        g = gen(('ln', M, C))
        self.x = (torch.randn(M, C, generator=g, device=DEV) * 2 + 0.5).to(dtype)
        self.dy = _randn(g, M, C, dtype=dtype)
        self.gamma = 1 + 0.2 * _randn(g, C)
        self.res = _randn(g, M, C, dtype=dtype) if res else None
        self.pre = _randn(g, C)

    def eval(self, backward, mut=()):
        """fp64 y = (x - mean) rstd gamma per row (biased variance, clamped at 0) and its gradients, with the bounds"""
        M, C, rnd = self.M, self.C, RND[self.dtype]
        x, gam = self.x.double(), self.gamma.double()
        rsum = lambda t: t.sum(dim=1, keepdim=True)
        acc = (C_ACC * math.sqrt(C) + 2) * U
        mean, E2 = rsum(x) / C, rsum(x * x) / C
        var = (E2 - mean * mean).clamp_min(0)
        rstd = (var + EPS).rsqrt()
        e_s_n, e_ss_n = acc * rsum(x.abs()) / C, acc * E2
        r_rel = _moments_err(mean, E2, var, e_s_n, e_ss_n)
        xh = (x - mean) * rstd
        e_xh = rstd * e_s_n + 3 * U * (x.abs() + mean.abs()) * rstd + xh.abs() * r_rel
        y = xh * gam
        if not backward:
            r = {'y': y}
            if 'last row taken from the previous row' in mut:
                r['y'] = torch.cat((y[:-1], y[-2:-1]))
            return r, {'y': rnd * y.abs() + C_EL * (gam.abs() * e_xh + 2 * U * y.abs())}
        dy = self.dy.double()
        res = self.res.double() if self.res is not None else torch.zeros(1, 1, dtype=torch.float64, device=x.device)
        dxh = dy * gam
        a, bb = rsum(dxh) / C, rsum(dxh * xh) / C
        e_a = acc * rsum(dxh.abs()) / C
        e_b = rsum(dxh.abs() * e_xh) / C + acc * rsum((dxh * xh).abs()) / C
        core = dxh - a - xh * bb
        e_core = e_a + xh.abs() * e_b + bb.abs() * e_xh + 3 * U * (dxh.abs() + a.abs() + (xh * bb).abs())
        dx0 = rstd * core
        e_dx = rstd * e_core + (r_rel + 2 * U) * dx0.abs() + U * (dx0.abs() + res.abs())
        pre = self.pre.double()
        r = {'dx': dx0 + (0 if 'dx_residual missing' in mut else res), 'dgamma': pre + (dy * xh).sum(dim=0)}
        b = {'dx': rnd * (dx0 + res).abs() + C_EL * e_dx,
             'dgamma': C_EL * (dy.abs() * e_xh + U * (dy * xh).abs()).sum(dim=0)
             + C_ACC * math.sqrt(M) * U * (pre.abs() + (dy * xh).abs().sum(dim=0))}
        return r, b

    def run(self, backward):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        M, C = self.M, self.C
        obuf, o = guarded(M * C, self.dtype)
        if not backward:
            call('pidm_layernorm_c_fwd', self.x, self.gamma, o, M, C, EPS, CODE[self.dtype], stream())
            torch.cuda.synchronize()
            return {'y': o.view(M, C)}, guards_intact(obuf)
        gbuf, dg = guarded(C)
        dg.copy_(self.pre)
        call('pidm_layernorm_c_bwd', self.x, self.dy, self.gamma, o, dg, self.res, M, C, EPS, CODE[self.dtype], stream())
        torch.cuda.synchronize()
        return {'dx': o.view(M, C), 'dgamma': dg}, guards_intact(obuf) and guards_intact(gbuf)


# ----------------------------------------------------------------------------------------------------------------------
# replay
# ----------------------------------------------------------------------------------------------------------------------
def _check_stats(c, sums, where):
    rs = {'sum': ratio((sums[..., 0].double() - c.sums[..., 0]).abs(), c.e_sums[..., 0]),
          'sum of squares': ratio((sums[..., 1].double() - c.sums[..., 1]).abs(), c.e_sums[..., 1])}
    note_all(TAG, f'gn_stats {NAME[c.dtype]}', rs)
    assert_ok(rs, where + ' statistics')


def replay_gn_fwd(c, where):
    given = c.sums.float()
    out, _, ok = c.run_fwd(given)
    assert ok, f'{where}: a store landed outside y or the sums'
    rs = ratios(out, *c.eval(given, end_to_end=False, backward=False))
    note_all(TAG, f'gn_apply {NAME[c.dtype]} given statistics', rs)
    assert_ok(rs, where + ' given the statistics')
    out, sums, ok = c.run_fwd(None)
    assert ok, f'{where}: a store landed outside y or the sums'
    _check_stats(c, sums, where)
    rs = ratios(out, *c.eval(c.sums, end_to_end=True, backward=False))
    note_all(TAG, f'gn_apply {NAME[c.dtype]} end to end', rs)
    assert_ok(rs, where + ' end to end')
    return out, sums


def replay_gn_bwd(c, dss, dbias, where):
    path = PATHS[c.plan()['path']]
    given = c.sums.float()
    out, ok = c.run_bwd(given, dss, dbias)
    assert ok, f'{where}: a store landed outside the outputs'
    r, b = c.eval(given, end_to_end=False, dss=dss, dbias=dbias)
    del r['y']
    rs = ratios(out, r, b)
    note_all(TAG, f'gn_bwd {path} {NAME[c.dtype]} given statistics', rs)
    assert_ok(rs, f'{where} given the statistics (plan {c.plan()})')
    _, sums, _ = c.run_fwd(None)
    out, ok = c.run_bwd(sums, dss, dbias)
    assert ok, f'{where}: a store landed outside the outputs'
    r, b = c.eval(c.sums, end_to_end=True, dss=dss, dbias=dbias)
    del r['y']
    rs = ratios(out, r, b)
    note_all(TAG, f'gn_bwd {path} {NAME[c.dtype]} end to end', rs)
    assert_ok(rs, f'{where} end to end (plan {c.plan()})')
    return out


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', GN_FWD_ROWS, ids=_id)
def test_groupnorm_fwd_replay(k, dtype):
    B, HW, C, G, ss, res, _ = k
    replay_gn_fwd(GnCase(B, HW, C, G, dtype, ss, res), f'gn_fwd {k} {NAME[dtype]}')


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', GN_BWD_ROWS, ids=_id)
def test_groupnorm_bwd_replay(k, dtype):
    B, HW, C, G, ss, dss, dbias = k
    replay_gn_bwd(GnCase(B, HW, C, G, dtype, ss), dss, dbias, f'gn_bwd {k} {NAME[dtype]}')


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', LN_FWD_ROWS, ids=_id)
def test_layernorm_fwd_replay(k, dtype):
    c = LnCase(*k, dtype)
    out, ok = c.run(False)
    assert ok, f'ln_fwd {k}: a store landed outside y'
    rs = ratios(out, *c.eval(False))
    note_all(TAG, f'{plan_ln(*k, False)["kernel"]}_fwd {NAME[dtype]}', rs)
    assert_ok(rs, f'ln_fwd {k} {NAME[dtype]} (plan {plan_ln(*k, False)})')


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', LN_BWD_ROWS, ids=_id)
def test_layernorm_bwd_replay(k, dtype):
    M, C, res = k
    c = LnCase(M, C, dtype, res)
    out, ok = c.run(True)
    assert ok, f'ln_bwd {k}: a store landed outside dx or dgamma'
    rs = ratios(out, *c.eval(True))
    note_all(TAG, f'{plan_ln(M, C, True)["kernel"]}_bwd {NAME[dtype]}', rs)
    assert_ok(rs, f'ln_bwd {k} {NAME[dtype]} (plan {plan_ln(M, C, True)})')


def colsum_eval(x, pre, M):
    xd = x.double()
    return ({'colsum': pre.double() + xd.sum(dim=0)},
            {'colsum': C_ACC * math.sqrt(M) * U * (pre.double().abs() + xd.abs().sum(dim=0))})


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('k', COLSUM_ROWS, ids=_id)
def test_colsum_replay(k, dtype):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    M, C = k
    g = gen(('colsum', M, C))
    x, pre = _randn(g, M, C, dtype=dtype), _randn(g, C)
    buf, out = guarded(C)
    out.copy_(pre)
    call('pidm_colsum', x, out, M, C, CODE[dtype], stream())
    torch.cuda.synchronize()
    assert guards_intact(buf), f'colsum {k}: a store landed outside the output'
    rs = ratios({'colsum': out}, *colsum_eval(x, pre, M))
    note_all(TAG, f'colsum {NAME[dtype]}', rs)
    assert_ok(rs, f'colsum {k} {NAME[dtype]}')


# ----------------------------------------------------------------------------------------------------------------------
# conditioning: groups whose mean is far from zero, and a constant group
# ----------------------------------------------------------------------------------------------------------------------
COND_SHAPE = (4, 1024, 64, 8)


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
@pytest.mark.parametrize('m_over_sigma', [0, 8, 64])
def test_groupnorm_conditioning(m_over_sigma, dtype):
    """x = m + z: the variance loses a factor kappa = 1 + (m / sigma)^2 of accuracy (sum of squares minus squared mean
    in fp32) and the bound follows it, so the assertion is that the kernels lose no more than the formula in pidm.h
    must.  The worst absolute error of y is printed; DESIGN.md section 2 records it."""
    c = GnCase(*COND_SHAPE, dtype, ss=1, m_over_sigma=m_over_sigma)
    where = f'm/sigma = {m_over_sigma} {NAME[dtype]}'
    out, _ = replay_gn_fwd(c, where)
    r, _ = c.eval(c.sums, end_to_end=True, backward=False)
    err = (out['y'].double() - r['y']).abs()
    rounding = RND[dtype] * r['y'].abs()
    print(f'[norm census] conditioning {where}: max |y - r| = {err.max().item():.3g}, beyond the output rounding '
          f'{(err - rounding).clamp_min(0).max().item():.3g} (max |r| = {r["y"].abs().max().item():.3g})')
    replay_gn_bwd(c, 1, 1, where)


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_groupnorm_constant_group(dtype):
    """a group that is one constant has var = 0: rstd = 1/sqrt(eps), xhat = 0, y = silu(beta (1 + scale) + shift), and dx
    is rstd times the mean-free part of gamma (1 + scale) dz; all finite and inside the same bounds"""
    c = GnCase(*COND_SHAPE, dtype, ss=1, constant_group=True)
    out, sums = replay_gn_fwd(c, f'constant group {NAME[dtype]}')
    assert sums[0, 0, 0].item() == 2.0 * c.n and sums[0, 0, 1].item() == 4.0 * c.n
    dout = replay_gn_bwd(c, 1, 1, f'constant group {NAME[dtype]}')
    assert torch.isfinite(out['y']).all() and torch.isfinite(dout['dx']).all()
    r, _ = c.eval(c.sums, end_to_end=False)
    cpg = c.shape[2] // c.shape[3]
    assert r['dx'][0, :, :cpg].abs().max().item() > 10.0          # rstd = 316: the group's dx is large, not suppressed


# ----------------------------------------------------------------------------------------------------------------------
# the predicates reject subtly wrong outputs (edits of the fp64 reference; no faulty code runs on the GPU)
# ----------------------------------------------------------------------------------------------------------------------
def _gn_mutant(shape, dtype, mutation, output, ss=1, res=0):
    c = GnCase(*shape, dtype, ss, res)
    sums = c.sums.float()
    r, b = c.eval(sums, end_to_end=False)
    assert max(ratios(rounded(r, dtype, ACT), r, b).values()) <= 1.0
    m, _ = c.eval(sums, end_to_end=False, mut=(mutation,))
    return ratios(rounded(m, dtype, ACT), r, b)[output]


def test_mutant_variance_over_n_minus_1():
    """n = 64 * 4: the unbiased variance moves rstd by 1 / (2n) = 2e-3.  fp32 activations see it in y and dx.  With bf16
    activations 2e-3 is half of the output rounding 2^-8, so y and dx cannot be relied on to see it; the fp32 parameter
    gradients do"""
    shape = (2, 64, 32, 8)
    assert _gn_mutant(shape, torch.float32, 'variance over n - 1', 'y') > 1.0
    assert _gn_mutant(shape, torch.float32, 'variance over n - 1', 'dx') > 1.0
    assert _gn_mutant(shape, torch.bfloat16, 'variance over n - 1', 'dgamma') > 1.0


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_mutant_last_cluster_rank_missing_from_the_group_sums(dtype):
    hit = set()
    for shape in GN_SHAPES_SYNTHETIC:
        p = plan_gn(*shape, dtype)
        if p['cl'] > 1 and p['rows_per_cta'] * p['cl'] > shape[1] and p['path'] not in hit:
            hit.add(p['path'])
            assert _gn_mutant(shape, dtype, 'last cluster rank missing from the group sums', 'dx') > 1.0, (shape, p)
    assert len(hit) >= 3, hit


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_mutant_groupnorm_terms(dtype):
    shape = (5, 400, 256, 8)
    assert _gn_mutant(shape, dtype, 'one channel slab missing from dgamma', 'dgamma') > 1.0
    assert _gn_mutant(shape, dtype, 'scale + 1 applied as scale', 'y') > 1.0
    assert _gn_mutant(shape, dtype, 'residual missing', 'y', res=1) > 1.0
    assert _gn_mutant(shape, dtype, 'one sample missing from dbias', 'dbias') > 1.0
    assert _gn_mutant(shape, dtype, 'dbeta overwritten', 'dbeta') > 1.0


@pytest.mark.parametrize('dtype', DTYPES, ids=NAME.get)
def test_mutant_layernorm(dtype):
    c = LnCase(257, 32, dtype)
    r, b = c.eval(False)
    assert max(ratios(rounded(r, dtype, ACT), r, b).values()) <= 1.0
    m, _ = c.eval(False, mut=('last row taken from the previous row',))
    assert ratios(rounded(m, dtype, ACT), r, b)['y'] > 1.0
    c = LnCase(257, 32, dtype, res=1)
    r, b = c.eval(True)
    assert max(ratios(rounded(r, dtype, ACT), r, b).values()) <= 1.0
    m, _ = c.eval(True, mut=('dx_residual missing',))
    assert ratios(rounded(m, dtype, ACT), r, b)['dx'] > 1.0


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
def gn_coverage():
    bwd = [(k, dt, plan_gn(*k[:4], dt)) for k in GN_BWD_ROWS for dt in DTYPES]
    fwd = [(k, dt, plan_gn(*k[:4], dt)) for k in GN_FWD_ROWS for dt in DTYPES]
    ragged = lambda k, p: p['cl'] > 1 and p['rows_per_cta'] * p['cl'] > k[1]
    rpp = lambda k, dt: 256 // (k[2] // (8 if dt == torch.bfloat16 else 4))       # pixel rows of one apply CTA pass
    return {
        'backward path': {p['path'] for _, _, p in bwd},
        'cluster size': {p['cl'] for _, _, p in bwd if p['path']},
        'cluster size (bf16)': {p['cl'] for _, dt, p in bwd if p['path'] and dt == torch.bfloat16},
        'ragged last rank on path': {p['path'] for k, _, p in bwd if ragged(k, p)},
        'threads': {p['threads'] for _, _, p in bwd if p['path']},
        'channels per group': {k[2] // k[3] for k, _, _ in bwd},
        'groups': {k[3] for k, _, _ in bwd},
        'apply grid rules': {bit for _, _, p in fwd for bit in (1, 2, 4) if p['rules'] & bit},
        'no apply grid rule': any(p['rules'] == 0 for _, _, p in fwd),
        'apply grid does not divide HW': any(k[1] % (p['apply_chunks'] * rpp(k, dt)) for k, dt, p in fwd),
        'fwd flags': {k[4:] for k in GN_FWD_ROWS},
        'bwd flags': {k[4:] for k in GN_BWD_ROWS},
    }


def ln_coverage():
    out = {}
    for name, rows, bwd in (('fwd', LN_FWD_ROWS, False), ('bwd', LN_BWD_ROWS, True)):
        plans = [plan_ln(k[0], k[1], bwd) for k in rows]
        out[name] = {(p['kernel'], p['capped'], p['ragged']) for p in plans}
    out['dx_residual'] = {k[2] for k in LN_BWD_ROWS}
    return out


def test_plan_coverage():
    cv = gn_coverage()
    print(f'[norm census] groupnorm coverage {cv}')
    assert cv['backward path'] == {0, 1, 2, 3, 4}, cv
    assert cv['cluster size'] == {1, 2, 4, 8} and 8 in cv['cluster size (bf16)'], cv
    assert cv['ragged last rank on path'] == {1, 2, 3, 4}, cv
    assert cv['threads'] >= {256, 128, 64}, cv
    assert 4 in cv['channels per group'] and cv['groups'] - {8}, cv
    assert cv['apply grid rules'] == {1, 2, 4} and cv['no apply grid rule'] and cv['apply grid does not divide HW'], cv
    assert cv['fwd flags'] >= {(a, b, 0) for a in (0, 1) for b in (0, 1)} and any(k[2] for k in cv['fwd flags']), cv
    assert {k[0] for k in cv['bwd flags']} == {0, 1} and {k[1] for k in cv['bwd flags']} == {0, 1}, cv
    assert {k[2] for k in cv['bwd flags']} == {0, 1}, cv


def test_layernorm_plan_coverage():
    cv = ln_coverage()
    print(f'[norm census] layernorm coverage {cv}')
    for name in ('fwd', 'bwd'):
        for kernel in ('ln1', 'ln'):
            assert {(c, r) for k, c, r in cv[name] if k == kernel} >= {(False, True), (True, True)}, (name, kernel, cv)
            assert any(not r for k, c, r in cv[name] if k == kernel), (name, kernel, 'even tail', cv)
    assert cv['dx_residual'] == {0, 1}, cv


def test_rejected_shapes_are_refused_before_any_launch():
    from physicsinformeddiffusionmodels_b200._lib import call
    out = torch.zeros(10, dtype=torch.int32)
    for B, HW, C, G, code in ((1, 16, 24, 2, 1), (1, 16, 36, 4, 1), (1, 16, 32, 3, 1), (1, 16, 4096, 8, 0)):
        assert call('pidm_groupnorm_plan', B, HW, C, G, code, out.data_ptr()) != 0, (B, HW, C, G, code)

