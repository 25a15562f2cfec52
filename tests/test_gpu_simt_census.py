"""Every CUDA-core convolution launch of the fp32 exact mode, replayed element by element against an fp64 reference.

In the exact mode (`ops.set_precision('fp32')`), which every oracle-parity test runs, each convolution, dgrad and
ConvTranspose layer of the U-Net runs on pidm_conv2d_simt and each convolution weight and bias gradient on
pidm_conv2d_wgrad_simt (conv_simt.cu): the fp32 references the tensor-core kernels are judged against rest on them.  The
forward tiles M x N x K by 64 x 64 x 16, gathers regular, transposed (th % stride parity classes) and halo'd (circular)
geometries, and adds bias and residual in its epilogue; the weight gradient splits M by a rule of the SM count, rounds
the split to 16 pixels, adds the bias gradient from K tile 0 of each split, masks the padded stem channels and
accumulates through strides into either weight layout with atomics.  test_gpu_ops.py::test_conv_simt compares whole
tensors by a norm ratio at six small geometries, which a bug confined to one tile row or one split cannot move.  Here,
in the four parts of the other census files:

  1. census: the distinct keys of both entry points in one eager fp32 step of every workload bench.py times, of the
     guidance and circular Darcy training steps and of the circular mechanics U-Net (census.census_exact()) must equal
     the tables below (`python tests/census.py --print-table` regenerates them); one more test checks that every entry
     point the exact mode calls is checked per element somewhere;
  2. replay: every table row plus synthetic rows, through the C ABI, with bf16 and with fp32 activations, on seeded
     operands, against the fp64 evaluation of the pidm.h contract (checks.conv_ref; the weight gradient is its fp64
     gradient with respect to Wp, scattered to n*s_n + c*s_c + tap for c < Cin_real), per element.  With u = 2^-24 and
     A the same operation on absolute values (bias and residual included):
        forward, fp32 activations   |y - r| <= C_FWD (sqrt(K) + 2) u A        products, sum, two epilogue adds
        forward, bf16 activations   |y - r| <= 2^-8 |r| + C_FWD sqrt(K) u A   the products are exact
        dw, dbias                   |d - prefill - r| <= C_WG sqrt(M) u A + splits u (|prefill| + A),   M = B Ho Wo
     y sits between NaN guard regions; dw and dbias are prefilled buffers whose every element outside the contract
     (guards, padded stem channels) must keep its value -- a NaN guard cannot see a stray atomic add;
  3. mutants: the same predicates reject the fp64 reference edited the way a subtle kernel bug would change it;
  4. plan coverage: the grid and split arithmetic of conv_simt.cu, restated below, shows that the rows reach ragged M, N
     and K tiles, every split rule, every gather kind, 1x1 / 3x3 / 4x4 / 7x7 taps, the halo geometries and both weight
     layouts.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from census import assert_census_in_tables, assert_checked_or_listed, assert_tables_in_census, census_exact
from checks import CODE, DTYPES, NAME, U, call_sync, conv_ref, gen, guarded, guards_intact, note, ratio, sms

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TAG = 'simt census'
# Both stayed at 1 after a run on an H100 80GB HBM3 (700 W): the worst |err| / bound was 0.93 for the fp32 forward (the
# 1x1, K = 32 layer at B = 256, 805 M outputs) and 0.38 for dw; DESIGN.md section 2 records the rest.
C_FWD = 1.0
C_WG = 1.0

# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`); distinct keys per workload:
#   darcy_train_b32: simt 89, simt_wgrad 42
#   darcy_sample_b16: simt 42, simt_wgrad 0
#   darcy_sample_b64: simt 42, simt_wgrad 0
#   darcy_sample_b256: simt 42, simt_wgrad 0
#   darcy_sample_ddim0_b16: simt 42, simt_wgrad 0
#   mech_train_b32: simt 87, simt_wgrad 41
#   guidance_train_b32: simt 90, simt_wgrad 43
#   circular_train_b32: simt 92, simt_wgrad 43
#   circular_mech_b32: simt 87, simt_wgrad 41
#   distinct: simt 399, simt_wgrad 126
# ----------------------------------------------------------------------------------------------------------------------
# simt: B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed, bias, residual
SIMT_TABLE = [
    (16, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 256, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 32, 64, 64, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 256, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 512, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 512, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 128, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 512, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 8, 8, 1024, 1, 1, 1, 0, 0, 0, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 256, 8, 8, 1024, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 512, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 8, 8, 512, 3, 3, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 512, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 512, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 8, 8, 1024, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 8, 8, 1024, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 2048, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 8, 8, 2048, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 8, 8, 512, 16, 16, 512, 4, 4, 2, 1, 1, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 16, 16, 512, 4, 4, 2, 1, 1, 1, 0),  # mech_train_b32
    (32, 8, 8, 768, 8, 8, 128, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 768, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 768, 8, 8, 512, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 768, 8, 8, 1024, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 1024, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 1024, 8, 8, 512, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 1024, 8, 8, 512, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 1024, 8, 8, 1024, 3, 3, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 1024, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 1024, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 8, 8, 2048, 8, 8, 512, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 2048, 8, 8, 512, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 10, 10, 128, 8, 8, 128, 3, 3, 1, 0, 0, 0, 0),  # circular_train_b32
    (32, 10, 10, 128, 8, 8, 128, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 10, 10, 128, 8, 8, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 10, 10, 128, 8, 8, 256, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 10, 10, 128, 8, 8, 512, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 10, 10, 128, 16, 16, 128, 4, 4, 2, 3, 1, 0, 0),  # circular_train_b32
    (32, 10, 10, 128, 16, 16, 128, 4, 4, 2, 3, 1, 1, 0),  # circular_train_b32
    (32, 10, 10, 256, 8, 8, 128, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 10, 10, 256, 8, 8, 256, 3, 3, 1, 0, 0, 0, 0),  # circular_train_b32
    (32, 10, 10, 256, 8, 8, 256, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 10, 10, 256, 8, 8, 256, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 10, 10, 512, 8, 8, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 10, 10, 512, 8, 8, 512, 3, 3, 1, 0, 0, 0, 0),  # circular_mech_b32
    (32, 10, 10, 512, 8, 8, 512, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 10, 10, 512, 8, 8, 512, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 10, 10, 512, 8, 8, 1024, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 10, 10, 512, 8, 8, 2048, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 10, 10, 512, 16, 16, 512, 4, 4, 2, 3, 1, 0, 0),  # circular_mech_b32
    (32, 10, 10, 512, 16, 16, 512, 4, 4, 2, 3, 1, 1, 0),  # circular_mech_b32
    (32, 10, 10, 1024, 8, 8, 512, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 10, 10, 1024, 8, 8, 1024, 3, 3, 1, 0, 0, 0, 0),  # circular_mech_b32
    (32, 10, 10, 1024, 8, 8, 1024, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 10, 10, 1024, 8, 8, 1024, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 10, 10, 2048, 8, 8, 512, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 16, 16, 256, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 16, 16, 64, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 16, 16, 64, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 3, 3, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 512, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 16, 16, 512, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 16, 16, 1024, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 16, 16, 1024, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 16, 16, 256, 32, 32, 256, 4, 4, 2, 1, 1, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 32, 32, 256, 4, 4, 2, 1, 1, 1, 0),  # mech_train_b32
    (32, 16, 16, 512, 8, 8, 512, 4, 4, 2, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 8, 8, 512, 4, 4, 2, 1, 0, 1, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 512, 16, 16, 256, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 512, 3, 3, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 512, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 512, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 768, 16, 16, 64, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 768, 16, 16, 128, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 768, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 768, 16, 16, 512, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 1024, 16, 16, 256, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 1024, 16, 16, 256, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 18, 18, 64, 16, 16, 64, 3, 3, 1, 0, 0, 0, 0),  # circular_train_b32
    (32, 18, 18, 64, 16, 16, 64, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 18, 18, 64, 16, 16, 64, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 18, 18, 64, 16, 16, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 18, 18, 64, 16, 16, 256, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 18, 18, 64, 32, 32, 64, 4, 4, 2, 3, 1, 0, 0),  # circular_train_b32
    (32, 18, 18, 64, 32, 32, 64, 4, 4, 2, 3, 1, 1, 0),  # circular_train_b32
    (32, 18, 18, 128, 8, 8, 128, 4, 4, 2, 0, 0, 0, 0),  # circular_train_b32
    (32, 18, 18, 128, 8, 8, 128, 4, 4, 2, 0, 0, 1, 0),  # circular_train_b32
    (32, 18, 18, 128, 16, 16, 64, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 18, 18, 128, 16, 16, 128, 3, 3, 1, 0, 0, 0, 0),  # circular_train_b32
    (32, 18, 18, 128, 16, 16, 128, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 18, 18, 128, 16, 16, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 18, 18, 256, 16, 16, 64, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 18, 18, 256, 16, 16, 256, 3, 3, 1, 0, 0, 0, 0),  # circular_mech_b32
    (32, 18, 18, 256, 16, 16, 256, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 18, 18, 256, 16, 16, 256, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 18, 18, 256, 16, 16, 512, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 18, 18, 256, 16, 16, 1024, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 18, 18, 256, 32, 32, 256, 4, 4, 2, 3, 1, 0, 0),  # circular_mech_b32
    (32, 18, 18, 256, 32, 32, 256, 4, 4, 2, 3, 1, 1, 0),  # circular_mech_b32
    (32, 18, 18, 512, 8, 8, 512, 4, 4, 2, 0, 0, 0, 0),  # circular_mech_b32
    (32, 18, 18, 512, 8, 8, 512, 4, 4, 2, 0, 0, 1, 0),  # circular_mech_b32
    (32, 18, 18, 512, 16, 16, 256, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 18, 18, 512, 16, 16, 512, 3, 3, 1, 0, 0, 0, 0),  # circular_mech_b32
    (32, 18, 18, 512, 16, 16, 512, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 18, 18, 512, 16, 16, 512, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 18, 18, 1024, 16, 16, 256, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 128, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 128, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 32, 32, 32, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 32, 32, 32, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 128, 32, 32, 128, 3, 3, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 128, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 128, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 128, 32, 32, 256, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 128, 32, 32, 256, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 512, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 128, 32, 32, 512, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 128, 64, 64, 128, 4, 4, 2, 1, 1, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 64, 64, 128, 4, 4, 2, 1, 1, 1, 0),  # mech_train_b32
    (32, 32, 32, 256, 16, 16, 256, 4, 4, 2, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 16, 16, 256, 4, 4, 2, 1, 0, 1, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 256, 32, 32, 128, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 256, 32, 32, 128, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 256, 32, 32, 128, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 3, 3, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 512, 32, 32, 128, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 512, 32, 32, 128, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 32, 32, 768, 32, 32, 32, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 768, 32, 32, 64, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 768, 32, 32, 128, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 768, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 34, 34, 32, 32, 32, 32, 3, 3, 1, 0, 0, 0, 0),  # circular_train_b32
    (32, 34, 34, 32, 32, 32, 32, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 34, 34, 32, 32, 32, 32, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 34, 34, 32, 32, 32, 64, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 34, 34, 32, 32, 32, 128, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 34, 34, 32, 64, 64, 32, 4, 4, 2, 3, 1, 0, 0),  # circular_train_b32
    (32, 34, 34, 32, 64, 64, 32, 4, 4, 2, 3, 1, 1, 0),  # circular_train_b32
    (32, 34, 34, 64, 16, 16, 64, 4, 4, 2, 0, 0, 0, 0),  # circular_train_b32
    (32, 34, 34, 64, 16, 16, 64, 4, 4, 2, 0, 0, 1, 0),  # circular_train_b32
    (32, 34, 34, 64, 32, 32, 32, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 34, 34, 64, 32, 32, 64, 3, 3, 1, 0, 0, 0, 0),  # circular_train_b32
    (32, 34, 34, 64, 32, 32, 64, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 34, 34, 64, 32, 32, 64, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 34, 34, 128, 32, 32, 32, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 34, 34, 128, 32, 32, 128, 3, 3, 1, 0, 0, 0, 0),  # circular_mech_b32
    (32, 34, 34, 128, 32, 32, 128, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 34, 34, 128, 32, 32, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 34, 34, 128, 32, 32, 256, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 34, 34, 128, 32, 32, 512, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 34, 34, 128, 64, 64, 128, 4, 4, 2, 3, 1, 0, 0),  # circular_mech_b32
    (32, 34, 34, 128, 64, 64, 128, 4, 4, 2, 3, 1, 1, 0),  # circular_mech_b32
    (32, 34, 34, 256, 16, 16, 256, 4, 4, 2, 0, 0, 0, 0),  # circular_mech_b32
    (32, 34, 34, 256, 16, 16, 256, 4, 4, 2, 0, 0, 1, 0),  # circular_mech_b32
    (32, 34, 34, 256, 32, 32, 128, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 34, 34, 256, 32, 32, 256, 3, 3, 1, 0, 0, 0, 0),  # circular_mech_b32
    (32, 34, 34, 256, 32, 32, 256, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 34, 34, 256, 32, 32, 256, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 34, 34, 512, 32, 32, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 0, 0),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 64, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 64, 3, 3, 1, 1, 0, 0, 1),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 128, 7, 7, 1, 3, 0, 1, 0),  # mech_train_b32
    (32, 64, 64, 32, 64, 64, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 64, 64, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 0),  # circular_train_b32 guidance_train_b32
    (32, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 128, 32, 32, 128, 4, 4, 2, 1, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 32, 32, 128, 4, 4, 2, 1, 0, 1, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 128, 3, 3, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 128, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 128, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 256, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 64, 64, 128, 64, 64, 256, 3, 3, 1, 1, 0, 0, 1),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 768, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 64, 64, 256, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 256, 64, 64, 128, 1, 1, 1, 0, 0, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 64, 64, 256, 64, 64, 128, 3, 3, 1, 1, 0, 1, 0),  # mech_train_b32
    (32, 64, 64, 768, 64, 64, 32, 1, 1, 1, 0, 0, 0, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 768, 64, 64, 128, 1, 1, 1, 0, 0, 0, 0),  # circular_mech_b32 mech_train_b32
    (32, 66, 66, 32, 32, 32, 32, 4, 4, 2, 0, 0, 0, 0),  # circular_train_b32
    (32, 66, 66, 32, 32, 32, 32, 4, 4, 2, 0, 0, 1, 0),  # circular_train_b32
    (32, 66, 66, 32, 64, 64, 32, 3, 3, 1, 0, 0, 0, 0),  # circular_train_b32
    (32, 66, 66, 32, 64, 64, 32, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 66, 66, 32, 64, 64, 32, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 66, 66, 32, 64, 64, 64, 3, 3, 1, 0, 0, 0, 1),  # circular_train_b32
    (32, 66, 66, 64, 64, 64, 32, 3, 3, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 66, 66, 128, 32, 32, 128, 4, 4, 2, 0, 0, 0, 0),  # circular_mech_b32
    (32, 66, 66, 128, 32, 32, 128, 4, 4, 2, 0, 0, 1, 0),  # circular_mech_b32
    (32, 66, 66, 128, 64, 64, 128, 3, 3, 1, 0, 0, 0, 0),  # circular_mech_b32
    (32, 66, 66, 128, 64, 64, 128, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 66, 66, 128, 64, 64, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 66, 66, 128, 64, 64, 256, 3, 3, 1, 0, 0, 0, 1),  # circular_mech_b32
    (32, 66, 66, 256, 64, 64, 128, 3, 3, 1, 0, 0, 1, 0),  # circular_mech_b32
    (32, 70, 70, 32, 64, 64, 32, 7, 7, 1, 0, 0, 1, 0),  # circular_train_b32
    (32, 70, 70, 32, 64, 64, 128, 7, 7, 1, 0, 0, 1, 0),  # circular_mech_b32
    (64, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b64
    (64, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 32, 32, 32, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b64
    (64, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 32, 32, 256, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0),  # darcy_sample_b64
    (64, 64, 64, 32, 64, 64, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (64, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b64
    (64, 64, 64, 256, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b64
    (256, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b256
    (256, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 32, 32, 32, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0),  # darcy_sample_b256
    (256, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 32, 32, 256, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0),  # darcy_sample_b256
    (256, 64, 64, 32, 64, 64, 768, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
    (256, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0),  # darcy_sample_b256
    (256, 64, 64, 256, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1),  # darcy_sample_b256
]
# simt_wgrad: B, H, W, Cin, Cin_real, Ho, Wo, Cout, KH, KW, stride, pad, transposed, w_stride_n, w_stride_c, dbias
SIMT_WGRAD_TABLE = [
    (32, 8, 8, 128, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1152, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 128, 8, 8, 256, 1, 1, 1, 0, 0, 128, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1152, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 128, 8, 8, 768, 1, 1, 1, 0, 0, 128, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 128, 128, 16, 16, 128, 4, 4, 2, 1, 1, 16, 2048, 1),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 256, 8, 8, 128, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 256, 8, 8, 256, 1, 1, 1, 0, 0, 256, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 256, 8, 8, 256, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 256, 8, 8, 256, 3, 3, 1, 1, 0, 2304, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 256, 8, 8, 512, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 256, 256, 8, 8, 768, 1, 1, 1, 0, 0, 256, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 256, 256, 8, 8, 1024, 1, 1, 1, 0, 0, 256, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 256, 256, 8, 8, 1024, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 128, 1, 1, 1, 0, 0, 512, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 8, 8, 512, 512, 8, 8, 128, 3, 3, 1, 1, 0, 4608, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 8, 8, 512, 512, 8, 8, 512, 3, 3, 1, 1, 0, 4608, 9, 0),  # mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 768, 1, 1, 1, 0, 0, 512, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 1024, 1, 1, 1, 0, 0, 512, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 1024, 3, 3, 1, 1, 0, 4608, 9, 0),  # mech_train_b32
    (32, 8, 8, 512, 512, 16, 16, 512, 4, 4, 2, 1, 1, 16, 8192, 1),  # mech_train_b32
    (32, 8, 8, 1024, 1024, 8, 8, 768, 1, 1, 1, 0, 0, 1024, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 1024, 1024, 8, 8, 1024, 3, 3, 1, 1, 0, 9216, 9, 0),  # mech_train_b32
    (32, 8, 8, 2048, 2048, 8, 8, 512, 1, 1, 1, 0, 0, 2048, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 8, 8, 2048, 2048, 8, 8, 512, 3, 3, 1, 1, 0, 18432, 9, 0),  # mech_train_b32
    (32, 10, 10, 128, 128, 8, 8, 128, 3, 3, 1, 0, 0, 1152, 9, 0),  # circular_train_b32
    (32, 10, 10, 128, 128, 8, 8, 256, 3, 3, 1, 0, 0, 1152, 9, 0),  # circular_train_b32
    (32, 10, 10, 128, 128, 16, 16, 128, 4, 4, 2, 3, 1, 16, 2048, 1),  # circular_train_b32
    (32, 10, 10, 256, 256, 8, 8, 256, 3, 3, 1, 0, 0, 2304, 9, 0),  # circular_train_b32
    (32, 10, 10, 512, 512, 8, 8, 128, 3, 3, 1, 0, 0, 4608, 9, 0),  # circular_train_b32
    (32, 10, 10, 512, 512, 8, 8, 512, 3, 3, 1, 0, 0, 4608, 9, 0),  # circular_mech_b32
    (32, 10, 10, 512, 512, 8, 8, 1024, 3, 3, 1, 0, 0, 4608, 9, 0),  # circular_mech_b32
    (32, 10, 10, 512, 512, 16, 16, 512, 4, 4, 2, 3, 1, 16, 8192, 1),  # circular_mech_b32
    (32, 10, 10, 1024, 1024, 8, 8, 1024, 3, 3, 1, 0, 0, 9216, 9, 0),  # circular_mech_b32
    (32, 10, 10, 2048, 2048, 8, 8, 512, 3, 3, 1, 0, 0, 18432, 9, 0),  # circular_mech_b32
    (32, 16, 16, 64, 64, 16, 16, 64, 3, 3, 1, 1, 0, 576, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 64, 16, 16, 128, 1, 1, 1, 0, 0, 64, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 64, 16, 16, 128, 3, 3, 1, 1, 0, 576, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 64, 16, 16, 768, 1, 1, 1, 0, 0, 64, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 64, 64, 32, 32, 64, 4, 4, 2, 1, 1, 16, 1024, 1),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 128, 8, 8, 128, 4, 4, 2, 1, 0, 2048, 16, 1),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1152, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 128, 128, 16, 16, 768, 1, 1, 1, 0, 0, 128, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 256, 16, 16, 64, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 256, 16, 16, 64, 3, 3, 1, 1, 0, 2304, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 256, 16, 16, 128, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 16, 16, 256, 256, 16, 16, 256, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 256, 3, 3, 1, 1, 0, 2304, 9, 0),  # mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 512, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 512, 3, 3, 1, 1, 0, 2304, 9, 0),  # mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 768, 1, 1, 1, 0, 0, 256, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 256, 256, 32, 32, 256, 4, 4, 2, 1, 1, 16, 4096, 1),  # mech_train_b32
    (32, 16, 16, 512, 512, 8, 8, 512, 4, 4, 2, 1, 0, 8192, 16, 1),  # mech_train_b32
    (32, 16, 16, 512, 512, 16, 16, 512, 3, 3, 1, 1, 0, 4608, 9, 0),  # mech_train_b32
    (32, 16, 16, 512, 512, 16, 16, 768, 1, 1, 1, 0, 0, 512, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 1024, 1024, 16, 16, 256, 1, 1, 1, 0, 0, 1024, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 16, 16, 1024, 1024, 16, 16, 256, 3, 3, 1, 1, 0, 9216, 9, 0),  # mech_train_b32
    (32, 18, 18, 64, 64, 16, 16, 64, 3, 3, 1, 0, 0, 576, 9, 0),  # circular_train_b32
    (32, 18, 18, 64, 64, 16, 16, 128, 3, 3, 1, 0, 0, 576, 9, 0),  # circular_train_b32
    (32, 18, 18, 64, 64, 32, 32, 64, 4, 4, 2, 3, 1, 16, 1024, 1),  # circular_train_b32
    (32, 18, 18, 128, 128, 8, 8, 128, 4, 4, 2, 0, 0, 2048, 16, 1),  # circular_train_b32
    (32, 18, 18, 128, 128, 16, 16, 128, 3, 3, 1, 0, 0, 1152, 9, 0),  # circular_train_b32
    (32, 18, 18, 256, 256, 16, 16, 64, 3, 3, 1, 0, 0, 2304, 9, 0),  # circular_train_b32
    (32, 18, 18, 256, 256, 16, 16, 256, 3, 3, 1, 0, 0, 2304, 9, 0),  # circular_mech_b32
    (32, 18, 18, 256, 256, 16, 16, 512, 3, 3, 1, 0, 0, 2304, 9, 0),  # circular_mech_b32
    (32, 18, 18, 256, 256, 32, 32, 256, 4, 4, 2, 3, 1, 16, 4096, 1),  # circular_mech_b32
    (32, 18, 18, 512, 512, 8, 8, 512, 4, 4, 2, 0, 0, 8192, 16, 1),  # circular_mech_b32
    (32, 18, 18, 512, 512, 16, 16, 512, 3, 3, 1, 0, 0, 4608, 9, 0),  # circular_mech_b32
    (32, 18, 18, 1024, 1024, 16, 16, 256, 3, 3, 1, 0, 0, 9216, 9, 0),  # circular_mech_b32
    (32, 32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 288, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 32, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 288, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 32, 32, 768, 1, 1, 1, 0, 0, 32, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 16, 512, 1),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1024, 16, 1),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 64, 32, 32, 64, 3, 3, 1, 1, 0, 576, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 64, 64, 32, 32, 768, 1, 1, 1, 0, 0, 64, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 128, 128, 32, 32, 32, 1, 1, 1, 0, 0, 128, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 128, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1152, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 32, 32, 128, 128, 32, 32, 128, 3, 3, 1, 1, 0, 1152, 9, 0),  # mech_train_b32
    (32, 32, 32, 128, 128, 32, 32, 256, 1, 1, 1, 0, 0, 128, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 128, 128, 32, 32, 256, 3, 3, 1, 1, 0, 1152, 9, 0),  # mech_train_b32
    (32, 32, 32, 128, 128, 32, 32, 768, 1, 1, 1, 0, 0, 128, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 128, 128, 64, 64, 128, 4, 4, 2, 1, 1, 16, 2048, 1),  # mech_train_b32
    (32, 32, 32, 256, 256, 16, 16, 256, 4, 4, 2, 1, 0, 4096, 16, 1),  # mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 32, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 256, 256, 32, 32, 64, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 32, 32, 256, 256, 32, 32, 128, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 256, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 256, 3, 3, 1, 1, 0, 2304, 9, 0),  # mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 768, 1, 1, 1, 0, 0, 256, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 512, 512, 32, 32, 128, 1, 1, 1, 0, 0, 512, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 32, 32, 512, 512, 32, 32, 128, 3, 3, 1, 1, 0, 4608, 9, 0),  # mech_train_b32
    (32, 34, 34, 32, 32, 32, 32, 32, 3, 3, 1, 0, 0, 288, 9, 0),  # circular_train_b32
    (32, 34, 34, 32, 32, 32, 32, 64, 3, 3, 1, 0, 0, 288, 9, 0),  # circular_train_b32
    (32, 34, 34, 32, 32, 64, 64, 32, 4, 4, 2, 3, 1, 16, 512, 1),  # circular_train_b32
    (32, 34, 34, 64, 64, 16, 16, 64, 4, 4, 2, 0, 0, 1024, 16, 1),  # circular_train_b32
    (32, 34, 34, 64, 64, 32, 32, 64, 3, 3, 1, 0, 0, 576, 9, 0),  # circular_train_b32
    (32, 34, 34, 128, 128, 32, 32, 32, 3, 3, 1, 0, 0, 1152, 9, 0),  # circular_train_b32
    (32, 34, 34, 128, 128, 32, 32, 128, 3, 3, 1, 0, 0, 1152, 9, 0),  # circular_mech_b32
    (32, 34, 34, 128, 128, 32, 32, 256, 3, 3, 1, 0, 0, 1152, 9, 0),  # circular_mech_b32
    (32, 34, 34, 128, 128, 64, 64, 128, 4, 4, 2, 3, 1, 16, 2048, 1),  # circular_mech_b32
    (32, 34, 34, 256, 256, 16, 16, 256, 4, 4, 2, 0, 0, 4096, 16, 1),  # circular_mech_b32
    (32, 34, 34, 256, 256, 32, 32, 256, 3, 3, 1, 0, 0, 2304, 9, 0),  # circular_mech_b32
    (32, 34, 34, 512, 512, 32, 32, 128, 3, 3, 1, 0, 0, 4608, 9, 0),  # circular_mech_b32
    (32, 64, 64, 32, 2, 64, 64, 32, 7, 7, 1, 3, 0, 98, 49, 1),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 10, 64, 64, 128, 7, 7, 1, 3, 0, 490, 49, 1),  # mech_train_b32
    (32, 64, 64, 32, 32, 32, 32, 32, 4, 4, 2, 1, 0, 512, 16, 1),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 32, 64, 64, 32, 3, 3, 1, 1, 0, 288, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 32, 32, 64, 64, 32, 3, 3, 1, 1, 0, 288, 9, 1),  # circular_train_b32 guidance_train_b32
    (32, 64, 64, 32, 32, 64, 64, 768, 1, 1, 1, 0, 0, 32, 1, 0),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 64, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 576, 9, 0),  # darcy_train_b32 guidance_train_b32
    (32, 64, 64, 128, 128, 32, 32, 128, 4, 4, 2, 1, 0, 2048, 16, 1),  # mech_train_b32
    (32, 64, 64, 128, 128, 64, 64, 128, 3, 3, 1, 1, 0, 1152, 9, 0),  # mech_train_b32
    (32, 64, 64, 128, 128, 64, 64, 768, 1, 1, 1, 0, 0, 128, 1, 0),  # circular_mech_b32 mech_train_b32
    (32, 64, 64, 256, 256, 64, 64, 32, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_train_b32 darcy_train_b32 guidance_train_b32
    (32, 64, 64, 256, 256, 64, 64, 128, 1, 1, 1, 0, 0, 256, 1, 1),  # circular_mech_b32 mech_train_b32
    (32, 64, 64, 256, 256, 64, 64, 128, 3, 3, 1, 1, 0, 2304, 9, 0),  # mech_train_b32
    (32, 66, 66, 32, 32, 32, 32, 32, 4, 4, 2, 0, 0, 512, 16, 1),  # circular_train_b32
    (32, 66, 66, 32, 32, 64, 64, 32, 3, 3, 1, 0, 0, 288, 9, 0),  # circular_train_b32
    (32, 66, 66, 64, 64, 64, 64, 32, 3, 3, 1, 0, 0, 576, 9, 0),  # circular_train_b32
    (32, 66, 66, 128, 128, 32, 32, 128, 4, 4, 2, 0, 0, 2048, 16, 1),  # circular_mech_b32
    (32, 66, 66, 128, 128, 64, 64, 128, 3, 3, 1, 0, 0, 1152, 9, 0),  # circular_mech_b32
    (32, 66, 66, 256, 256, 64, 64, 128, 3, 3, 1, 0, 0, 2304, 9, 0),  # circular_mech_b32
    (32, 70, 70, 32, 2, 64, 64, 32, 7, 7, 1, 0, 0, 98, 49, 1),  # circular_train_b32
    (32, 70, 70, 32, 10, 64, 64, 128, 7, 7, 1, 0, 0, 490, 49, 1),  # circular_mech_b32
]
TABLES = {'simt': SIMT_TABLE, 'simt_wgrad': SIMT_WGRAD_TABLE}

# rows no recorded step produces, for the tile, gather and split cases the workloads do not reach (test_plan_coverage)
SIMT_SYNTHETIC = [
    (1, 7, 7, 4, 7, 7, 4, 3, 3, 1, 1, 0, 1, 1),          # B = 1, ragged M (49), K = 36, Cout = 4
    (3, 9, 9, 12, 9, 9, 36, 1, 1, 1, 0, 0, 1, 0),        # odd B, K = 12 (one partial K tile), ragged N
    (5, 9, 9, 12, 9, 9, 100, 3, 3, 1, 1, 0, 1, 1),       # K = 108, two N tiles with a ragged last one
    (5, 9, 9, 12, 9, 9, 100, 3, 3, 1, 1, 0, 0, 0),       # the same without bias and residual
    (3, 5, 5, 8, 9, 9, 12, 3, 3, 2, 1, 1, 1, 1),         # transposed stride 2, odd output size
    (3, 7, 7, 4, 7, 7, 100, 3, 3, 1, 1, 1, 0, 1),        # transposed stride 1
    (3, 9, 9, 12, 4, 4, 36, 4, 4, 2, 1, 0, 1, 0),        # regular stride 2, 4x4 over an odd input
]
SIMT_WGRAD_SYNTHETIC = [
    (1, 9, 9, 12, 12, 9, 9, 36, 3, 3, 1, 1, 0, 108, 9, 1),     # M = 81 < 256: one split; ragged K and N tiles
    (5, 9, 9, 12, 12, 9, 9, 100, 3, 3, 1, 1, 0, 108, 9, 1),    # M = 405: two splits of 208 (203 rounded), short last
    (5, 9, 9, 12, 12, 9, 9, 100, 3, 3, 1, 1, 0, 108, 9, 0),    # the same without dbias
    (7, 5, 5, 8, 6, 9, 9, 12, 3, 3, 2, 1, 1, 9, 108, 1),       # ConvTranspose layout, Cin_real < Cin, odd output
    (3, 7, 7, 16, 10, 7, 7, 4, 3, 3, 1, 1, 0, 90, 9, 0),       # Conv layout, Cin_real < Cin, Cout = 4
    (3, 7, 7, 12, 12, 7, 7, 12, 3, 3, 1, 1, 1, 9, 108, 1),     # transposed stride 1, square (Cout = Cin) blocks
]

def simt_id(k):
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p, tr, hb, hr = k
    return (f'B{B}_{H}x{W}_{Cin}to{Cout}_o{Ho}x{Wo}_k{KH}s{s}p{p}' + ('T' if tr else '') + ('_bias' if hb else '')
            + ('_res' if hr else ''))


def wgrad_id(k):
    B, H, W, Cin, Cr, Ho, Wo, Cout, KH, KW, s, p, tr, sn, sc, hdb = k
    return (f'B{B}_{H}x{W}x{Cin}r{Cr}_o{Ho}x{Wo}x{Cout}_k{KH}s{s}p{p}' + ('T' if tr else '') + f'_w{sn}.{sc}'
            + ('_db' if hdb else ''))


# ----------------------------------------------------------------------------------------------------------------------
# census
# ----------------------------------------------------------------------------------------------------------------------
def test_census_is_covered_by_the_table():
    assert_census_in_tables(TABLES)


def test_every_table_row_is_produced_by_the_census():
    assert_tables_in_census(TABLES)


def test_every_exact_mode_entry_point_is_checked_or_listed():
    assert_checked_or_listed(census_exact()[1], 'the exact mode')


# ----------------------------------------------------------------------------------------------------------------------
# launch arithmetic (restated from conv_simt.cu; the kernels have no plan query)
# ----------------------------------------------------------------------------------------------------------------------
BM, BN, BK = 64, 64, 16          # CS_BM, CS_BN, CS_BK: output tile M x N, K step (the weight gradient's K tile is BM)


def fwd_plan(k):
    """pidm_conv2d_simt: grid (ceil(M / BM), ceil(Cout / BN)), K walked in steps of BK"""
    B, Ho, Wo, Cout, KH, KW, Cin = k[0], k[4], k[5], k[6], k[7], k[8], k[3]
    M, K = B * Ho * Wo, KH * KW * Cin
    return dict(M=M, K=K, m_tiles=-(-M // BM), n_tiles=-(-Cout // BN))


def wgrad_plan(k, n_sms):
    """pidm_conv2d_wgrad_simt: grid (ceil(K / BM), ceil(Cout / BN), splits); splits = ceil(4 SMs / tiles) capped at
    ceil(M / 256), m_per_split = ceil(M / splits) rounded up to BK, and splits recounted from m_per_split"""
    B, Cin, Ho, Wo, Cout, KH, KW = k[0], k[3], k[5], k[6], k[7], k[8], k[9]
    M, K = B * Ho * Wo, KH * KW * Cin
    k_tiles = -(-K // BM)
    tiles = k_tiles * -(-Cout // BN)
    rule, cap = -(-4 * n_sms // tiles), -(-M // 256)
    first = max(min(rule, cap), 1)
    raw = -(-M // first)
    mps = -(-raw // BK) * BK
    return dict(M=M, K=K, k_tiles=k_tiles, rule=rule, cap=cap, first=first, raw=raw, mps=mps, splits=-(-M // mps))


# ----------------------------------------------------------------------------------------------------------------------
# operands, references, predicates
# ----------------------------------------------------------------------------------------------------------------------
def _randn(g, shape, dtype, scale=1.0):
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _d(t, absolute=False):
    if t is None:
        return None
    t = t.double()
    return t.abs() if absolute else t


class FwdCase:
    """operands, fp64 reference r, absolute-value reference A and bound of one pidm_conv2d_simt row"""

    def __init__(self, k, dtype):
        B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p, tr, hb, hr = k
        self.k, self.dtype = k, dtype
        self.M, self.K = B * Ho * Wo, KH * KW * Cin
        g = gen(('simt', NAME[dtype]) + tuple(k))
        self.x = _randn(g, (B, H, W, Cin), dtype)
        self.wp = _randn(g, (Cout, self.K), dtype, 1.0 / math.sqrt(self.K))
        self.bias = torch.randn(Cout, generator=g, device=DEV) if hb else None
        self.res = _randn(g, (B, Ho, Wo, Cout), dtype) if hr else None
        self.r = self.ref()
        A = self.ref(absolute=True)
        if dtype == torch.float32:
            self.bound = C_FWD * (math.sqrt(self.K) + 2) * U * A
        else:
            self.bound = 2.0 ** -8 * self.r.abs() + C_FWD * math.sqrt(self.K) * U * A

    def ref(self, x=None, wp=None, absolute=False, geom=None):
        """fp64 y of the contract for these operands; x, wp and geom replace the row's (mutants)"""
        x = self.x if x is None else x
        wp = self.wp if wp is None else wp
        return conv_ref(_d(x, absolute), _d(wp, absolute), _d(self.bias, absolute), _d(self.res, absolute),
                        geom or self.k).contiguous()

    def ratio(self, y):
        return ratio((y.double() - self.r).abs(), self.bound)

    def run(self):
        B, H, W, Cin, Ho, Wo, Cout = self.k[:7]
        buf, y = guarded(self.M * Cout, self.dtype)
        call_sync('pidm_conv2d_simt', self.x, self.wp, self.bias, self.res, y, *self.k[:12], CODE[self.dtype])
        return buf, y.view(B, Ho, Wo, Cout)


def _wgrad_ref(x, dy, geom):
    """fp64 dL/dWp [Cout][taps][Cin] of the forward contract for the cotangent dy"""
    Cout, K = geom[6], geom[7] * geom[8] * geom[3]
    wp = torch.zeros(Cout, K, dtype=torch.float64, device=DEV, requires_grad=True)
    (gw,) = torch.autograd.grad(conv_ref(x, wp, None, None, geom), wp, dy)
    return gw.view(Cout, geom[7] * geom[8], geom[3])


class WgradCase:
    """operands, fp64 references and prefilled output buffers of one pidm_conv2d_wgrad_simt row"""

    def __init__(self, k, dtype):
        B, H, W, Cin, Cr, Ho, Wo, Cout, KH, KW, s, p, tr, sn, sc, hdb = k
        self.k, self.dtype = k, dtype
        self.geom = (B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p, tr)
        self.plan = wgrad_plan(k, sms())
        g = gen(('simt_wgrad', NAME[dtype]) + tuple(k))
        self.x = _randn(g, (B, H, W, Cin), dtype)            # padded channels (>= Cin_real) random: must not reach dw
        self.dy = _randn(g, (B, Ho, Wo, Cout), dtype)
        self.D_all = _wgrad_ref(self.x.double(), self.dy.double(), self.geom)
        self.A = _wgrad_ref(self.x.double().abs(), self.dy.double().abs(), self.geom)[..., :Cr]
        self.D = self.D_all[..., :Cr]
        self.idx = self.index(sn, sc)
        self.n = int(self.idx.max()) + 1
        self.guard = max(1024, self.n)
        self.keep = torch.randn(self.n + 2 * self.guard, generator=g, device=DEV)
        self.db = self.dy.double().sum(dim=(0, 1, 2)) if hdb else None
        self.A_db = self.dy.double().abs().sum(dim=(0, 1, 2)) if hdb else None
        self.keep_db = torch.randn(Cout + 2 * 1024, generator=g, device=DEV) if hdb else None

    def index(self, sn, sc, c=None):
        """framework-layout indices n*sn + c*sc + tap [Cout, taps, Cin_real] (or of the one channel c)"""
        Cr, Cout, taps = self.k[4], self.k[7], self.k[8] * self.k[9]
        n = torch.arange(Cout, device=DEV).view(-1, 1, 1)
        t = torch.arange(taps, device=DEV).view(1, -1, 1)
        cc = torch.arange(Cr, device=DEV).view(1, 1, -1) if c is None else torch.full((1, 1, 1), c, device=DEV)
        return n * sn + cc * sc + t

    def bound(self, prefill, A):
        return C_WG * math.sqrt(self.plan['M']) * U * A + self.plan['splits'] * U * (prefill.abs() + A)

    def run(self):
        B, H, W, Cin, Cr, Ho, Wo, Cout, KH, KW, s, p, tr, sn, sc, hdb = self.k
        buf = self.keep.clone()
        dbuf = self.keep_db.clone() if hdb else None
        call_sync('pidm_conv2d_wgrad_simt', self.x, self.dy, buf[self.guard:], None if dbuf is None else dbuf[1024:],
                  B, H, W, Cin, Cr, Ho, Wo, Cout, KH, KW, s, p, tr, sn, sc, CODE[self.dtype])
        return buf, dbuf

    def exact(self, D=None, db=None, idx=None):
        """the buffers a kernel that accumulates D (at idx) and db exactly would leave (mutants edit D, db or idx)"""
        D = self.D if D is None else D
        idx = self.idx if idx is None else idx
        buf = self.keep.double()
        buf.index_put_((self.guard + idx.reshape(-1),), D.reshape(-1), accumulate=True)
        dbuf = None
        if self.db is not None:
            dbuf = self.keep_db.double()
            dbuf[1024:1024 + self.k[7]] += self.db if db is None else db
        return buf.float(), None if dbuf is None else dbuf.float()

    def judge(self, buf, dbuf):
        """{output: worst |err| / bound}; an element outside the contract that changed counts as infinitely bad"""
        touched = torch.zeros_like(buf, dtype=torch.bool)
        touched[self.guard + self.idx.reshape(-1)] = True
        pre = self.keep.double()[self.guard + self.idx]
        out = {'dw': ratio((buf.double()[self.guard + self.idx] - pre - self.D).abs(), self.bound(pre, self.A)),
               'dw_untouched': 0.0 if bool((buf[~touched] == self.keep[~touched]).all()) else math.inf}
        if self.db is not None:
            Cout = self.k[7]
            pre_b = self.keep_db.double()[1024:1024 + Cout]
            out['db'] = ratio((dbuf.double()[1024:1024 + Cout] - pre_b - self.db).abs(), self.bound(pre_b, self.A_db))
            guards = torch.cat((dbuf[:1024], dbuf[1024 + Cout:]))
            keep = torch.cat((self.keep_db[:1024], self.keep_db[1024 + Cout:]))
            out['db_untouched'] = 0.0 if bool((guards == keep).all()) else math.inf
        return out


# ----------------------------------------------------------------------------------------------------------------------
# replay
# ----------------------------------------------------------------------------------------------------------------------
FWD_ROWS = SIMT_TABLE + SIMT_SYNTHETIC
WGRAD_ROWS = SIMT_WGRAD_TABLE + SIMT_WGRAD_SYNTHETIC


@pytest.mark.parametrize('dtype', DTYPES, ids=[NAME[d] for d in DTYPES])
@pytest.mark.parametrize('k', FWD_ROWS, ids=[simt_id(k) for k in FWD_ROWS])
def test_simt_replay(k, dtype):
    c = FwdCase(k, dtype)
    buf, y = c.run()
    assert guards_intact(buf), f'{simt_id(k)}: a store landed outside y'
    q = c.ratio(y)
    note(TAG, f'simt {NAME[dtype]} y {simt_id(k)}', q)
    assert q <= 1.0, f'{simt_id(k)} {NAME[dtype]}: worst |err| / bound = {q:.4g} ({fwd_plan(k)})'


@pytest.mark.parametrize('dtype', DTYPES, ids=[NAME[d] for d in DTYPES])
@pytest.mark.parametrize('k', WGRAD_ROWS, ids=[wgrad_id(k) for k in WGRAD_ROWS])
def test_simt_wgrad_replay(k, dtype):
    c = WgradCase(k, dtype)
    rs = c.judge(*c.run())
    for name in ('dw', 'db'):
        if name in rs:
            note(TAG, f'simt_wgrad {NAME[dtype]} {name} {wgrad_id(k)}', rs[name])
    assert max(rs.values()) <= 1.0, f'{wgrad_id(k)} {NAME[dtype]}: worst |err| / bound = {rs} ({c.plan})'


# ----------------------------------------------------------------------------------------------------------------------
# the predicates reject subtly wrong outputs (edits of the fp64 reference; no faulty code runs on the GPU)
# ----------------------------------------------------------------------------------------------------------------------
def _row(pred, rows):
    """the cheapest row (fewest multiply-adds) with the property a mutant needs"""
    rows = [k for k in rows if pred(k)]
    if not rows:
        pytest.fail('no row has the property this mutant needs')
    return min(rows, key=lambda k: fwd_plan(k)['M'] * fwd_plan(k)['K'] * k[6])


def _fwd_rejects(c, y):
    assert c.ratio(c.r.to(c.dtype)) <= 1.0, 'the unedited reference must pass'
    return c.ratio(y.to(c.dtype)) > 1.0


DT = pytest.mark.parametrize('dtype', DTYPES, ids=[NAME[d] for d in DTYPES])


@DT
def test_mutant_last_k_tile_dropped(dtype):
    """the last 16-wide K tile missing: a partial one (K % 16 != 0) of a synthetic row, a full one of a product row"""
    for k in (_row(lambda k: fwd_plan(k)['K'] % BK, SIMT_SYNTHETIC), _row(lambda k: fwd_plan(k)['K'] % BK == 0
                                                                           and fwd_plan(k)['K'] >= 256, SIMT_TABLE)):
        c = FwdCase(k, dtype)
        wp = c.wp.clone()
        wp[:, (c.K - 1) // BK * BK:] = 0
        assert _fwd_rejects(c, c.ref(wp=wp)), simt_id(k)


@DT
def test_mutant_border_tap_from_the_nearest_row(dtype):
    """taps at ih = -1 read row 0 instead of zero"""
    k = _row(lambda k: not k[11] and k[10] >= 1, SIMT_TABLE)
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p = k[:11]
    c = FwdCase(k, dtype)
    xp = F.pad(c.x.double(), (0, 0, p, p, p, p))
    xp[:, p - 1, p:p + W] = c.x.double()[:, 0]
    assert _fwd_rejects(c, c.ref(x=xp, geom=(B, H + 2 * p, W + 2 * p, Cin, Ho, Wo, Cout, KH, KW, s, 0, 0))), simt_id(k)


@DT
def test_mutant_transposed_parity_class_shifted(dtype):
    """the output rows of one th % 2 parity class gather from the input row one pixel further down"""
    for k in (_row(lambda k: k[11] and k[9] == 2, SIMT_SYNTHETIC), _row(lambda k: k[11] and k[9] == 2, SIMT_TABLE)):
        c = FwdCase(k, dtype)
        xs = torch.zeros_like(c.x)
        xs[:, :-1] = c.x[:, 1:]
        y = c.r.clone()
        y[:, 0::2] = c.ref(x=xs)[:, 0::2]
        assert _fwd_rejects(c, y), simt_id(k)


@DT
def test_mutant_bias_missing_from_the_ragged_n_tile(dtype):
    k = _row(lambda k: k[12] and k[6] > BN and k[6] % BN, FWD_ROWS)
    c = FwdCase(k, dtype)
    n0 = (k[6] - 1) // BN * BN
    y = c.r.clone()
    y[..., n0:] -= c.bias.double()[n0:]
    assert _fwd_rejects(c, y), simt_id(k)


@DT
def test_mutant_residual_missing_from_the_last_m_tile(dtype):
    for k in (_row(lambda k: k[13] and fwd_plan(k)['M'] % BM, SIMT_SYNTHETIC), _row(lambda k: k[13], SIMT_TABLE)):
        c = FwdCase(k, dtype)
        M, Cout = c.M, k[6]
        m0 = (M - 1) // BM * BM
        y = c.r.clone()
        y.view(M, Cout)[m0:] -= c.res.double().view(M, Cout)[m0:]
        assert _fwd_rejects(c, y), simt_id(k)


@DT
def test_mutant_last_pixel_of_last_sample_zeroed(dtype):
    for k in (_row(lambda k: True, SIMT_TABLE), SIMT_SYNTHETIC[0]):
        c = FwdCase(k, dtype)
        y = c.r.clone()
        y[-1, -1, -1, :] = 0
        assert _fwd_rejects(c, y), simt_id(k)


def _wgrad_rejects(c, D=None, db=None, idx=None):
    assert max(c.judge(*c.exact()).values()) <= 1.0, 'the unedited reference must pass'
    return max(c.judge(*c.exact(D, db, idx)).values()) > 1.0


def _wgrad_row(pred, rows=None):
    rows = [k for k in (rows or WGRAD_ROWS) if pred(k)]
    if not rows:
        pytest.fail('no row has the property this mutant needs')
    return min(rows, key=lambda k: wgrad_plan(k, sms())['M'] * wgrad_plan(k, sms())['K'] * k[7])


@DT
def test_mutant_wgrad_short_last_split_missing(dtype):
    k = _wgrad_row(lambda k: wgrad_plan(k, sms())['splits'] > 1 and wgrad_plan(k, sms())['M'] %
                   wgrad_plan(k, sms())['mps'])
    c = WgradCase(k, dtype)
    m0 = (c.plan['splits'] - 1) * c.plan['mps']
    dy = c.dy.double().clone().view(c.plan['M'], -1)
    dy[:m0] = 0
    part = _wgrad_ref(c.x.double(), dy.view(c.dy.shape), c.geom)[..., :k[4]]
    db = None if c.db is None else c.db - dy.sum(0)
    assert _wgrad_rejects(c, D=c.D - part, db=db), (wgrad_id(k), c.plan)


@DT
def test_mutant_dbias_once_per_k_tile(dtype):
    k = _wgrad_row(lambda k: k[15] and wgrad_plan(k, sms())['k_tiles'] > 1)
    c = WgradCase(k, dtype)
    assert _wgrad_rejects(c, db=c.plan['k_tiles'] * c.db), (wgrad_id(k), c.plan)


@DT
def test_mutant_padded_stem_channel_written(dtype):
    """the gradient of channel c = Cin_real stored as if it were real, in both weight layouts"""
    for k in (_wgrad_row(lambda k: k[4] < k[3] and k[14] == k[8] * k[9]),
              _wgrad_row(lambda k: k[4] < k[3] and k[13] == k[8] * k[9])):
        c = WgradCase(k, dtype)
        Cr = k[4]
        D = torch.cat((c.D, c.D_all[..., Cr:Cr + 1]), dim=-1)
        idx = torch.cat((c.idx, c.index(k[13], k[14], Cr)), dim=-1)
        assert _wgrad_rejects(c, D=D, idx=idx), wgrad_id(k)


@DT
def test_mutant_convtranspose_strides_swapped(dtype):
    k = _wgrad_row(lambda k: k[12] and k[13] == k[8] * k[9] and k[14] != k[13])
    c = WgradCase(k, dtype)
    assert _wgrad_rejects(c, idx=c.index(k[14], k[13])), wgrad_id(k)


@DT
def test_mutant_wgrad_tap_block_transposed(dtype):
    k = _wgrad_row(lambda k: k[4] == k[7] and k[8] * k[9] > 1)
    c = WgradCase(k, dtype)
    D = c.D.clone()
    tap = k[8] * k[9] // 2
    D[:, tap, :] = c.D[:, tap, :].t()
    assert _wgrad_rejects(c, D=D), wgrad_id(k)


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
def _halo(transposed, KH, pad):
    """the geometries of a circular layer (ops._halo_geometry): a valid convolution over the halo'd input, or the
    transposed gather with pad = KH / 2 + 1 (every tap one pixel further in)"""
    return pad >= KH // 2 + 1 if transposed else (pad == 0 and KH > 1)


def fwd_coverage():
    plans = [(k, fwd_plan(k)) for k in FWD_ROWS]
    return {
        'ragged M tile': any(p['M'] % BM for _, p in plans),
        'ragged N tile': any(k[6] % BN for k, _ in plans),
        'ragged N tile after a full one': any(k[6] > BN and k[6] % BN for k, _ in plans),
        'partial K tile': any(p['K'] % BK for _, p in plans),
        'gathers (transposed, stride)': {(k[11], k[9]) for k, _ in plans},
        'taps': {k[7] * k[8] for k, _ in plans},
        'halo regular': any(not k[11] and _halo(0, k[7], k[10]) for k, _ in plans),
        'halo transposed': any(k[11] and _halo(1, k[7], k[10]) for k, _ in plans),
        'bias': {k[12] for k, _ in plans},
        'residual': {k[13] for k, _ in plans},
        'B = 1 and odd B': {1, 3} <= {k[0] for k, _ in plans},
        'longest K': max(p['K'] for _, p in plans),
    }


def wgrad_coverage(n_sms):
    plans = [(k, wgrad_plan(k, n_sms)) for k in WGRAD_ROWS]
    conv_layout = lambda k: k[14] == k[8] * k[9]          # [Cout][Cin][taps]: s_c = taps
    return {
        'one split (M < 256)': any(p['splits'] == 1 and p['M'] < 256 for _, p in plans),
        'cap ceil(M/256) binds': any(1 < p['cap'] < p['rule'] for _, p in plans),
        'SM-count rule binds': any(1 < p['rule'] < p['cap'] for _, p in plans),
        'short last split': any(p['splits'] > 1 and p['M'] % p['mps'] for _, p in plans),
        'm_per_split rounded up': any(p['raw'] % BK for _, p in plans),
        'ragged K tile': any(p['K'] % BM for _, p in plans),
        'ragged N tile': any(k[7] % BN for k, _ in plans),
        'gathers (transposed, stride)': {(k[12], k[10]) for k, _ in plans},
        'taps': {k[8] * k[9] for k, _ in plans},
        'halo regular': any(not k[12] and _halo(0, k[8], k[11]) for k, _ in plans),
        'halo transposed': any(k[12] and _halo(1, k[8], k[11]) for k, _ in plans),
        'layouts': {conv_layout(k) for k, _ in plans},
        'Cin_real < Cin per layout': {conv_layout(k) for k, _ in plans if k[4] < k[3]},
        'dbias': {k[15] for k, _ in plans},
    }


def test_plan_coverage():
    assert sms() == 132, 'the synthetic rows are chosen for the 132-SM H100'
    fc, wc = fwd_coverage(), wgrad_coverage(sms())
    print(f'[{TAG}] forward coverage {fc}\n[{TAG}] weight-gradient coverage {wc}')
    gathers = {(0, 1), (0, 2), (1, 1), (1, 2)}
    assert all(v for v in fc.values()), fc
    assert fc['gathers (transposed, stride)'] == gathers and {1, 9, 16, 49} <= fc['taps'], fc
    assert fc['bias'] == {0, 1} and fc['residual'] == {0, 1}, fc
    assert all(v for v in wc.values()), wc
    assert wc['gathers (transposed, stride)'] == gathers and {1, 9, 16, 49} <= wc['taps'], wc
    assert wc['layouts'] == {True, False} and wc['Cin_real < Cin per layout'] == {True, False}, wc
    assert wc['dbias'] == {0, 1}, wc
