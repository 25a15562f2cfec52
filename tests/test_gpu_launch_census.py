"""Every tensor-core launch of the benchmarked steps, replayed element by element against an fp64 reference.

The convolution (conv_tc.cu), the two weight-gradient kernels (wgrad_tc.cu) and the linear-attention block
(attention_fused.cu) choose their plan -- tile widths, persistent-grid waves, pixel splits, pixel chunks -- from the batch
size and the SM count.  The per-op tests in test_gpu_ops.py run small batches, so they see few of the plans the
benchmark runs, and they compare whole tensors by a norm ratio, which a bug confined to one tile row cannot move.  Here:

  1. census: the distinct integer arguments of every tensor-core call in one eager step of every workload bench.py times
     (recorded by tests/census.py) must equal the tables below (`python tests/census.py --print-table` regenerates
     them);
  2. replay: every table row (plus a few synthetic rows that reach the planner choices the workloads do not) is run
     directly through the C ABI on fresh seeded bf16-exact operands and compared with an fp64 reference of the contract
     in include/pidm.h, per element:
        conv (bf16 out)         |y - r| <= 2^-8 |r| + C_ACC sqrt(K) 2^-24 A      A = the same op on |x|, |W|, |bias|, |res|
        wgrad, gn_sums (fp32)   |y - r| <=              C_ACC sqrt(K) 2^-24 A      K = summed pixels (elements)
        attention block         |y - r| <= A_ATT |r| + B_ATT rms(r over a slice)  (+ 2^-14 |prefill| when accumulated)
     The block's residual and bias are scaled to the rms of its attention term, so that each of the three terms of y is
     visible to the bound.  Output buffers sit between sentinel guard regions that must survive the launch;
     accumulating outputs are prefilled;
  3. mutants: the same predicates reject the fp64 reference edited the way a subtle kernel bug would change it;
  4. plan coverage: the C-ABI plan queries show that the table plus the synthetic rows reach every tile instantiation and
     every planner branch (ragged persistent waves, short last splits, ragged last chunks, odd batch with TN = 2).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from census import assert_census_in_tables, assert_tables_in_census
from checks import conv_ref, gen, note, ratio

pytestmark = pytest.mark.gpu

DEV = 'cuda'

# Error-bound constants.  Products of bf16 operands are exact in fp32, so the only kernel-side errors are the fp32
# accumulation (bounded by C_ACC sqrt(K) 2^-24 times the absolute-value reference) and, for bf16 outputs, one rounding.
# The attention block keeps q / k / v / ctx / out / dout as bf16 tensor-core operands, hence the relative + slice-rms
# form.  C_ACC, A_ATT and B_ATT were set from H100 80GB HBM3 runs of this file; the worst |err| / bound observed per
# kernel family is recorded in DESIGN.md section 2.
C_ACC = 1.0
A_ATT = 2.0 ** -7
# y and dxn: slice = sample; dW_qkv: slice = (q | k | v, head); dW_out: slice = one head's 32 columns; db: whole vector
B_ATT = {'fwd': 2.0 ** -3, 'bwd': 2.0 ** -2, 'wgrad': 2.0 ** -4}     # y, dxn, dW_qkv / dW_out / db
PREFILL = 2.0 ** -14     # fp32 accumulation into a prefilled gradient: one rounding of the prefill
GUARD_BF16 = 0x7FBF            # a NaN bit pattern: an unwritten output element fails every bound


# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`); distinct keys per workload:
#   darcy_train_b32: conv 81, wgrad 34, laf 6
#   darcy_sample_b16: conv 38, wgrad 0, laf 2
#   darcy_sample_b64: conv 38, wgrad 0, laf 2
#   darcy_sample_b256: conv 38, wgrad 0, laf 2
#   darcy_sample_ddim0_b16: conv 38, wgrad 0, laf 2
#   mech_train_b32: conv 87, wgrad 37, laf 0
#   distinct: conv 282, wgrad 71, laf 12
# ----------------------------------------------------------------------------------------------------------------------
# conv: B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed, bias, residual, gn_sums, gn_groups, gn_sums_zeroed
CONV_TABLE = [
    (16, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (16, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (32, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 512, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 512, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 128, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 512, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 256, 8, 8, 1024, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 256, 8, 8, 1024, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 8, 8, 512, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 512, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 512, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 512, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 1024, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 1024, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 2048, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 8, 8, 2048, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 16, 16, 512, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 512, 16, 16, 512, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 768, 8, 8, 128, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 768, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 8, 8, 768, 8, 8, 512, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 768, 8, 8, 1024, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 512, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 512, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 1024, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 1024, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 1024, 8, 8, 1024, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 8, 8, 2048, 8, 8, 512, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 8, 8, 2048, 8, 8, 512, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 16, 16, 64, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 64, 16, 16, 256, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 16, 16, 64, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 16, 16, 64, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 16, 16, 128, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 256, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 512, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 512, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 1024, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 16, 16, 1024, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 32, 32, 256, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 256, 32, 32, 256, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 8, 8, 512, 4, 4, 2, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 8, 8, 512, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 256, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 512, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 512, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 512, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 16, 16, 512, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 768, 16, 16, 64, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 768, 16, 16, 128, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 16, 16, 768, 16, 16, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 768, 16, 16, 512, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 1024, 16, 16, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 16, 16, 1024, 16, 16, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 128, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 128, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 32, 32, 32, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 32, 32, 32, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 32, 32, 64, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 32, 32, 128, 32, 32, 128, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 128, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 512, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 512, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 64, 64, 128, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 128, 64, 64, 128, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 16, 16, 256, 4, 4, 2, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 16, 16, 256, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 256, 32, 32, 128, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 128, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 32, 32, 256, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 512, 32, 32, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 512, 32, 32, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 32, 32, 768, 32, 32, 64, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 32, 32, 768, 32, 32, 128, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 32, 32, 768, 32, 32, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 32, 64, 64, 64, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 32, 64, 64, 64, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 32, 64, 64, 128, 7, 7, 1, 3, 0, 1, 0, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_train_b32
    (32, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_train_b32
    (32, 64, 64, 128, 32, 32, 128, 4, 4, 2, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 32, 32, 128, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 128, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 128, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 256, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 256, 3, 3, 1, 1, 0, 0, 1, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 128, 64, 64, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 256, 64, 64, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # mech_train_b32
    (32, 64, 64, 256, 64, 64, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # mech_train_b32
    (32, 64, 64, 768, 64, 64, 128, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # mech_train_b32
    (64, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (64, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0, 0, 0, 0),  # darcy_sample_b64
    (64, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b64
    (64, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b64
    (256, 8, 8, 128, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 8, 8, 128, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 128, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 8, 8, 128, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 128, 16, 16, 128, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 256, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 8, 8, 256, 8, 8, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 512, 8, 8, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 8, 8, 512, 8, 8, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 16, 16, 64, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 64, 32, 32, 64, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 128, 8, 8, 128, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 128, 16, 16, 128, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 16, 16, 128, 16, 16, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 256, 16, 16, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 16, 16, 256, 16, 16, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 16, 16, 256, 16, 16, 128, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 32, 32, 32, 64, 64, 32, 4, 4, 2, 1, 1, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 64, 16, 16, 64, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 32, 32, 64, 32, 32, 768, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 128, 32, 32, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 32, 32, 128, 32, 32, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 32, 32, 256, 32, 32, 64, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 64, 64, 32, 32, 32, 32, 4, 4, 2, 1, 0, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 64, 64, 32, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
    (256, 64, 64, 32, 64, 64, 32, 7, 7, 1, 3, 0, 1, 0, 0, 0, 0),  # darcy_sample_b256
    (256, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0),  # darcy_sample_b256
    (256, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 0, 1, 0, 1, 8, 1),  # darcy_sample_b256
]
# wgrad: B, HA, WA, CA, CA_real, GH, GW, CB, KH, KW, a_stride, pad, s_row, s_col
WGRAD_TABLE = [
    (32, 8, 8, 128, 128, 8, 8, 128, 3, 3, 1, 1, 9, 1152),  # darcy_train_b32
    (32, 8, 8, 128, 128, 8, 8, 256, 1, 1, 1, 0, 1, 128),  # darcy_train_b32
    (32, 8, 8, 128, 128, 8, 8, 256, 3, 3, 1, 1, 9, 1152),  # darcy_train_b32
    (32, 8, 8, 128, 128, 8, 8, 768, 1, 1, 1, 0, 1, 128),  # darcy_train_b32
    (32, 8, 8, 256, 256, 8, 8, 128, 1, 1, 1, 0, 1, 256),  # darcy_train_b32
    (32, 8, 8, 256, 256, 8, 8, 256, 1, 1, 1, 0, 1, 256),  # darcy_train_b32
    (32, 8, 8, 256, 256, 8, 8, 256, 3, 3, 1, 1, 9, 2304),  # darcy_train_b32
    (32, 8, 8, 256, 256, 8, 8, 512, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 8, 8, 256, 256, 8, 8, 768, 1, 1, 1, 0, 1, 256),  # darcy_train_b32
    (32, 8, 8, 256, 256, 8, 8, 1024, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 128, 1, 1, 1, 0, 1, 512),  # darcy_train_b32
    (32, 8, 8, 512, 512, 8, 8, 128, 3, 3, 1, 1, 9, 4608),  # darcy_train_b32
    (32, 8, 8, 512, 512, 8, 8, 512, 3, 3, 1, 1, 9, 4608),  # mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 768, 1, 1, 1, 0, 1, 512),  # mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 1024, 1, 1, 1, 0, 1, 512),  # mech_train_b32
    (32, 8, 8, 512, 512, 8, 8, 1024, 3, 3, 1, 1, 9, 4608),  # mech_train_b32
    (32, 8, 8, 1024, 1024, 8, 8, 768, 1, 1, 1, 0, 1, 1024),  # mech_train_b32
    (32, 8, 8, 1024, 1024, 8, 8, 1024, 3, 3, 1, 1, 9, 9216),  # mech_train_b32
    (32, 8, 8, 2048, 2048, 8, 8, 512, 1, 1, 1, 0, 1, 2048),  # mech_train_b32
    (32, 8, 8, 2048, 2048, 8, 8, 512, 3, 3, 1, 1, 9, 18432),  # mech_train_b32
    (32, 16, 16, 64, 64, 16, 16, 64, 3, 3, 1, 1, 9, 576),  # darcy_train_b32
    (32, 16, 16, 64, 64, 16, 16, 128, 1, 1, 1, 0, 1, 64),  # darcy_train_b32
    (32, 16, 16, 64, 64, 16, 16, 128, 3, 3, 1, 1, 9, 576),  # darcy_train_b32
    (32, 16, 16, 64, 64, 16, 16, 768, 1, 1, 1, 0, 1, 64),  # darcy_train_b32
    (32, 16, 16, 128, 128, 8, 8, 128, 4, 4, 2, 1, 16, 2048),  # darcy_train_b32
    (32, 16, 16, 128, 128, 16, 16, 128, 3, 3, 1, 1, 9, 1152),  # darcy_train_b32
    (32, 16, 16, 128, 128, 16, 16, 768, 1, 1, 1, 0, 1, 128),  # darcy_train_b32
    (32, 16, 16, 256, 256, 16, 16, 64, 1, 1, 1, 0, 1, 256),  # darcy_train_b32
    (32, 16, 16, 256, 256, 16, 16, 64, 3, 3, 1, 1, 9, 2304),  # darcy_train_b32
    (32, 16, 16, 256, 256, 16, 16, 128, 1, 1, 1, 0, 1, 256),  # darcy_train_b32
    (32, 16, 16, 256, 256, 16, 16, 256, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 256, 3, 3, 1, 1, 9, 2304),  # mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 512, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 512, 3, 3, 1, 1, 9, 2304),  # mech_train_b32
    (32, 16, 16, 256, 256, 16, 16, 768, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 16, 16, 512, 512, 8, 8, 512, 4, 4, 2, 1, 16, 8192),  # mech_train_b32
    (32, 16, 16, 512, 512, 16, 16, 512, 3, 3, 1, 1, 9, 4608),  # mech_train_b32
    (32, 16, 16, 512, 512, 16, 16, 768, 1, 1, 1, 0, 1, 512),  # mech_train_b32
    (32, 16, 16, 1024, 1024, 16, 16, 256, 1, 1, 1, 0, 1, 1024),  # mech_train_b32
    (32, 16, 16, 1024, 1024, 16, 16, 256, 3, 3, 1, 1, 9, 9216),  # mech_train_b32
    (32, 32, 32, 32, 32, 32, 32, 32, 3, 3, 1, 1, 9, 288),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 32, 64, 1, 1, 1, 0, 1, 32),  # darcy_train_b32
    (32, 32, 32, 32, 32, 32, 32, 64, 3, 3, 1, 1, 9, 288),  # darcy_train_b32
    (32, 32, 32, 64, 64, 16, 16, 64, 4, 4, 2, 1, 16, 1024),  # darcy_train_b32
    (32, 32, 32, 64, 64, 32, 32, 64, 3, 3, 1, 1, 9, 576),  # darcy_train_b32
    (32, 32, 32, 64, 64, 32, 32, 768, 1, 1, 1, 0, 1, 64),  # darcy_train_b32
    (32, 32, 32, 128, 128, 32, 32, 32, 1, 1, 1, 0, 1, 128),  # darcy_train_b32
    (32, 32, 32, 128, 128, 32, 32, 32, 3, 3, 1, 1, 9, 1152),  # darcy_train_b32
    (32, 32, 32, 128, 128, 32, 32, 128, 3, 3, 1, 1, 9, 1152),  # mech_train_b32
    (32, 32, 32, 128, 128, 32, 32, 256, 1, 1, 1, 0, 1, 128),  # mech_train_b32
    (32, 32, 32, 128, 128, 32, 32, 256, 3, 3, 1, 1, 9, 1152),  # mech_train_b32
    (32, 32, 32, 128, 128, 32, 32, 768, 1, 1, 1, 0, 1, 128),  # mech_train_b32
    (32, 32, 32, 256, 256, 16, 16, 256, 4, 4, 2, 1, 16, 4096),  # mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 64, 1, 1, 1, 0, 1, 256),  # darcy_train_b32
    (32, 32, 32, 256, 256, 32, 32, 128, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 256, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 256, 3, 3, 1, 1, 9, 2304),  # mech_train_b32
    (32, 32, 32, 256, 256, 32, 32, 768, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 32, 32, 512, 512, 32, 32, 128, 1, 1, 1, 0, 1, 512),  # mech_train_b32
    (32, 32, 32, 512, 512, 32, 32, 128, 3, 3, 1, 1, 9, 4608),  # mech_train_b32
    (32, 64, 64, 32, 2, 64, 64, 32, 7, 7, 1, 3, 49, 98),  # darcy_train_b32
    (32, 64, 64, 32, 10, 64, 64, 128, 7, 7, 1, 3, 49, 490),  # mech_train_b32
    (32, 64, 64, 32, 32, 32, 32, 32, 4, 4, 2, 1, 16, 512),  # darcy_train_b32
    (32, 64, 64, 32, 32, 64, 64, 32, 3, 3, 1, 1, 9, 288),  # darcy_train_b32
    (32, 64, 64, 64, 64, 64, 64, 32, 1, 1, 1, 0, 1, 64),  # darcy_train_b32
    (32, 64, 64, 64, 64, 64, 64, 32, 3, 3, 1, 1, 9, 576),  # darcy_train_b32
    (32, 64, 64, 128, 128, 32, 32, 128, 4, 4, 2, 1, 16, 2048),  # mech_train_b32
    (32, 64, 64, 128, 128, 64, 64, 128, 3, 3, 1, 1, 9, 1152),  # mech_train_b32
    (32, 64, 64, 128, 128, 64, 64, 768, 1, 1, 1, 0, 1, 128),  # mech_train_b32
    (32, 64, 64, 256, 256, 64, 64, 128, 1, 1, 1, 0, 1, 256),  # mech_train_b32
    (32, 64, 64, 256, 256, 64, 64, 128, 3, 3, 1, 1, 9, 2304),  # mech_train_b32
]
# linear-attention block: kernel, B, N, qkv_stride_n, qkv_stride_c, out_stride_n, out_stride_c
LAF_TABLE = [
    ('bwd', 32, 1024, 0, 0, 0, 0),  # darcy_train_b32
    ('bwd', 32, 4096, 0, 0, 0, 0),  # darcy_train_b32
    ('fwd', 16, 1024, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    ('fwd', 16, 4096, 0, 0, 0, 0),  # darcy_sample_b16 darcy_sample_ddim0_b16
    ('fwd', 32, 1024, 0, 0, 0, 0),  # darcy_train_b32
    ('fwd', 32, 4096, 0, 0, 0, 0),  # darcy_train_b32
    ('fwd', 64, 1024, 0, 0, 0, 0),  # darcy_sample_b64
    ('fwd', 64, 4096, 0, 0, 0, 0),  # darcy_sample_b64
    ('fwd', 256, 1024, 0, 0, 0, 0),  # darcy_sample_b256
    ('fwd', 256, 4096, 0, 0, 0, 0),  # darcy_sample_b256
    ('wgrad', 32, 1024, 32, 1, 256, 1),  # darcy_train_b32
    ('wgrad', 32, 4096, 32, 1, 256, 1),  # darcy_train_b32
]
TABLES = {'conv': CONV_TABLE, 'wgrad': WGRAD_TABLE, 'laf': LAF_TABLE}

# rows no benchmarked step produces, for planner branches the workloads do not reach (see test_plan_coverage)
CONV_SYNTHETIC = [
    (3, 8, 8, 256, 8, 8, 256, 3, 3, 1, 1, 0, 1, 1, 1, 8, 0),       # odd batch, TN = 2: masked rows of the last tile
]
WGRAD_SYNTHETIC = [
]
LAF_SYNTHETIC = [
    ('fwd', 5, 4096, 0, 0, 0, 0), ('bwd', 5, 4096, 0, 0, 0, 0), ('wgrad', 5, 4096, 32, 1, 256, 1),
    ('fwd', 24, 4096, 0, 0, 0, 0), ('bwd', 24, 4096, 0, 0, 0, 0), ('wgrad', 24, 4096, 32, 1, 256, 1),
]


def conv_id(k):
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p, tr, hb, hr, hg, G, z = k
    t = f'B{B}_{H}x{W}_{Cin}to{Cout}_k{KH}s{s}p{p}' + ('T' if tr else '')
    return t + ('_bias' if hb else '') + ('_res' if hr else '') + (f'_gn{G}z{z}' if hg else '')


def wgrad_id(k):
    B, HA, WA, CA, CAr, GH, GW, CB, KH, KW, s, p, sr, sc = k
    return f'B{B}_a{HA}x{WA}x{CA}r{CAr}_g{GH}x{GW}x{CB}_k{KH}s{s}p{p}_w{sr}.{sc}'


def laf_id(k):
    kind, B, N, sn, sc, osn, osc = k
    return f'{kind}_B{B}_N{N}' + (f'_w{sn}.{sc}_o{osn}.{osc}' if kind == 'wgrad' else '')


# ----------------------------------------------------------------------------------------------------------------------
# census
# ----------------------------------------------------------------------------------------------------------------------
def test_census_is_covered_by_the_table():
    assert_census_in_tables(TABLES)


def test_every_table_row_is_produced_by_the_census():
    assert_tables_in_census(TABLES)


# ----------------------------------------------------------------------------------------------------------------------
# operands, references, predicates
# ----------------------------------------------------------------------------------------------------------------------
def _randn(g, *shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _guarded(n, fill_bits):
    """n bf16 elements inside a buffer with guard regions on both sides, all set to the bit pattern fill_bits"""
    guard = max(4096, n // 8) // 64 * 64
    buf = torch.full((n + 2 * guard,), fill_bits, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    return buf, buf[guard:guard + n], guard


def _guards_intact(buf, guard, n, fill_bits):
    b = buf.view(torch.int16)
    return bool((b[:guard] == fill_bits).all() and (b[guard + n:] == fill_bits).all())


def plan_conv(k):
    from physicsinformeddiffusionmodels_b200._lib import call
    out = torch.zeros(10, dtype=torch.int32)
    rc = call('pidm_conv2d_tc_plan', *k[:12], out.data_ptr())
    assert rc == 0, f'no tensor-core plan for {k}'
    BN, BK, rg, resident, stages, tiles, grid, TN, TH, TW = out.tolist()
    return dict(BN=BN, BK=BK, rg=rg, resident=resident, stages=stages, tiles=tiles, grid=grid, TN=TN, TH=TH, TW=TW)


def plan_wgrad(k):
    from physicsinformeddiffusionmodels_b200._lib import call
    out = torch.zeros(12, dtype=torch.int32)
    rc = call('pidm_conv2d_wgrad_tc_plan', *k, out.data_ptr())
    assert rc == 0, f'no tensor-core wgrad plan for {k}'
    v = out.tolist()
    return dict(w3=v[0], NP=v[1], AA=v[2], AB=v[3], splits=v[4], tps=v[5], n_pix_tiles=v[6], ctas=v[7], rg=v[8],
                TN=v[9], TH=v[10], TW=v[11])


def plan_laf(B, N):
    from physicsinformeddiffusionmodels_b200._lib import call
    out = torch.zeros(5, dtype=torch.int32)
    assert call('pidm_linattn_block_plan', B, N, out.data_ptr()) == 0
    v = out.tolist()
    return dict(stat=v[0], ctx=v[1], fwd=v[2], bwd=v[3], wgrad=v[4])


# ---- convolution ------------------------------------------------------------------------------------------------------
class ConvCase:
    """operands + fp64 reference (r) + absolute-value reference (A) of one table row"""

    def __init__(self, k):
        B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p, tr, hb, hr, hg, G, z = k
        self.k, self.K = k, KH * KW * Cin
        g = gen(('conv',) + tuple(k))
        self.x = _randn(g, B, H, W, Cin)
        self.wp = _randn(g, Cout, self.K, scale=1.0 / math.sqrt(self.K))
        self.bias = torch.randn(Cout, generator=g, device=DEV) if hb else None
        self.res = _randn(g, B, Ho, Wo, Cout) if hr else None
        d = lambda t: None if t is None else t.double()
        self.r = conv_ref(d(self.x), d(self.wp), d(self.bias), d(self.res), k)
        self.A = conv_ref(d(self.x).abs(), d(self.wp).abs(), None if self.bias is None else d(self.bias).abs(),
                          None if self.res is None else d(self.res).abs(), k)

    def acc_bound(self):
        return C_ACC * math.sqrt(self.K) * 2.0 ** -24 * self.A

    def ratio(self, y):
        """worst |y - r| / (2^-8 |r| + C_ACC sqrt(K) 2^-24 A) over all elements.  The first term is the exact worst case
        of one round-to-nearest bf16 rounding, reached by values just above a power of two, so on large tensors this
        ratio approaches 1 by construction; the margin lies in the accumulation term (acc_ratio)."""
        return ratio((y.double() - self.r).abs(), 2.0 ** -8 * self.r.abs() + self.acc_bound())

    def acc_ratio(self, y):
        """worst (|y - r| - 2^-8 |r|) / (C_ACC sqrt(K) 2^-24 A): the share of the accumulation term that is used"""
        return ratio(((y.double() - self.r).abs() - 2.0 ** -8 * self.r.abs()).clamp_min(0), self.acc_bound())

    def run(self):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p, tr, hb, hr, hg, G, z = self.k
        n = B * Ho * Wo * Cout
        buf, y, guard = _guarded(n, GUARD_BF16)
        sums = None
        if hg:
            sums = torch.zeros(B, G, 2, device=DEV) if z else torch.full((B, G, 2), 1.0e6, device=DEV)
        call('pidm_conv2d_tc_general', self.x, self.wp, self.bias, self.res, y, B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p,
             tr, sums, G if hg else 0, z, stream())
        torch.cuda.synchronize()
        return buf, y.view(B, Ho, Wo, Cout), guard, n, sums

    def gn_ratio(self, sums):
        """fused GroupNorm statistics vs fp64 sums of the exact output: per (sample, group) sum and sum of squares"""
        B, Ho, Wo, Cout, G = self.k[0], self.k[4], self.k[5], self.k[6], self.k[15]
        r = self.r.reshape(B, Ho * Wo, G, Cout // G)
        e = self.acc_bound().reshape(r.shape)            # per-element error of the fp32 value the epilogue sums
        M = Ho * Wo * (Cout // G)
        c = C_ACC * math.sqrt(M) * 2.0 ** -24
        s1, s2 = r.sum(dim=(1, 3)), (r * r).sum(dim=(1, 3))
        b1 = e.sum(dim=(1, 3)) + c * r.abs().sum(dim=(1, 3))
        b2 = (2 * r.abs() * e + e * e).sum(dim=(1, 3)) + c * s2
        sd = sums.double()
        return max(ratio((sd[..., 0] - s1).abs(), b1), ratio((sd[..., 1] - s2).abs(), b2))


# ---- weight gradient --------------------------------------------------------------------------------------------------
def _wgrad_ref(a, b, k):
    """fp64 D[cA][cB][tap] = sum over grid pixels g of a[a_stride*g - pad + tap][cA] * b[g][cB] (a, b NHWC)"""
    B, HA, WA, CA, CAr, GH, GW, CB, KH, KW, s, p = k[:12]
    an = a.permute(0, 3, 1, 2)
    ph = max(0, s * (GH - 1) + KH - (HA + p))
    pw = max(0, s * (GW - 1) + KW - (WA + p))
    ap = F.pad(an, (p, pw, p, ph))
    D = torch.empty(CA, CB, KH * KW, dtype=a.dtype, device=a.device)
    for r in range(KH):
        for q in range(KW):
            sl = ap[:, :, r:r + s * (GH - 1) + 1:s, q:q + s * (GW - 1) + 1:s]
            D[:, :, r * KW + q] = torch.einsum('bchw,bhwd->cd', sl, b)
    return D


def _wgrad_index(k):
    B, HA, WA, CA, CAr, GH, GW, CB, KH, KW, s, p, sr, sc = k
    ca = torch.arange(CAr, device=DEV).view(-1, 1, 1)
    cb = torch.arange(CB, device=DEV).view(1, -1, 1)
    tap = torch.arange(KH * KW, device=DEV).view(1, 1, -1)
    return ca * sr + cb * sc + tap                        # [CA_real, CB, taps]


class WgradCase:
    def __init__(self, k):
        B, HA, WA, CA, CAr, GH, GW, CB, KH, KW, s, p, sr, sc = k
        self.k, self.K = k, B * GH * GW
        g = gen(('wgrad',) + tuple(k))
        self.a = _randn(g, B, HA, WA, CA)                    # padding channels (>= CA_real) are random: must be dropped
        self.b = _randn(g, B, GH, GW, CB)
        self.idx = _wgrad_index(k)
        self.n = int(self.idx.max().item()) + 1
        self.prefill = torch.randn(self.n, generator=g, device=DEV)
        self.D = _wgrad_ref(self.a.double(), self.b.double(), k)[:CAr]
        self.A = _wgrad_ref(self.a.double().abs(), self.b.double().abs(), k)[:CAr]

    def bound(self):
        return C_ACC * math.sqrt(self.K) * 2.0 ** -24 * (self.A + self.prefill.double()[self.idx].abs())

    def ratio(self, dw):
        """dw: the accumulated fp32 buffer (prefill + D) at the contract's positions"""
        got = dw.double()[self.idx] - self.prefill.double()[self.idx]
        return ratio((got - self.D).abs(), self.bound())

    def run(self):
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        guard = 4096
        buf = torch.randn(self.n + 2 * guard, generator=gen(('wgrad-guard',) + tuple(self.k)), device=DEV)
        buf[guard:guard + self.n] = self.prefill
        keep = buf.clone()
        dw = buf[guard:]
        call('pidm_conv2d_wgrad_tc', self.a, self.b, dw, *self.k, stream())
        torch.cuda.synchronize()
        touched = torch.zeros_like(buf, dtype=torch.bool)
        touched[guard + self.idx.reshape(-1)] = True
        untouched_ok = bool((buf[~touched] == keep[~touched]).all())
        return dw, untouched_ok


# ---- linear-attention block -------------------------------------------------------------------------------------------
def _ref(xn, wq, wo, bo, res, dy, need_grad, chunk=8):
    """fp64: y = res + bo + attention(xn Wq^T) Wo^T (reference unet_model.py:275-297 and the Residual wrapper's `+ x`),
    computed per group of samples, and with need_grad the gradients for the cotangent dy.
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
            q, k, v = (xr @ wqr.t()).view(nb, N, 3, 8, 32).permute(2, 0, 3, 4, 1)      # [nb, heads, 32, N]
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
    return A_ATT * r.abs() + B_ATT['fwd'] * rms


def dx_bound(r):                      # [B, N, 32]: slice = sample
    rms = r.pow(2).mean(dim=(1, 2), keepdim=True).sqrt()
    return A_ATT * r.abs() + B_ATT['bwd'] * rms


def gq_bound(r, prefill):             # [768, 32]: slice = the 32 rows of one (q | k | v, head)
    rh = r.view(24, 32, 32)
    rms = rh.pow(2).mean(dim=(1, 2), keepdim=True).sqrt()
    return (A_ATT * rh.abs() + B_ATT['wgrad'] * rms).view(768, 32) + PREFILL * prefill.abs()


def go_bound(r, prefill):             # [32, 256]: slice = one head's 32 columns
    rh = r.view(32, 8, 32)
    rms = rh.pow(2).mean(dim=(0, 2), keepdim=True).sqrt()
    return (A_ATT * rh.abs() + B_ATT['wgrad'] * rms).view(32, 256) + PREFILL * prefill.abs()


def db_bound(r, prefill):             # [32]: slice = the whole vector
    return A_ATT * r.abs() + B_ATT['wgrad'] * r.pow(2).mean().sqrt() + PREFILL * prefill.abs()


class BlockCase:
    """operands + fp64 reference of one attention row: a fwd row checks y, a bwd row dxn, a wgrad row dW_qkv, dW_out and
    the bias gradient"""

    def __init__(self, k):
        kind, B, N = k[:3]
        self.k = k
        g = gen(('linattn-block', B, N))                   # same operands for the fwd / bwd / wgrad rows of a shape
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
            self.xn, self.wq, self.wo, self.bo, self.res, self.dy, kind != 'fwd')

    def run(self):
        """launches fwd (and bwd / wgrad as the row asks); returns {output: worst |err| / bound} and whether every
        element outside the outputs (guard regions, the rest of the gradient buffer) survived"""
        from physicsinformeddiffusionmodels_b200._lib import call, stream
        kind, B, N, sn, sc, osn, osc = self.k
        ctx = torch.empty(B, 8, 32, 32, device=DEV)
        kmax, kzinv = torch.empty(B, 8, 32, device=DEV), torch.empty(B, 8, 32, device=DEV)
        ws = torch.empty(call('pidm_linattn_block_workspace_floats', B, N), device=DEV)
        n = B * N * 32
        buf, y, guard = _guarded(n, GUARD_BF16)
        call('pidm_linattn_block_fwd', self.xn, self.wq, self.wo, self.bo, self.res, y, ctx, kmax, kzinv, ws, B, N,
             stream())
        if kind == 'fwd':
            torch.cuda.synchronize()
            return {'y': self.y_ratio(y.view(B, N, 32))}, _guards_intact(buf, guard, n, GUARD_BF16)
        buf, dx, guard = _guarded(n, GUARD_BF16)
        dctx = torch.empty_like(ctx)
        call('pidm_linattn_block_bwd', self.xn, self.wq, self.wo, self.dy, ctx, kmax, kzinv, dx, dctx, B, N, stream())
        if kind == 'bwd':
            torch.cuda.synchronize()
            r = ratio((dx.view(B, N, 32).double() - self.dx_r).abs(), dx_bound(self.dx_r))
            return {'dxn': r}, _guards_intact(buf, guard, n, GUARD_BF16)
        # both weight gradients accumulate into strided views of one prefilled flat buffer (as the engine's flat
        # gradient buffer), and pidm_colsum the bias gradient into the same buffer
        g = gen(('linattn-block-gw', B, N))
        guard = 1024
        nq, no = 767 * sn + 31 * sc + 1, 31 * osn + 255 * osc + 1
        oq, oo, ob = guard, 2 * guard + nq, 3 * guard + nq + no
        gbuf = torch.randn(ob + 32 + guard, generator=g, device=DEV)
        keep = gbuf.clone()

        def views(t):
            return (torch.as_strided(t, (768, 32), (sn, sc), oq), torch.as_strided(t, (32, 256), (osn, osc), oo),
                    t[ob:ob + 32])
        gq, go, gb = views(gbuf)
        call('pidm_linattn_block_wgrad', self.xn, self.wq, self.wo, self.dy, ctx, dctx, kmax, kzinv, gq, sn, sc, go, osn,
             osc, B, N, stream())
        call('pidm_colsum', self.dy, gb, B * N, 32, 1, stream())
        torch.cuda.synchronize()
        touched = torch.zeros_like(gbuf, dtype=torch.bool)
        for v in views(touched):
            v.fill_(True)
        ok = bool((gbuf[~touched] == keep[~touched]).all())
        pq, po, pb = (v.double() for v in views(keep))
        return {'dWqkv': ratio((gq.double() - pq - self.gq_r).abs(), gq_bound(self.gq_r, pq)),
                'dWout': self.go_ratio(go.double() - po, po),
                'db': ratio((gb.double() - pb - self.db_r).abs(), db_bound(self.db_r, pb))}, ok

    def y_ratio(self, y):
        return ratio((y.double() - self.y_r).abs(), y_bound(self.y_r))

    def go_ratio(self, go, prefill):
        return ratio((go.double() - self.go_r).abs(), go_bound(self.go_r, prefill))


# ----------------------------------------------------------------------------------------------------------------------
# replay
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module', autouse=True)
def _bf16_mode():
    from physicsinformeddiffusionmodels_b200 import ops
    ops.set_precision('bf16')
    ops.set_tensor_core_conv(True)
    yield


CONV_ROWS = CONV_TABLE + CONV_SYNTHETIC
WGRAD_ROWS = WGRAD_TABLE + WGRAD_SYNTHETIC
LAF_ROWS = LAF_TABLE + LAF_SYNTHETIC


@pytest.mark.parametrize('k', CONV_ROWS, ids=[conv_id(k) for k in CONV_ROWS])
def test_conv_replay(k):
    c = ConvCase(k)
    buf, y, guard, n, sums = c.run()
    assert _guards_intact(buf, guard, n, GUARD_BF16), f'{conv_id(k)}: a store landed outside y'
    r = c.ratio(y)
    note('census', 'conv worst', r)
    note('census', 'conv_accumulation worst', c.acc_ratio(y))
    assert r <= 1.0, f'{conv_id(k)}: worst |err| / bound = {r:.3g} (plan {plan_conv(k)})'
    if k[14]:
        rg = c.gn_ratio(sums)
        note('census', 'gn_sums worst', rg)
        assert rg <= 1.0, f'{conv_id(k)}: fused GroupNorm statistics off, worst |err| / bound = {rg:.3g}'


@pytest.mark.parametrize('k', WGRAD_ROWS, ids=[wgrad_id(k) for k in WGRAD_ROWS])
def test_wgrad_replay(k):
    c = WgradCase(k)
    dw, untouched_ok = c.run()
    assert untouched_ok, f'{wgrad_id(k)}: an element outside the contract (guard, padding row cA >= CA_real) changed'
    r = c.ratio(dw)
    note('census', ('wgrad3' if plan_wgrad(k)['w3'] else 'wgrad') + ' worst', r)
    assert r <= 1.0, f'{wgrad_id(k)}: worst |err| / bound = {r:.3g} (plan {plan_wgrad(k)})'


@pytest.mark.parametrize('k', LAF_ROWS, ids=[laf_id(k) for k in LAF_ROWS])
def test_attention_block_replay(k):
    ratios, ok = BlockCase(k).run()
    assert ok, f'{laf_id(k)}: a store landed outside the outputs'
    for name, r in ratios.items():
        note('census', f'laf_{name} worst', r)
    assert max(ratios.values()) <= 1.0, f'{laf_id(k)}: worst |err| / bound = {ratios} (plan {plan_laf(k[1], k[2])})'


# ----------------------------------------------------------------------------------------------------------------------
# the predicates reject subtly wrong outputs (edits of the fp64 reference; no faulty code runs on the GPU)
# ----------------------------------------------------------------------------------------------------------------------
def _bf16(t):
    return t.to(torch.bfloat16)


def _largest_k_row():
    return max(CONV_ROWS, key=lambda k: (k[7] * k[8] * k[3], k[0]))


def _row(pred, rows):
    for k in rows:
        if pred(k):
            return k
    pytest.fail('no table row has the property this mutant needs')


def test_mutant_conv_dropped_k_slice():
    """one 32-channel K-slice of one tap missing, at the largest K of the table"""
    k = _largest_k_row()
    c = ConvCase(k)
    assert c.ratio(_bf16(c.r)) <= 1.0
    B, H, W, Cin, Ho, Wo, Cout, KH, KW = k[:9]
    tap, c0 = (KH * KW) // 2, Cin // 2 // 32 * 32
    wm = torch.zeros(Cout, KH * KW, Cin, dtype=torch.float64, device=DEV)
    wm[:, tap, c0:c0 + 32] = c.wp.double().view(Cout, KH * KW, Cin)[:, tap, c0:c0 + 32]
    part = conv_ref(c.x.double(), wm.view(Cout, -1), None, None, k)
    assert c.ratio(_bf16(c.r - part)) > 1.0, conv_id(k)


def test_mutant_conv_tile_replaced_by_neighbour():
    k = _row(lambda k: k[0] >= 16 and k[4] >= 32, CONV_ROWS)
    c = ConvCase(k)
    p = plan_conv(k)
    y = c.r.clone()
    TH, TW = p['TH'], p['TW']
    if k[5] >= 2 * TW:
        y[-1, :TH, :TW] = c.r[-1, :TH, TW:2 * TW]
    else:
        y[-1, :TH, :TW] = c.r[-1, TH:2 * TH, :TW]
    assert c.ratio(_bf16(y)) > 1.0, conv_id(k)


def test_mutant_conv_last_pixel_of_last_sample_zeroed():
    for k in (CONV_ROWS[0], CONV_SYNTHETIC[0]):
        c = ConvCase(k)
        y = c.r.clone()
        y[-1, -1, -1, :] = 0
        assert c.ratio(_bf16(y)) > 1.0, conv_id(k)


def test_mutant_conv_bias_missing_on_one_n_tile():
    k = _row(lambda k: k[12] and k[6] > plan_conv(k)['BN'], CONV_ROWS)
    c = ConvCase(k)
    BN = plan_conv(k)['BN']
    y = c.r.clone()
    y[..., BN:2 * BN] -= c.bias.double()[BN:2 * BN]
    assert c.ratio(_bf16(y)) > 1.0, conv_id(k)


def _split_partial(c, p, s):
    """contribution of the pixel tiles of split s to D"""
    B, HA, WA, CA, CAr, GH, GW = c.k[:7]
    bb = torch.arange(B, device=DEV).view(-1, 1, 1)
    hh = torch.arange(GH, device=DEV).view(1, -1, 1)
    ww = torch.arange(GW, device=DEV).view(1, 1, -1)
    tiles_h, tiles_w = GH // p['TH'], GW // p['TW']
    pt = ((bb // p['TN']) * tiles_h + hh // p['TH']) * tiles_w + ww // p['TW']
    mask = ((pt >= s * p['tps']) & (pt < (s + 1) * p['tps'])).to(torch.float64)
    return _wgrad_ref(c.a.double(), c.b.double() * mask[..., None], c.k)[:CAr]


def test_mutant_wgrad_split_partial_missing():
    for w3 in (0, 1):
        k = max((k for k in WGRAD_ROWS if plan_wgrad(k)['w3'] == w3 and plan_wgrad(k)['splits'] > 1),
                key=lambda k: plan_wgrad(k)['splits'])
        c = WgradCase(k)
        p = plan_wgrad(k)
        exact = c.prefill.clone()
        exact[c.idx.reshape(-1)] += c.D.reshape(-1).float()
        assert c.ratio(exact) <= 1.0
        part = _split_partial(c, p, p['splits'] - 1)
        mut = c.prefill.double().clone()
        mut[c.idx.reshape(-1)] += (c.D - part).reshape(-1)
        assert c.ratio(mut.float()) > 1.0, (wgrad_id(k), p)


def _ragged_fwd_row():
    return _row(lambda k: k[0] == 'fwd' and k[2] % plan_laf(k[1], k[2])['fwd'] != 0, LAF_ROWS)


def test_mutant_attention_block_last_chunk_from_previous_chunk():
    k = _ragged_fwd_row()
    c = BlockCase(k)
    N, px = k[2], plan_laf(k[1], k[2])['fwd']
    last = (N - 1) // px * px
    L = N - last
    y = c.y_r.clone()
    y[:, last:] = c.y_r[:, last - px:last - px + L]
    assert c.y_ratio(_bf16(c.y_r)) <= 1.0
    assert c.y_ratio(_bf16(y)) > 1.0, laf_id(k)


def test_mutant_attention_block_term_missing():
    """one head's partial, the bias or the residual missing from y"""
    k = _ragged_fwd_row()
    c = BlockCase(k)
    head = c.out_r[..., 3 * 32:4 * 32] @ c.wo.double()[:, 3 * 32:4 * 32].t()
    for name, term in (('one head partial', head), ('bias', c.bo.double()), ('residual', c.res.double())):
        assert c.y_ratio(_bf16(c.y_r - term)) > 1.0, (laf_id(k), name)


def test_mutant_attention_block_dw_out_head_transposed():
    k = _row(lambda k: k[0] == 'wgrad', LAF_ROWS)
    c = BlockCase(k)
    zero = torch.zeros(32, 256, dtype=torch.float64, device=DEV)
    assert c.go_ratio(c.go_r.float(), zero) <= 1.0
    go = c.go_r.clone()
    go[:, 32 * 5:32 * 6] = c.go_r[:, 32 * 5:32 * 6].t()
    assert c.go_ratio(go.float(), zero) > 1.0, laf_id(k)


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
TC_CASES = {(128, 64), (64, 64), (32, 64), (128, 32), (64, 32), (32, 32)}        # conv_tc.cu TC_CASE
WG_CASES = {(128, 64, 64), (128, 32, 64), (64, 64, 64), (64, 32, 64), (32, 64, 32), (32, 32, 32)}   # wgrad_tc.cu WG_CASE
W3_CASES = {(64, 64), (32, 32)}                                                   # wgrad_tc.cu W3_CASE


def conv_coverage():
    plans = [(k, plan_conv(k)) for k in CONV_ROWS]
    return {
        'BN x BK': {(p['BN'], p['BK']) for _, p in plans},
        'row-group': {p['rg'] for _, p in plans},
        'resident': {p['resident'] for _, p in plans},
        'transposed': {k[11] for k, _ in plans},
        'ragged persistent wave': any(p['tiles'] > p['grid'] and p['tiles'] % p['grid'] for _, p in plans),
        'odd B with TN=2': any(k[0] % 2 and p['TN'] == 2 for k, p in plans),
        'gn cpg': {k[6] // k[15] for k, _ in plans if k[14]},
    }


def wgrad_coverage():
    plans = [(k, plan_wgrad(k)) for k in WGRAD_ROWS]
    return {
        'generic NP x AA x AB': {(p['NP'], p['AA'], p['AB']) for _, p in plans if not p['w3']},
        'wgrad3 NP x AB': {(p['NP'], p['AB']) for _, p in plans if p['w3']},
        'wgrad3 row-group': {p['rg'] for _, p in plans if p['w3']},
        'short last split': any(p['tps'] > 1 and p['n_pix_tiles'] % p['tps'] for _, p in plans),
        'CA_real < CA': any(k[4] < k[3] for k, _ in plans),
    }


def laf_coverage():
    out = {}
    for kind in ('fwd', 'bwd', 'wgrad'):
        out[f'ragged last chunk ({kind})'] = any(
            k[0] == kind and k[2] % plan_laf(k[1], k[2])[kind] for k in LAF_ROWS)
    return out


def test_plan_coverage():
    cv, wg = conv_coverage(), wgrad_coverage()
    assert cv['BN x BK'] == TC_CASES, cv
    assert cv['row-group'] == {0, 1} and cv['resident'] == {0, 1} and cv['transposed'] == {0, 1}, cv
    assert cv['ragged persistent wave'] and cv['odd B with TN=2'], cv
    assert wg['generic NP x AA x AB'] == WG_CASES, wg
    assert wg['wgrad3 NP x AB'] == W3_CASES and wg['wgrad3 row-group'] == {0, 1}, wg
    assert wg['short last split'] and wg['CA_real < CA'], wg


def test_attention_block_plan_coverage():
    la = laf_coverage()
    assert all(la.values()), la

