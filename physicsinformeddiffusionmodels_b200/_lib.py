"""ctypes binding of libpidm.so (C ABI in include/pidm.h).

The library is REQUIRED: there is no fallback.  Import of this module raises if the shared object is
missing (run `python __graft_entry__.py` to build it) and every call raises RuntimeError with
pidm_last_error() when the library reports a failure."""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libpidm.so')

P = ctypes.c_void_p
I = ctypes.c_int
L = ctypes.c_longlong
F = ctypes.c_float
D = ctypes.c_double

# name -> argument ctypes (return type is always int unless noted)
_SIGS = {
    'pidm_qsample': [P, P, P, P, P, P, I, I, P],
    'pidm_posterior_step': [P, P, P, P, F, F, F, L, P],
    'pidm_scale': [P, P, P, L, P],
    'pidm_ddim_coefs': [P, P, P, P, P, P, P, P, P, I, P],
    'pidm_axpby_per_sample': [P, P, P, P, P, P, P, I, I, P],
    'pidm_toy_pidm_loss': [P, P, P, P, P, P, P, P, F, F, F, F, P, P, P, P, P, I, I, P],
    'pidm_fd_stencil': [P, P, I, I, I, F, F, P],
    'pidm_darcy_residual_fwd': [P, P, P, I, I, F, I, I, P],
    'pidm_darcy_residual_bwd': [P, P, P, P, I, I, F, I, I, P],
    'pidm_darcy_jacobian_max': [P, P, I, I, F, I, I, P],
    'pidm_darcy_cocogen': [P, P, P, P, I, I, I, I, F, I, I, P],
    'pidm_darcy_abs_residual_grad': [P, P, P, I, L, I, F, I, I, P],
    'pidm_darcy_pidm_loss': [P, P, P, P, P, P, P, F, F, P, P, P, I, I, F, I, I, P],
    'pidm_nchw_to_nhwc': [P, P, I, I, I, I, I, P],
    'pidm_cond_embed_fwd': [P, P, P, P, P, I, I, I, I, P],
    'pidm_cond_embed_wgrad': [P, P, P, P, P, P, P, I, I, I, I, P],
    'pidm_concat_channels': [P, P, P, L, I, I, I, P],
    'pidm_split_channels': [P, P, P, L, I, I, I, P],
    'pidm_wrap_pad_nhwc': [P, P, I, I, I, I, I, I, P],
    'pidm_pack_entry_size': [],
    'pidm_pack_weights': [P, I, I, P],
    'pidm_pack_pair_entry_size': [],
    'pidm_pack_weights_pairs': [P, P, I, I, I, I, P],
    'pidm_conv2d_simt': [P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, I, I, I, P],
    'pidm_conv2d_wgrad_simt': [P, P, P, P, I, I, I, I, I, I, I, I, I, I, I, I, I, L, L, I, P],
    'pidm_conv2d_tc_general': [P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, I, I, P, I, I, P],
    'pidm_conv2d_tc_general_supported': [I, I, I, I, I, I, I, I, I, I, I, I],
    'pidm_conv2d_tc_plan': [I, I, I, I, I, I, I, I, I, I, I, I, P],
    'pidm_conv2d_wgrad_tc': [P, P, P, I, I, I, I, I, I, I, I, I, I, I, I, L, L, P],
    'pidm_conv2d_wgrad_tc_supported': [I, I, I, I, I, I, I, I],
    'pidm_conv2d_wgrad_tc_plan': [I, I, I, I, I, I, I, I, I, I, I, I, L, L, P],
    'pidm_colsum': [P, P, L, I, I, P],
    'pidm_groupnorm_silu_fwd': [P, P, P, P, P, P, P, I, I, I, I, I, F, I, P],
    'pidm_groupnorm_silu_bwd': [P, P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, F, I, P],
    'pidm_groupnorm_plan': [I, I, I, I, I, P],
    'pidm_layernorm_c_fwd': [P, P, P, L, I, F, I, P],
    'pidm_layernorm_c_bwd': [P, P, P, P, P, P, L, I, F, I, P],
    'pidm_linattn_workspace_floats': [I, I, I],
    'pidm_linattn_block_supported': [I, I, I, I],
    'pidm_linattn_block_workspace_floats': [I, I],
    'pidm_linattn_block_plan': [I, I, P],
    'pidm_linattn_block_fwd': [P, P, P, P, P, P, P, P, P, P, I, I, P],
    'pidm_linattn_block_bwd': [P, P, P, P, P, P, P, P, P, I, I, P],
    'pidm_linattn_block_wgrad': [P, P, P, P, P, P, P, P, P, L, L, P, L, L, I, I, P],
    'pidm_linattn_fwd': [P, P, P, P, P, P, I, I, I, I, P],
    'pidm_linattn_bwd': [P, P, P, P, P, P, P, I, I, I, I, P],
    'pidm_linattn_plan': [I, I, I, I, P],
    'pidm_attn_fwd': [P, P, I, I, I, I, P],
    'pidm_attn_bwd': [P, P, P, I, I, I, I, P],
    'pidm_time_embed_fwd': [P, P, P, P, P, P, P, P, P, I, I, I, P],
    'pidm_time_embed_bwd': [P, P, P, P, P, P, P, P, P, P, I, I, I, I, P],
    'pidm_mlp_entry_size': [],
    'pidm_block_mlps_fwd': [P, I, I, P, I, I, P],
    'pidm_block_mlps_bwd': [P, I, I, P, P, I, I, I, P],
    'pidm_head_fwd': [P, P, P, P, I, I, I, I, I, I, P],
    'pidm_head_bwd': [P, P, P, P, P, P, P, I, I, I, I, I, I, P],
    'pidm_sumsq': [P, L, P, P, P],
    'pidm_adam_ema_step': [P, P, P, P, P, L, F, D, D, F, I, P, P, F, F, F, I, I, P],
    'pidm_swap_f32': [P, P, L, P],
    'pidm_mechanics_residual_fwd': [P, P, P, P, P, P, I, I, P],
    'pidm_mechanics_residual_bwd': [P, P, P, P, P, P, P, P, P, I, I, P],
    'pidm_mech_pidm_loss': [P, P, P, P, P, P, P, P, P, F, F, F, F, P, P, P, P, P, I, I, P],
    'pidm_bilinear_resize_fwd': [P, P, I, I, I, P],
    'pidm_bilinear_resize_bwd': [P, P, I, I, I, P],
    'pidm_mech_sample_input': [P, P, P, I, I, I, P],
    'pidm_mech_posterior_step': [P, P, P, P, P, P, P, P, I, I, P],
    'pidm_mech_fem_pcg': [P, P, P, P, P, P, D, I, I, I, P],
    'pidm_mech_floating_material': [P, P, I, I, P],
    'pidm_darcy_gen_kle': [P, P, P, I, I, I, P],
    'pidm_darcy_gen_workspace_bytes': [I, I],
    'pidm_darcy_gen_solve': [P, P, P, P, P, P, L, I, I, D, I, I, I, P],
    'pidm_version': [],
}
_RESTYPES = {'pidm_darcy_gen_workspace_bytes': ctypes.c_longlong}
# functions whose int return value is a result, not an error code
_VALUE_RETURN = {'pidm_pack_entry_size', 'pidm_pack_pair_entry_size', 'pidm_mlp_entry_size', 'pidm_linattn_workspace_floats', 'pidm_version',
                 'pidm_linattn_block_supported', 'pidm_linattn_block_workspace_floats',
                 'pidm_conv2d_tc_supported', 'pidm_conv2d_wgrad_tc_supported', 'pidm_conv2d_tc_general_supported',
                 'pidm_conv2d_tc_plan', 'pidm_conv2d_wgrad_tc_plan', 'pidm_linattn_block_plan', 'pidm_groupnorm_plan',
                 'pidm_linattn_plan',
                 'pidm_darcy_gen_workspace_bytes'}

if not os.path.exists(LIB_PATH):
    raise ImportError(f'{LIB_PATH} is missing: build it with `python __graft_entry__.py` (nvcc, sm_90a). '
                      'There is no CPU / PyTorch fallback for the PIDM hot path.')

_lib = ctypes.CDLL(LIB_PATH)
_lib.pidm_last_error.restype = ctypes.c_char_p
_lib.pidm_last_error.argtypes = []
for _n, _a in _SIGS.items():
    _f = getattr(_lib, _n)          # AttributeError here == header/library mismatch
    _f.argtypes = _a
    _f.restype = _RESTYPES.get(_n, ctypes.c_int)

launch_count = 0     # number of libpidm entry-point calls (each issues >= 1 kernel); read by bench.py


def exported_symbols():
    return sorted(_SIGS) + ['pidm_last_error']


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    """Call a libpidm entry point; tensors are passed as raw device pointers."""
    global launch_count
    conv = []
    for a in args:
        if isinstance(a, torch.Tensor):
            conv.append(a.data_ptr())
        else:
            conv.append(a)
    rc = getattr(_lib, name)(*conv)
    if name in _VALUE_RETURN:
        return rc
    launch_count += 1
    if rc != 0:
        raise RuntimeError(f'{name} failed (code {rc}): {_lib.pidm_last_error().decode()}')
    return 0


DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1}
