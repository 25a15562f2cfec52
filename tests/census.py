"""The census of the benchmarked and sampling steps, shared by the eight per-element census files
(tests/test_gpu_*_census.py).

One eager step of every workload bench.py times (Darcy training at batch 32, one Darcy sampling step at batch 16 / 64 /
256 in mean mode and at batch 16 in sample mode with ddim_steps = 0, mechanics training at batch 32 with Unet3D(dim=128))
is run with the C ABI's `call` swapped for a recorder, which keeps every entry point called and, for the entry points in
KEYS, the distinct (family, key) pairs of their arguments.  Keys are integer and flag arguments, which optional pointers
are set and geometry decoded from device tables, never pointers.  There are three recordings: census() runs the
workloads as bench.py does (bf16), census_exact() runs them and the guidance and circular training steps in the fp32
exact mode that every oracle-parity test uses, where every convolution runs on the CUDA-core kernels of conv_simt.cu,
and census_sampling() runs one step of each sampling-side workload the package offers beside them (DDIM walks, CoCoGen
corrections, the drop-in p_sample, conditional mechanics sampling and the toy study) in bf16.  Each census file commits
one table per family and checks it against its recording (RECORDING) both ways; `python tests/census.py --print-table`
regenerates every table.  The product package is imported inside the functions, so importing this module builds
nothing."""
import functools
import os
import sys

import numpy as np
import torch

from checks import DTYPE, NAME

DEV = 'cuda'


# ----------------------------------------------------------------------------------------------------------------------
# keys: entry point -> [(family, key)] of one call (a: the arguments, stream last)
# ----------------------------------------------------------------------------------------------------------------------
def _has(t):
    return int(t is not None)


def _dt(code):
    return NAME[DTYPE[int(code)]]


def _decode(table_dev, dt, n):
    return np.frombuffer(table_dev.cpu().numpy().tobytes(), dtype=dt)[:n]


def _mlp_rows(a):
    from physicsinformeddiffusionmodels_b200 import packing
    return tuple(int(r['n']) for r in _decode(a[0], packing._MLP_DT, int(a[1])))


def _pack_keys(a):
    from physicsinformeddiffusionmodels_b200 import packing
    return [('pack', (int(a[2]), int(r['N']), int(r['C']), int(r['Cpad']), int(r['taps']), int(r['flip']),
                      int(r['s_n']), int(r['s_c']))) for r in _decode(a[0], packing._PACK_DT, int(a[1]))]


def _pair_keys(a):
    from physicsinformeddiffusionmodels_b200 import packing
    tile_base, n_tiles = int(a[2]), int(a[3])
    tmap = a[1].cpu().numpy().view(np.int32)
    used = sorted(set(tmap[tile_base:tile_base + n_tiles].tolist()))
    rows = _decode(a[0], packing._PAIR_DT, max(used) + 1)
    keys = [('pair_launch', (int(a[5]), tile_base, n_tiles, int(a[4])))]
    for i in used:
        r = rows[i]
        keys.append(('pair', (int(a[5]), int(r['Cout']), int(r['Cin']), int(r['taps']), int(r['flip']),
                              int(int(r['s_ci']) == int(r['taps'])), int(int(r['dst_d']) != 0))))
    return keys


def _darcy_key(fam, i):
    return lambda a: [(fam, (int(a[i]), int(a[i + 1]), float(a[i + 2]), int(a[i + 3]), int(a[i + 4])))]


KEYS = {
    # test_gpu_launch_census.py
    'pidm_conv2d_tc_general': lambda a: [('conv', tuple(int(v) for v in a[5:17]) + (
        _has(a[2]), _has(a[3]), _has(a[17]), int(a[18]), int(a[19])))],
    'pidm_conv2d_wgrad_tc': lambda a: [('wgrad', tuple(int(v) for v in a[3:17]))],
    'pidm_linattn_block_fwd': lambda a: [('laf', ('fwd', int(a[10]), int(a[11]), 0, 0, 0, 0))],
    'pidm_linattn_block_bwd': lambda a: [('laf', ('bwd', int(a[9]), int(a[10]), 0, 0, 0, 0))],
    'pidm_linattn_block_wgrad': lambda a: [('laf', ('wgrad', int(a[14]), int(a[15]), int(a[9]), int(a[10]), int(a[12]),
                                                    int(a[13])))],
    # test_gpu_norm_census.py
    'pidm_groupnorm_silu_fwd': lambda a: [('gn_fwd', (int(a[8]), int(a[9]), int(a[10]), int(a[11]), _has(a[3]),
                                                      _has(a[4]), int(a[7])))],
    'pidm_groupnorm_silu_bwd': lambda a: [('gn_bwd', (int(a[12]), int(a[13]), int(a[14]), int(a[15]), _has(a[5]),
                                                      _has(a[9]), _has(a[10])))],
    'pidm_layernorm_c_fwd': lambda a: [('ln_fwd', (int(a[3]), int(a[4])))],
    'pidm_layernorm_c_bwd': lambda a: [('ln_bwd', (int(a[6]), int(a[7]), _has(a[5])))],
    'pidm_colsum': lambda a: [('colsum', (int(a[2]), int(a[3])))],
    # test_gpu_attention_census.py
    'pidm_linattn_fwd': lambda a: [('la_fwd', (int(a[6]), int(a[7]), int(a[8]), _dt(a[9])))],
    'pidm_linattn_bwd': lambda a: [('la_bwd', (int(a[7]), int(a[8]), int(a[9]), _dt(a[10])))],
    'pidm_attn_fwd': lambda a: [('attn_fwd', (int(a[2]), int(a[3]), int(a[4]), _dt(a[5])))],
    'pidm_attn_bwd': lambda a: [('attn_bwd', (int(a[3]), int(a[4]), int(a[5]), _dt(a[6])))],
    'pidm_head_fwd': lambda a: [('head_fwd', (int(a[4]), int(a[5]), int(a[6]), int(a[7]), int(a[8]), _dt(a[9])))],
    'pidm_head_bwd': lambda a: [('head_bwd', (int(a[7]), int(a[8]), int(a[9]), int(a[10]), int(a[11]), _dt(a[12])))],
    # test_gpu_physics_census.py
    'pidm_darcy_residual_fwd': _darcy_key('darcy_fwd', 3),
    'pidm_darcy_residual_bwd': _darcy_key('darcy_bwd', 4),
    'pidm_darcy_pidm_loss': lambda a: [('darcy_loss', (
        int(a[12]), int(a[13]), float(a[14]), int(a[15]), int(a[16]),
        int(a[1] is a[0] or a[1].data_ptr() == a[0].data_ptr()), _has(a[10]), _has(a[11])))],
    'pidm_mechanics_residual_fwd': lambda a: [('mech_fwd', (int(a[6]), int(a[7]), _has(a[5])))],
    'pidm_mechanics_residual_bwd': lambda a: [('mech_bwd', (int(a[9]), int(a[10]), _has(a[4]), _has(a[5])))],
    'pidm_mech_pidm_loss': lambda a: [('mech_loss', (int(a[18]), int(a[19])))],
    'pidm_bilinear_resize_fwd': lambda a: [('resize_fwd', (int(a[2]), int(a[3]), int(a[4])))],
    'pidm_bilinear_resize_bwd': lambda a: [('resize_bwd', (int(a[2]), int(a[3]), int(a[4])))],
    # test_gpu_glue_census.py
    'pidm_time_embed_fwd': lambda a: [('time_fwd', (int(a[9]), int(a[10]), int(a[11])))],
    'pidm_time_embed_bwd': lambda a: [('time_bwd', (int(a[10]), int(a[11]), int(a[12]), int(a[13])))],
    'pidm_block_mlps_fwd': lambda a: [('mlp_fwd', (int(a[4]), int(a[5]), int(a[2]), _mlp_rows(a)))],
    'pidm_block_mlps_bwd': lambda a: [('mlp_bwd', (int(a[5]), int(a[6]), int(a[2]), _mlp_rows(a), int(a[7])))],
    'pidm_sumsq': lambda a: [('sumsq', (int(a[1]),))],
    'pidm_adam_ema_step': lambda a: [('adam', (int(a[5]), _has(a[11]), float(a[13]), float(a[14]), int(a[16]),
                                               int(a[17])))],
    'pidm_pack_weights': _pack_keys,
    'pidm_pack_weights_pairs': _pair_keys,
    'pidm_qsample': lambda a: [('qsample', (int(a[6]), int(a[7])))],
    'pidm_axpby_per_sample': lambda a: [('axpby', (int(a[7]), int(a[8])))],
    'pidm_scale': lambda a: [('scale', (int(a[3]),))],
    'pidm_concat_channels': lambda a: [('concat', (int(a[3]), int(a[4]), int(a[5]), int(a[6])))],
    'pidm_split_channels': lambda a: [('split', (int(a[3]), int(a[4]), int(a[5]), int(a[6])))],
    'pidm_nchw_to_nhwc': lambda a: [('nchw', tuple(int(v) for v in a[2:7]))],
    # test_gpu_simt_census.py (the dtype is left out: every row is replayed in both)
    'pidm_conv2d_simt': lambda a: [('simt', tuple(int(v) for v in a[5:17]) + (_has(a[2]), _has(a[3])))],
    'pidm_conv2d_wgrad_simt': lambda a: [('simt_wgrad', tuple(int(v) for v in a[4:19]) + (_has(a[3]),))],
    # test_gpu_sampling_census.py
    'pidm_ddim_coefs': lambda a: [('ddim', (int(a[9]),))],
    'pidm_posterior_step': lambda a: [('posterior', (int(a[7]),))],
    'pidm_darcy_cocogen': lambda a: [('cocogen', (int(a[6]), int(a[7]), float(a[8]), int(a[9]), int(a[10]), int(a[5]),
                                                  int(a[4]), _has(a[3])))],
    'pidm_toy_pidm_loss': lambda a: [('toy_loss', (int(a[17]), int(a[18]), _has(a[3]), _has(a[4]), _has(a[6])))],
    # test_gpu_mech_eval_census.py
    'pidm_mech_sample_input': lambda a: [('mech_input', (int(a[3]), int(a[4]), int(a[5])))],
    'pidm_mech_posterior_step': lambda a: [('mech_post', (int(a[8]), int(a[9])))],
    'pidm_mech_fem_pcg': lambda a: [('pcg', (int(a[8]), int(a[9]), float(a[6]), int(a[7])))],
    'pidm_mech_floating_material': lambda a: [('fm', (int(a[2]), int(a[3])))],
}

# the families of KEYS by the census file that holds their tables, in the order of its tables
FAMILIES = {
    'test_gpu_launch_census.py': ('conv', 'wgrad', 'laf'),
    'test_gpu_norm_census.py': ('gn_fwd', 'gn_bwd', 'ln_fwd', 'ln_bwd', 'colsum'),
    'test_gpu_attention_census.py': ('la_fwd', 'la_bwd', 'attn_fwd', 'attn_bwd', 'head_fwd', 'head_bwd'),
    'test_gpu_physics_census.py': ('darcy_fwd', 'darcy_bwd', 'darcy_loss', 'mech_fwd', 'mech_bwd', 'mech_loss',
                                   'resize_fwd', 'resize_bwd'),
    'test_gpu_glue_census.py': ('time_fwd', 'time_bwd', 'mlp_fwd', 'mlp_bwd', 'sumsq', 'adam', 'pack', 'pair',
                                'pair_launch', 'qsample', 'axpby', 'scale', 'concat', 'split', 'nchw'),
    'test_gpu_simt_census.py': ('simt', 'simt_wgrad'),
    'test_gpu_sampling_census.py': ('ddim', 'posterior', 'cocogen', 'toy_loss'),
    'test_gpu_mech_eval_census.py': ('mech_input', 'mech_post', 'pcg', 'fm'),
}
# the recording each census file's tables are checked against, where it is not census()
RECORDING = {'test_gpu_simt_census.py': 'census_exact', 'test_gpu_sampling_census.py': 'census_sampling',
             'test_gpu_mech_eval_census.py': 'census_sampling'}

# Entry points the benchmarked steps call that launch nothing: host-side capability and size queries.
LAUNCHES_NOTHING = [
    'pidm_conv2d_tc_general_supported',
    'pidm_conv2d_wgrad_tc_supported',
    'pidm_linattn_block_supported',
    'pidm_linattn_block_workspace_floats',
    'pidm_linattn_workspace_floats',
    'pidm_mlp_entry_size',
    'pidm_pack_entry_size',
    'pidm_pack_pair_entry_size',
]

# Entry points of the exact mode that no census family keys, with the per-element or bitwise test that checks them
CHECKED_ELSEWHERE = {
    'pidm_wrap_pad_nhwc': 'test_gpu_circular.py::test_wrap_pad_is_bitwise_circular_pad',
    'pidm_cond_embed_fwd': 'test_gpu_guidance.py::test_cond_embed_per_element',
    'pidm_cond_embed_wgrad': 'test_gpu_guidance.py::test_cond_embed_wgrad_per_element',
    'pidm_darcy_abs_residual_grad': 'test_gpu_guidance.py::test_abs_residual_grad_per_element',
}


def assert_checked_or_listed(names, what):
    """every entry point in `names` is keyed, launches nothing or is CHECKED_ELSEWHERE by a test that exists"""
    import re
    unchecked = sorted(set(names) - set(KEYS) - set(LAUNCHES_NOTHING) - set(CHECKED_ELSEWHERE))
    assert not unchecked, (f'entry points of {what} that no test checks per element: add a census family, or name the '
                           'test that checks them in census.CHECKED_ELSEWHERE:\n' + '\n'.join(unchecked))
    here = os.path.dirname(os.path.abspath(__file__))
    for name, test in CHECKED_ELSEWHERE.items():
        file, fn = test.split('::')
        with open(os.path.join(here, file)) as f:
            assert re.search(rf'^def {fn}\(', f.read(), re.M), f'{name}: {test} does not exist'


# ----------------------------------------------------------------------------------------------------------------------
# recorder and workloads
# ----------------------------------------------------------------------------------------------------------------------
def _record(fn):
    """(set of (family, key), set of entry points) of the libpidm calls fn makes.  `call` is swapped in _lib and in
    every package module that imported it (ops, engine, residuals_mechanics_K, ...), and put back in any module that
    imported the recorder meanwhile."""
    from physicsinformeddiffusionmodels_b200 import _lib
    seen, names = set(), set()
    orig = _lib.call

    def rec(name, *a):
        names.add(name)
        if name in KEYS:
            seen.update(KEYS[name](a))
        return orig(name, *a)

    def package_modules(binding):
        return [m for n, m in list(sys.modules.items())
                if n.startswith('physicsinformeddiffusionmodels_b200') and getattr(m, 'call', None) is binding]
    for m in package_modules(orig):
        m.call = rec
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        for m in package_modules(rec):
            m.call = orig
    return seen, names


def _darcy_model(dev):
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    torch.manual_seed(0)
    return Unet3D(dim=32, channels=2).to(dev)


def _darcy_sample_engine(model, diff, B, t=None, **options):
    """an eager Darcy SampleEngine of batch B, as bench.py's sampling_bench builds it, on normal x at t [B] (default
    n_steps - 1) with the packed weights fresh; `options` go to ResidualsDarcy, or to SampleEngine for the CoCoGen
    ones"""
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    engine_options = {k: options.pop(k) for k in ('N_correction', 'M_correction', 'correction_mode') if k in options}
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                         device=DEV, **{'bcs': 'none', 'domain_length': 1., **options})
    se = SampleEngine(model, diff, res, batch=B, use_graph=False, **engine_options)
    packer = getattr(model, '_packer', None)
    if packer is not None:
        packer.refresh_if_stale(ops.act_dtype())
    se.x.normal_()
    se.t.copy_(torch.full((B,), diff.n_steps - 1) if t is None else torch.as_tensor(t))
    return se


def _ddim0_step(model, diff):
    """bench.py's sample-mode step: x0 by the DDIM walk with ddim_steps = 0, batch 16"""
    return {'darcy_sample_ddim0_b16': _record(_darcy_sample_engine(model, diff, 16, use_ddim_x0=True,
                                                                   ddim_steps=0)._step_body)}


def run_census(precision='bf16'):
    """{workload: _record(one eager step of it)} for every workload bench.py times, in ops precision `precision`"""
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    dev = torch.device(DEV)
    ops.set_precision(precision)
    ops.set_tensor_core_conv(True)
    out = {}
    model = _darcy_model(dev)
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True, device=dev,
                         bcs='none', domain_length=1.)
    eng = TrainEngine(model, DenoisingDiffusion(100, dev), res, lr=1e-4, max_norm=1.0, ema_mu=0.99, c_data=1.0,
                      c_residual=1e-3, use_graph=False)
    x0 = torch.randn(32, 2, 64, 64, generator=torch.Generator().manual_seed(1)).to(dev)
    out['darcy_train_b32'] = _record(lambda: eng.step(x0))
    del eng
    model.eval()
    diff = DenoisingDiffusion(250, dev)
    for B in (16, 64, 256):
        out[f'darcy_sample_b{B}'] = _record(_darcy_sample_engine(model, diff, B)._step_body)
    out.update(_ddim0_step(model, diff))
    del model
    torch.manual_seed(0)
    mech = Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True).to(dev)
    res = ResidualsMechanics(model=mech, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=dev)
    eng = TrainEngine(mech, DenoisingDiffusion(100, dev), res, lr=1e-4, max_norm=1.0, ema_mu=0.99, c_data=1.0,
                      c_residual=1e-2, c_ineq=0., lambda_opt=1e-3, use_graph=False)
    g = torch.Generator().manual_seed(5)
    B = 32
    cond = torch.rand(B, 3, 65, 65, generator=g)
    x0 = torch.cat((0.2 * torch.randn(B, 2, 65, 65, generator=g), torch.rand(B, 1, 65, 65, generator=g).clamp(1e-3, 1.)), 1)
    bcs = torch.zeros(B, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    bcs[:, 3, 32, 64] = -1.
    inp = torch.cat((cond, x0, bcs), dim=1).to(dev)
    out['mech_train_b32'] = _record(lambda: eng.step(inp))
    del eng, mech
    torch.cuda.empty_cache()
    return out


def _train_step(model, diff, res, B, seed):
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    eng = TrainEngine(model, diff, res, lr=1e-4, max_norm=1.0, ema_mu=0.99, c_data=1.0, c_residual=1e-3,
                      use_graph=False)
    x0 = torch.randn(B, 2, 64, 64, generator=torch.Generator().manual_seed(seed)).to(DEV)
    return _record(lambda: eng.step(x0))


def run_census_exact():
    """{workload: _record(one eager step of it)} in the fp32 exact mode: the workloads of run_census(), the Darcy
    training step of the guidance study and of the circular study with residual-gradient guidance (the halo'd
    geometries, and emb_conv[2], which stays zero-padded inside a circular model), and forward + backward of a scalar
    loss through the circular mechanics U-Net.  Leaves the package in bf16."""
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    from study import build_darcy
    try:
        out = run_census('fp32')
        out['guidance_train_b32'] = _train_step(*build_darcy('guidance'), 32, 2)
        out['circular_train_b32'] = _train_step(*build_darcy('circular', residual_grad_guidance=True), 32, 3)
        torch.manual_seed(0)
        mech = Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True, padding_mode='circular').to(DEV)
        g = torch.Generator().manual_seed(4)
        x = torch.randn(32, 10, 64, 64, generator=g).to(DEV)
        t = torch.randint(0, 100, (32,), generator=g).to(DEV)
        out['circular_mech_b32'] = _record(lambda: mech(x, t).square().mean().backward())
        del mech
        torch.cuda.empty_cache()
    finally:
        ops.set_precision('bf16')
    return out


def _toy_residual(x):
    return torch.sum(x ** 2, dim=1) - 1.0


def _toy_ineq(x):
    density = torch.sum(torch.abs(x), dim=1)
    return torch.relu(density - 1.0), density


def _toy_opt(x):
    return x[:, 0]


def run_census_sampling():
    """{workload: _record(one eager step of it)} of the sampling side in bf16: bench.py's sample-mode step, a Darcy
    SampleEngine step with ddim_steps = 3 at per-sample t, CoCoGen SampleEngine steps in both correction modes for both
    boundary conditions at per-sample t that leave some samples inactive, the M_correction launch after the loop, one
    drop-in DenoisingDiffusion.p_sample step, conditional mechanics SampleEngine steps in mean and sample mode and the
    evaluation of their last x0 prediction (topopt_eval, with a solution), the toy training loss in x0 and eps mode, and
    one toy p_sample step at an odd batch (whose posterior step takes the scalar path)"""
    import mech_sample_inputs as MI
    from physicsinformeddiffusionmodels_b200 import denoising_toy_utils as T
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    dev = torch.device(DEV)
    ops.set_precision('bf16')
    ops.set_tensor_core_conv(True)
    out = {}
    model = _darcy_model(dev)
    model.eval()
    diff = DenoisingDiffusion(250, dev)
    out.update(_ddim0_step(model, diff))
    out['darcy_sample_ddim3_b4'] = _record(_darcy_sample_engine(model, diff, 4, [249, 100, 3, 0], use_ddim_x0=True,
                                                                ddim_steps=3)._step_body)
    diff6 = DenoisingDiffusion(6, dev)
    for bcs in ('none', 'periodic'):
        for mode in ('xt', 'x0'):
            se = _darcy_sample_engine(model, diff6, 4, [3, 1, 0, 2], bcs=bcs, N_correction=2, M_correction=3,
                                      correction_mode=mode)
            out[f'cocogen_{mode}_{bcs}_b4'] = _record(se._step_body)
        out[f'cocogen_M3_{bcs}_b4'] = _record(lambda: se.residuals.cocogen(se.x, se.residual, se.M_correction))
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True, device=dev)
    x = torch.randn(2, 2, 64, 64, device=dev)
    out['p_sample_b2'] = _record(lambda: diff6.p_sample(x, None, 5, residual_func=res, surpress_noise=True))
    del model, se
    torch.manual_seed(0)
    mech = Unet3D(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True).to(dev)
    mech.eval()
    cond, bcs, rho = MI.conditioning_batch()
    solution = torch.zeros(MI.B, 3, 65, 65)
    solution[:, 2, :-1, :-1] = rho
    ci = (cond.to(dev), bcs.to(dev), solution.to(dev))
    for mode in ('mean', 'sample'):
        res = ResidualsMechanics(model=mech, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=dev,
                                 topopt_eval=True, use_ddim_x0=mode == 'sample', ddim_steps=0)
        se = SampleEngine(mech, diff6, res, batch=MI.B, image_shape=(3, 65, 65), use_graph=False)
        n = se._mech_condition(ci)
        se.x.normal_()
        se.t.fill_(diff6.n_steps - 1)
        out[f'mech_sample_{mode}_b{MI.B}'] = _record(se._step_body)
    out[f'mech_aux_b{MI.B}'] = _record(lambda: se._mech_aux(ci, n))
    del mech, se
    torch.manual_seed(0)
    toy = T.ConditionalModel(2, 100).to(dev)
    dd = T.create_diff_dict(100, dev)
    x0 = torch.randn(128, 2, device=dev)
    for mode, extra in (('x0', dict(ineq_func=_toy_ineq, opt_func=_toy_opt)), ('eps', {})):
        out[f'toy_loss_{mode}_b128'] = _record(lambda: T.model_estimation_loss(
            toy, x0, 100, dd, model_pred_mode=mode, residual_func=_toy_residual, c_data=1.0, c_residual=0.005,
            c_ineq=0.3, lambda_opt=0.01, **extra)[0].backward())
    out['toy_p_sample_b63'] = _record(lambda: T.p_sample(toy, torch.randn(63, 2, device=dev), 5, dd, model_pred_mode='x0'))
    torch.cuda.empty_cache()
    return out


def _summary(raw):
    return {wl: keys for wl, (keys, _) in raw.items()}, set().union(*(names for _, names in raw.values()))


@functools.cache
def census():
    """({workload: set of (family, key)}, set of every entry point called), recorded once per process"""
    return _summary(run_census())


@functools.cache
def census_exact():
    """census() of the fp32 exact mode (run_census_exact), recorded once per process"""
    return _summary(run_census_exact())


@functools.cache
def census_sampling():
    """census() of the sampling-side workloads (run_census_sampling), recorded once per process"""
    return _summary(run_census_sampling())


def _recording(file):
    return globals()[RECORDING.get(file, 'census')]


def _file_of(tables):
    """the census file whose families are the keys of `tables`"""
    files = [f for f, fams in FAMILIES.items() if set(tables) <= set(fams)]
    assert len(files) == 1, f'tables of no single census file: {sorted(tables)}'
    return files[0]


# ----------------------------------------------------------------------------------------------------------------------
# the two-way check of a census file's tables ({family: rows})
# ----------------------------------------------------------------------------------------------------------------------
def assert_census_in_tables(tables):
    keys, _ = _recording(_file_of(tables))()
    missing = [f'{fam} {k!r}  # {wl}' for wl, ks in keys.items()
               for fam, k in sorted(fk for fk in ks if fk[0] in tables) if k not in tables[fam]]
    assert not missing, ('launches of the benchmarked steps that the tables do not replay (add them; '
                         '`python tests/census.py --print-table`):\n' + '\n'.join(missing))


def assert_tables_in_census(tables):
    keys, _ = _recording(_file_of(tables))()
    produced = {fk for ks in keys.values() for fk in ks}
    stale = [f'{fam} {k!r}' for fam, table in tables.items() for k in table if (fam, k) not in produced]
    assert not stale, ('table rows that no benchmarked step launches (drop them, or move a row kept for plan coverage '
                       'to the synthetic rows; `python tests/census.py --print-table`):\n' + '\n'.join(stale))


def print_tables():
    for file, families in FAMILIES.items():
        keys, _ = _recording(file)()
        rows = {f: {} for f in families}
        for wl, ks in keys.items():
            for fam, k in ks:
                if fam in rows:
                    rows[fam].setdefault(k, []).append(wl)
        print(f'# tests/{file}')
        for fam, table in rows.items():
            print(f'{fam.upper()}_TABLE = [')
            for k in sorted(table):
                print(f'    {k!r},  # {" ".join(sorted(table[k]))}')
            print(']')
        for wl, ks in keys.items():
            print(f'# {wl}: ' + ', '.join(f'{f} {sum(1 for ff, _ in ks if ff == f)}' for f in families))
        print('# distinct: ' + ', '.join(f'{f} {len(v)}' for f, v in rows.items()))
    _, names = census()
    print('# tests/census.py')
    print('LAUNCHES_NOTHING = [')
    for n in sorted(names - set(KEYS)):
        print(f'    {n!r},')
    print(']')


if __name__ == '__main__':
    if '--print-table' in sys.argv:
        sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))     # the repository root
        print_tables()
