"""CPU-side checks (no GPU needed): the C-ABI library loads and exports every symbol include/pidm.h declares,
the host-side mirror of the reference interface (module tree / state_dict / schedule tables) matches the
reference, and the data-parallel host logic (sharding + flat-gradient all-reduce, gloo, world_size 2)."""
import os
import re
import subprocess
import sys

import pytest
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_loads_and_exports_header_symbols():
    import __graft_entry__
    __graft_entry__.build()
    from physicsinformeddiffusionmodels_b200 import _lib
    hdr = open(os.path.join(ROOT, 'include', 'pidm.h')).read()
    declared = set(re.findall(r'\b(pidm_[a-z0-9_]+)\s*\(', hdr))
    assert len(declared) >= 40
    for name in declared:
        assert hasattr(_lib._lib, name), f'{name} is declared in pidm.h but not exported by libpidm.so'
    assert declared == set(_lib.exported_symbols()), declared ^ set(_lib.exported_symbols())
    assert _lib.call('pidm_version') == 100
    assert _lib.call('pidm_pack_entry_size') == 56 and _lib.call('pidm_mlp_entry_size') == 56


# Entry points of include/pidm.h that no census recording calls: host queries that launch nothing, and kernels with a
# named per-element or bitwise test of their own
HOST_QUERIES = ['pidm_version', 'pidm_last_error', 'pidm_conv2d_tc_plan', 'pidm_conv2d_wgrad_tc_plan',
                'pidm_groupnorm_plan', 'pidm_linattn_block_plan', 'pidm_linattn_plan', 'pidm_darcy_gen_workspace_bytes']
TESTED_OUTSIDE_THE_RECORDINGS = {
    'pidm_darcy_gen_kle': 'test_gpu_darcy_gen_replay.py::test_kle_known_answer',  # the Darcy training-data generator
    'pidm_darcy_gen_solve': 'test_gpu_darcy_gen_replay.py::test_stages_within_bounds',
    'pidm_swap_f32': 'test_gpu_ema_eval.py::test_swap_is_an_exact_exchange',  # the EMA weight swap
    'pidm_fd_stencil': 'test_gpu_physics_census.py::test_darcy_fd_stencil_replay',
    'pidm_darcy_jacobian_max': 'test_gpu_physics_census.py::test_darcy_jacobian_max_replay',
}


def test_every_header_entry_point_is_accounted_for():
    """every pidm_* of include/pidm.h is keyed by a census family, launches nothing, is checked elsewhere, is a host
    query or has a named test; an entry point nothing calls is removed, not listed"""
    import census
    hdr = open(os.path.join(ROOT, 'include', 'pidm.h')).read()
    declared = set(re.findall(r'\b(pidm_[a-z0-9_]+)\s*\(', hdr))
    lists = {'census.KEYS': set(census.KEYS), 'census.LAUNCHES_NOTHING': set(census.LAUNCHES_NOTHING),
             'census.CHECKED_ELSEWHERE': set(census.CHECKED_ELSEWHERE), 'HOST_QUERIES': set(HOST_QUERIES),
             'TESTED_OUTSIDE_THE_RECORDINGS': set(TESTED_OUTSIDE_THE_RECORDINGS)}
    covered = set().union(*lists.values())
    assert not declared - covered, f'entry points of pidm.h that nothing accounts for: {sorted(declared - covered)}'
    assert not covered - declared, f'listed entry points that pidm.h does not declare: {sorted(covered - declared)}'
    for a in ('HOST_QUERIES', 'TESTED_OUTSIDE_THE_RECORDINGS'):
        for b, names in lists.items():
            assert a == b or not lists[a] & names, f'{sorted(lists[a] & names)} listed in both {a} and {b}'
    for name, test in TESTED_OUTSIDE_THE_RECORDINGS.items():
        file, fn = test.split('::')
        with open(os.path.join(ROOT, 'tests', file)) as f:
            assert re.search(rf'^def {fn}\(', f.read(), re.M), f'{name}: {test} does not exist'


@pytest.mark.parametrize('name,args,what', [
    ('pidm_mech_fem_pcg', dict(nel=67), 'nel'), ('pidm_mech_fem_pcg', dict(nel=1), 'nel'),
    ('pidm_mech_fem_pcg', dict(B=0), 'B='), ('pidm_mech_fem_pcg', dict(max_iter=-1), 'max_iter'),
    ('pidm_mech_fem_pcg', dict(tol=-1e-9), 'tol'),
    ('pidm_mech_floating_material', dict(nel=0), 'nel'), ('pidm_mech_floating_material', dict(nel=129), 'nel'),
    ('pidm_mech_floating_material', dict(B=0), 'B='),
    ('pidm_mech_posterior_step', dict(P=1), 'P='), ('pidm_mech_posterior_step', dict(B=0), 'B='),
    ('pidm_mech_sample_input', dict(P=1), 'P='), ('pidm_mech_sample_input', dict(B=0), 'B='),
], ids=lambda v: v if isinstance(v, str) else '-'.join(f'{k}{x}' for k, x in v.items()) if isinstance(v, dict) else '')
def test_mech_eval_sizes_are_refused_before_any_launch(name, args, what):
    """sizes the topology-optimisation kernels do not support fail the size check (error code 2), which runs before
    any CUDA call: null pointers and no device are enough"""
    from physicsinformeddiffusionmodels_b200._lib import call
    a = {**dict(B=2, nel=64, P=64, tol=1e-6, max_iter=10), **args}
    argv = {'pidm_mech_fem_pcg': (None,) * 6 + (a['tol'], a['max_iter'], a['B'], a['nel'], None),
            'pidm_mech_floating_material': (None, None, a['B'], a['nel'], None),
            'pidm_mech_posterior_step': (None,) * 8 + (a['B'], a['P'], None),
            'pidm_mech_sample_input': (None,) * 3 + (a['B'], 7, a['P'], None)}[name]
    with pytest.raises(RuntimeError, match=rf'\(code 2\): {name[5:]}: .*{what}'):
        call(name, *argv)


def test_no_oracle_import_on_product_path():
    """The product package must never reach into oracle/ (selftest.smoke is the one sanctioned checker)."""
    pkg = os.path.join(ROOT, 'physicsinformeddiffusionmodels_b200')
    for fn in os.listdir(pkg):
        if fn.endswith('.py') and fn != 'selftest.py':
            src = open(os.path.join(pkg, fn)).read()
            assert 'oracle' not in src, fn


def test_unet_state_dict_matches_reference_layout():
    from oracle import pidm_oracle as O
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    for kw, cfg in ((dict(dim=32, channels=2), O.unet_config(dim=32, channels=2)),
                    (dict(dim=16, channels=10, out_dim=3, sigmoid_last_channel=True),
                     O.unet_config(dim=16, channels=10, out_dim=3, sigmoid_last_channel=True))):
        m = Unet3D(**kw)
        sd = m.state_dict()
        shapes = O.unet_param_shapes(cfg)
        assert list(sd.keys()) == list(shapes.keys())
        for k, v in sd.items():
            assert tuple(v.shape) == tuple(shapes[k]), k
    m = Unet3D(dim=32, channels=2)
    assert sum(p.numel() for p in m.parameters() if p.requires_grad) == 10386482      # SURVEY.md section 2
    m.load_state_dict(O.make_test_state_dict(O.unet_config(), 0), strict=True)


def test_unet_default_init_is_bitwise_the_reference_init(golden):
    """Same seed -> same initial weights as the reference (holders are constructed in the reference's order)."""
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    gd = golden('unet_init_seed0.pt')
    torch.manual_seed(0)
    sd = Unet3D(dim=32, channels=2).state_dict()
    for k, v in sd.items():
        assert abs(v.double().sum().item() - gd[k][0].item()) < 1e-9 and \
            abs(v.double().abs().sum().item() - gd[k][1].item()) < 1e-9, k


@pytest.mark.parametrize('n', [100, 250])
def test_schedule_tables_match_reference(golden, n):
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    ref = golden(f'schedule_{n}.pt')
    d = DenoisingDiffusion(n, 'cpu')
    assert list(d.diff_dict.keys()) == list(ref.keys())
    for k in ref:
        assert torch.allclose(d.diff_dict[k], ref[k], rtol=1e-6, atol=1e-7), k


def test_cpu_tensors_are_rejected_not_silently_computed():
    from physicsinformeddiffusionmodels_b200 import ops
    with pytest.raises(RuntimeError):
        ops.darcy_residual(torch.zeros(1, 2, 64, 64), torch.zeros(4096))
    with pytest.raises(RuntimeError):
        ops.q_sample(torch.zeros(1, 2, 64, 64), torch.zeros(1, 2, 64, 64), torch.zeros(1, dtype=torch.long),
                     torch.zeros(100), torch.zeros(100))


def test_drop_in_module_names_resolve():
    import importlib
    for name, syms in (('src.unet_model', ['Unet3D']), ('src.residuals_darcy', ['ResidualsDarcy']),
                       ('src.residuals_mechanics_K', ['ResidualsMechanics']),
                       ('src.denoising_utils', ['DenoisingDiffusion', 'EMA', 'device', 'noop', 'exists', 'save_model',
                                                'load_model', 'fix_seeds', 'np', 'Path',
                                                'generalized_image_to_b_xy_c', 'generalized_b_xy_c_to_image']),
                       ('src.data_utils', ['Dataset', 'Dataset_Paths', 'cycle', 'pd', 'np', 'torch', 'Path'])):
        mod = importlib.import_module(name)
        for s in syms:
            assert hasattr(mod, s), (name, s)


def test_layout_helpers_roundtrip():
    from physicsinformeddiffusionmodels_b200.denoising_utils import b_xy_c_to_image, image_to_b_xy_c
    from physicsinformeddiffusionmodels_b200.grad_utils import generalized_b_xy_c_to_image, generalized_image_to_b_xy_c
    x = torch.arange(2 * 3 * 4 * 4, dtype=torch.float32).reshape(2, 3, 4, 4)
    assert torch.equal(b_xy_c_to_image(image_to_b_xy_c(x)), x)
    assert torch.equal(generalized_image_to_b_xy_c(x), image_to_b_xy_c(x))
    y = torch.arange(2 * 3 * 2 * 4 * 4, dtype=torch.float32).reshape(2, 3, 2, 4, 4)
    assert torch.equal(generalized_b_xy_c_to_image(generalized_image_to_b_xy_c(y)), y)
    assert generalized_image_to_b_xy_c(y).shape == (2, 16, 3, 2)


_DDP_SCRIPT = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from physicsinformeddiffusionmodels_b200.engine import shard_rows, allreduce_flat_grad
dist.init_process_group('gloo')
rank, world = dist.get_rank(), dist.get_world_size()
torch.manual_seed(0)
W = torch.randn(7, 5)
X, Y = torch.randn(8, 5), torch.randn(8, 7)
def grad(rows):
    w = W.clone().requires_grad_(True)
    ((X[rows] @ w.T - Y[rows]) ** 2).mean().backward()
    return w.grad.reshape(-1)
lo, hi = shard_rows(8, rank, world)
g = grad(slice(lo, hi)).clone()
allreduce_flat_grad(g, world)
g /= world
full = grad(slice(0, 8))
assert torch.allclose(g, full, atol=1e-6), (g - full).abs().max()
# only the live prefix of the flat gradient is exchanged: the tail (parameters the forward never uses) stays untouched
h = torch.full((10,), float(rank + 1))
allreduce_flat_grad(h, world, live=6)
assert torch.equal(h[:6], torch.full((6,), 3.0)) and torch.equal(h[6:], torch.full((4,), float(rank + 1)))
# global-batch draws (SURVEY 8e): with identical generator states the rank shards are the rows of the one-process draws
from physicsinformeddiffusionmodels_b200.denoising_utils import draw_t_and_noise
x_shard = torch.zeros(4, 2, 8, 8)
torch.manual_seed(123)
t_r, e_r = draw_t_and_noise(100, x_shard, (rank, world))
torch.manual_seed(123)
t_1, e_1 = draw_t_and_noise(100, torch.zeros(4 * world, 2, 8, 8), None)
assert torch.equal(t_r, t_1[4 * rank:4 * rank + 4]) and torch.equal(e_r, e_1[4 * rank:4 * rank + 4])
print('rank', rank, 'ok')
'''


def test_datasets_follow_the_reference_file_formats(tmp_path):
    """reference data_utils.py:31-119: one CSV per channel with one flattened sample per row -> [C, P, P] (row-major
    pixels); .npy samples stored channels-last, visited in NUMERIC file-name order, handed out channels-first."""
    from physicsinformeddiffusionmodels_b200.data_utils import Dataset, Dataset_Paths
    rng = np.random.default_rng(3)
    a, b = rng.standard_normal((5, 16)).astype(np.float32), rng.standard_normal((5, 16)).astype(np.float32)
    np.savetxt(tmp_path / 'p.csv', a, delimiter=',')
    np.savetxt(tmp_path / 'k.csv', b, delimiter=',')
    ds = Dataset((str(tmp_path / 'p.csv'), str(tmp_path / 'k.csv')))
    assert len(ds) == 5 and ds[3].shape == (2, 4, 4) and ds[3].dtype == torch.float32
    assert np.allclose(ds[3][0].numpy(), a[3].reshape(4, 4), atol=1e-6) and np.allclose(ds[3][1].numpy(), b[3].reshape(4, 4), atol=1e-6)
    assert Dataset((str(tmp_path / 'p.csv'), str(tmp_path / 'k.csv')), use_double=True)[0].dtype == torch.float64
    with pytest.raises(IndexError):
        ds[5]
    os.makedirs(tmp_path / 'npy' / 'sub')
    for i in (10, 2, 33):
        np.save(tmp_path / 'npy' / ('sub' if i == 2 else '') / f'{i}.npy', np.full((6, 6, 10), float(i)) + np.arange(10))
    dp = Dataset_Paths(str(tmp_path / 'npy'))
    assert len(dp) == 3 and [int(dp[i][0, 0, 0]) for i in range(3)] == [2, 10, 33]
    assert dp[1].shape == (10, 6, 6) and float(dp[1][7, 3, 3]) == 17.0


def test_floating_material_check_matches_cv2_semantics():
    """reference :376-380: exactly one 8-connected solid component <=> no floating material"""
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import check_floating_material
    img = np.full((8, 8), 1e-3)
    img[1:4, 1:4] = 1.0
    assert not check_floating_material(img)
    img[4, 4] = 1.0                                   # touches diagonally: still one piece (8-connectivity)
    assert not check_floating_material(img)
    img[6, 6] = 1.0                                   # detached island
    assert check_floating_material(img)
    assert check_floating_material(np.full((8, 8), 1e-3))     # no material at all


def test_flat_layout_puts_unused_parameters_last():
    """FlatParams: the 56 parameters forward never touches (the reference leaves their .grad at None) form the tail of
    the flat buffers, so the data-parallel exchange covers only [0, live_total)."""
    from physicsinformeddiffusionmodels_b200.engine import FlatParams
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    model = Unet3D(dim=32, channels=2)
    dead = set(model.unused_parameter_names())
    with open(os.path.join(ROOT, 'tests', 'golden', 'params_without_grad.txt')) as f:
        ref_dead = {k for k in f.read().split() if not k.endswith('rotary_emb.freqs')}
    assert dead == ref_dead
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    fp = FlatParams(model, with_optimizer_state=False)
    names = {id(p): n for n, p in model.named_parameters()}
    for p, o in zip(fp.params, fp.offsets):
        assert (o >= fp.live_total) == (names[id(p)] in dead), names[id(p)]
        assert torch.equal(p.detach(), before[names[id(p)]])          # re-homing keeps the values
    assert 0 < fp.total - fp.live_total < 1.6e6 and fp.live_total % 64 == 0


def test_data_parallel_gradient_is_full_batch_gradient_gloo(tmp_path):
    """world_size 2 on CPU (gloo): averaged shard gradients == full-batch gradient (the engine's exchange step)."""
    script = tmp_path / 'ddp.py'
    script.write_text(_DDP_SCRIPT)
    env = dict(os.environ, MASTER_ADDR='127.0.0.1', MASTER_PORT='29533')
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29533', str(script), ROOT],
                       capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count('ok') == 2
