"""Host checks (no GPU) of the topology-optimisation sampling oracle (oracle/pidm_oracle.py) against the unmodified
reference: its ancestral loop with a conditioning input reproduces tests/golden/mechanics_sample_loop.pt
(oracle/make_golden.py mech_sample; inputs and draws rebuilt by tests/mech_sample_inputs.py) in both x0 modes, which
pins the draw order, and its fp64 sparse solve reproduces the
displacements of tests/golden/mechanics_eval.pt (the reference's dense fp64 solve)."""
import pytest
import torch

import mech_sample_inputs as MI
from checks import rel
from oracle import pidm_oracle as O


@pytest.mark.parametrize('mode', ['mean', 'sample'])
def test_oracle_sampler_reproduces_reference(golden, mode):
    gd = golden('mechanics_sample_loop.pt')
    cfg = O.unet_config(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in O.make_test_state_dict(cfg, seed=3).items()}
    n = int(gd['n_steps'])
    cond, bcs, _ = MI.inputs(gd)
    x_T, zs, _ = MI.replay_draws(gd, mode)
    out = O.mechanics_p_sample_loop(sd, cfg, x_T.double(), zs.double(), cond.double(), bcs.double(), O.diffusion_tables(n),
                                    n, use_ddim_x0=mode == 'sample')
    gs = lambda k: O.golden_sample(out[k], MI.SAMPLE)
    for k in ('x_first', 'x_final', 'x0_pred_last'):
        assert rel(gs(k), gd[f'{mode}_{k}']) < 1e-5, (k, rel(gs(k), gd[f'{mode}_{k}']))
    assert (out['x0_pred_last'][:, 2] - gd[f'{mode}_rho_last'].double()).abs().max() < 1e-5
    # the reference assembles a dense fp32 K (summation order differs): the residual is a difference of O(1) terms
    assert rel(gs('residual'), gd[f'{mode}_residual']) < 1e-4, rel(gs('residual'), gd[f'{mode}_residual'])
    assert rel(out['compliance'], gd[f'{mode}_compliance']) < 1e-4
    assert (out['inequality'] - gd[f'{mode}_inequality'].double()).abs().max() < 1e-6


def test_sparse_solve_reproduces_reference_solution(golden):
    ev = golden('mechanics_eval.pt')
    KE = golden('mechanics_residual.pt')['KE']                  # the reference's element matrix (fp32 values)
    rho = ev['solution'][:, 2, :-1, :-1]
    u = O.fem_solve(rho, ev['bcs'], KE)
    assert rel(u, ev['solution'][:, :2]) < 1e-6, rel(u, ev['solution'][:, :2])
    _, bcs, sol = MI.inputs(golden('mechanics_sample_loop.pt'))
    u = O.fem_solve(sol[:, 2, :-1, :-1], bcs, KE)
    assert rel(u, sol[:, :2]) < 1e-6, rel(u, sol[:, :2])


def test_sparse_system_is_the_reference_modification():
    """identity rows on the Dirichlet dofs, the columns left as they are, f zeroed there"""
    g = torch.Generator().manual_seed(0)
    rho = torch.rand(1, 4, 4, generator=g).double()
    bcs = torch.zeros(1, 4, 5, 5, dtype=torch.float64)
    bcs[0, 0, :, 0] = 1.
    bcs[0, 1, 2, 0] = 1.
    bcs[0, 2:] = torch.randn(2, 5, 5, generator=g).double()
    K, f = O.reduced_system(rho[0], bcs[0])
    Kd = K.toarray()
    fixed = torch.stack((bcs[0, 0].reshape(-1), bcs[0, 1].reshape(-1)), dim=1).reshape(-1).numpy() != 0
    assert (Kd[fixed][:, fixed] == torch.eye(int(fixed.sum())).numpy()).all()
    assert (Kd[fixed][:, ~fixed] == 0).all() and (Kd[~fixed][:, fixed] != 0).any()
    assert (f[fixed] == 0).all()
    # the free block is the matrix-free operator of oracle/pidm_oracle.py
    v = torch.randn(1, 2, 5, 5, generator=g).double()
    u_flat = v.permute(0, 2, 3, 1).reshape(-1).numpy()
    r_free = (Kd @ u_flat)[~fixed]
    dofs = O.mechanics_mesh(4)
    KE = O.q4_plane_stress_stiffness()
    Ku = torch.zeros(50, dtype=torch.float64).index_add_(0, dofs.reshape(-1), (torch.einsum(
        'ij,ej->ei', KE, torch.from_numpy(u_flat)[dofs]) * rho.reshape(-1, 1)).reshape(-1))
    assert torch.allclose(torch.from_numpy(r_free), Ku[torch.from_numpy(~fixed)], atol=1e-12)
