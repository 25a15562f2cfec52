"""Golden vectors for conditional sampling of the topology-optimisation model.  TEST INFRASTRUCTURE ONLY; runs on CPU.

Runs the UNMODIFIED reference modules (checkout in PIDM_REFERENCE, imported through oracle/ref_shims/ exactly as
oracle/make_golden.py does): `DenoisingDiffusion.p_sample_loop` with a `conditioning_input` (reference
denoising_utils.py:388-545, sample.py:244-262) at B = 2 over 6 diffusion steps, with `eval_residuals`,
`return_optimizer`, `return_inequality` and `topopt_eval=True` (dense LU of the binarised designs at t = 0), for both
x0 estimates ('mean': one network call; 'sample': `use_ddim_x0=True, ddim_steps=0`).  The data samples are consistent
(their displacements solve K(rho_simp) u = f, the construction of oracle/make_golden.py for mechanics_eval.pt), so the
reference's data-residual check passes.  Writes the NEW fixture tests/golden/mechanics_sample_loop.pt; every existing
fixture is left as it is.  The inputs and the draws are rebuilt by tests/mech_sample_inputs.py and only checksummed here;
large outputs are stored as oracle.pidm_oracle.golden_sample(., 4096).  Keys:

    seed, n_steps, input_checksum, solution      the loop's seed, the inputs' checksums, the consistent data samples
per mode (prefix 'mean_' / 'sample_'):
    noise_checksum                               per-draw sums of x_T, the posterior z and (in 'sample' mode) the DDIM
                                                 walk's draws, in the reference's order
    x_first, x_final, x0_pred_last, residual     golden samples of the sample after the first / last step, the last x0
                                                 estimate (the last network output) and the residual of the last step
    rho_last                                     the density channel of that x0 estimate, whole (binarisation checks)
    compliance, inequality, rel_CE_error, vf_error, fm_error    the aux outputs of the last step

    PIDM_REFERENCE=<checkout of the original project> python scripts/make_golden_mech_sample.py
"""
import importlib.util
import os
import tempfile

import torch
from torch.nn.functional import pad as F_pad

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_spec = importlib.util.spec_from_file_location('make_golden', os.path.join(ROOT, 'oracle', 'make_golden.py'))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
O = MG.O
_spec = importlib.util.spec_from_file_location('mech_sample_inputs', os.path.join(ROOT, 'tests', 'mech_sample_inputs.py'))
MI = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MI)

B = MI.B
N_STEPS = 6
SEED = 2024


def consistent_solution(st, rho_simp, bcs):
    """[1,3,65,65] = (u_x, u_y, rho_simp padded) with u solving the reference's modified dense system (fp64), as
    oracle/make_golden.py builds the mechanics_eval.pt sample."""
    Kd = torch.zeros(st.neq, st.neq, dtype=torch.float64)
    kl = st.tot_local_stiffness.double() * rho_simp.reshape(-1).double()[:, None, None]
    idx = st.glob_assembler_idcs
    Kd.index_put_((idx[:, :, 0].reshape(-1), idx[:, :, 1].reshape(-1)),
                  kl[:, st.indices_ext[:, 0], st.indices_ext[:, 1]].reshape(-1), accumulate=True)
    bcx = st.image_to_stiffness_coord(bcs[:, 0], 0) + st.image_to_stiffness_coord(bcs[:, 1], 1)
    fg = (st.image_to_stiffness_coord(bcs[:, 2], 0) + st.image_to_stiffness_coord(bcs[:, 3], 1))[0].double()
    mk = bcx[0] != 0
    Kd[mk] = 0
    Kd[mk, mk] = 1
    fg[mk] = 0
    u = torch.linalg.solve(Kd, fg).float()[None]
    sol = torch.stack((st.stiffness_to_image_coord(u, 0), st.stiffness_to_image_coord(u, 1)), dim=1)
    return torch.cat((sol, F_pad(rho_simp, (0, 1, 0, 1)).unsqueeze(1)), dim=1)


def main():
    torch.set_num_threads(8)
    import src.unet_model as _um
    assert os.path.abspath(_um.__file__).startswith(os.path.abspath(MG.REF)), _um.__file__
    from src.denoising_utils import DenoisingDiffusion
    from src.residuals_mechanics_K import ResidualsMechanics
    from src.unet_model import Unet3D

    cfg = O.unet_config(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
    model = Unet3D(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
    model.load_state_dict(O.make_test_state_dict(cfg, seed=3), strict=True)
    model.eval()
    last = {}
    model.register_forward_hook(lambda m, i, o: last.__setitem__('y', o.detach().clone()))
    cond, bcs, rho = MI.conditioning_batch()
    out = {'n_steps': torch.tensor(N_STEPS), 'seed': torch.tensor(SEED),
           'input_checksum': torch.stack([cond.double().sum(), bcs.double().sum(), rho.double().sum()])}
    gs = lambda t: O.golden_sample(t, MI.SAMPLE)
    with tempfile.TemporaryDirectory() as td:
        MG.write_mesh(td)
        for mode in ('mean', 'sample'):
            res = ResidualsMechanics(model=model, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder=td + '/',
                                     device='cpu', topopt_eval=True, use_ddim_x0=mode == 'sample', ddim_steps=0)
            if mode == 'mean':
                sol = torch.cat([consistent_solution(res.stiffs, rho[b][None], bcs[b:b + 1]) for b in range(B)], dim=0)
                out['solution'] = sol
            diff = DenoisingDiffusion(N_STEPS, 'cpu')
            torch.manual_seed(SEED)
            with torch.no_grad():
                (x_seq, _), aux = diff.p_sample_loop((cond, bcs, sol), (B, 3, 65, 65), save_output=True,
                                                     surpress_noise=True, residual_func=res, eval_residuals=True,
                                                     return_optimizer=True, return_inequality=True)
            x_T, zs, ddim = MI.draws(SEED, N_STEPS, mode)     # replay the draws in the reference's order
            assert torch.equal(x_T, x_seq[0])
            out.update({f'{mode}_{k}': v for k, v in dict(
                noise_checksum=MI.checksums(x_T, zs, ddim), x_first=gs(x_seq[1]), x_final=gs(x_seq[-1]),
                x0_pred_last=gs(last['y']), rho_last=last['y'][:, 2].clone(), residual=gs(aux['residual'].detach()),
                compliance=aux['optimized_quant'].detach(), inequality=aux['inequality_quant'].detach(),
                rel_CE_error=aux['rel_CE_error_full_batch'].detach(), vf_error=aux['vf_error_full_batch'].detach(),
                fm_error=aux['fm_error_full_batch']).items()})
            print(mode, 'rel_CE_error', aux['rel_CE_error_full_batch'].tolist(), 'fm', aux['fm_error_full_batch'].tolist(),
                  '|rho - 0.5| min', (last['y'][:, 2] - 0.5).abs().min().item())
    MG.save('mechanics_sample_loop.pt', out)


if __name__ == '__main__':
    main()
