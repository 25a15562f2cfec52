"""Golden vectors for CoCoGen residual corrections.  TEST INFRASTRUCTURE ONLY; runs on CPU, not on the GPU box.

Runs the UNMODIFIED reference modules (checkout in PIDM_REFERENCE, imported through oracle/ref_shims/ exactly as
oracle/make_golden.py does) and writes two NEW fixtures to tests/golden/.  Every existing fixture is left as it is:

    cocogen_steps.pt         five successive residual_correction calls (vmap(jacfwd) Jacobian) on the two fields of
                             cocogen.pt: the p plane after every call and the residual after the last
    sample_loop_cocogen.pt   the sample_loop_6 recipe (6 steps, B=1, seed-0 test weights, seed-77 draws) run with
                             N_correction=2, M_correction=3, 'xt' and with N_correction=2, M_correction=0, 'x0'

    PIDM_REFERENCE=<checkout of the original project> python scripts/make_golden_cocogen.py
"""
import importlib.util
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# make_golden sets up the import path (reference first, shims, repository root removed) and provides the helpers
_spec = importlib.util.spec_from_file_location('make_golden', os.path.join(ROOT, 'oracle', 'make_golden.py'))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
O = MG.O

N_CALLS = 5


def main():
    torch.set_num_threads(8)
    import src.unet_model as _ref_mod
    assert os.path.abspath(_ref_mod.__file__).startswith(os.path.abspath(MG.REF)), _ref_mod.__file__
    from src.denoising_utils import DenoisingDiffusion
    from src.residuals_darcy import ResidualsDarcy
    from src.unet_model import Unet3D

    cfg = O.unet_config(dim=32, channels=2)
    model = Unet3D(dim=32, channels=2)
    model.load_state_dict(O.make_test_state_dict(cfg, seed=0), strict=True)
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                         device='cpu', bcs='none', domain_length=1.)

    # ---- five successive corrections of the cocogen.pt fields ------------------------------------------------------
    x0p = torch.load(os.path.join(MG.OUT, 'cocogen.pt'), weights_only=True)['x0_pred']
    xin = x0p.permute(0, 2, 3, 1).reshape(2, 4096, 2).clone()
    p_iterates, r = [], None
    for _ in range(N_CALLS):
        xin, r = res.residual_correction(xin)                # in place, like p_sample_loop's post-loop corrections
        p_iterates.append(xin[:, :, 0].reshape(2, 64, 64).detach().clone())
    MG.save('cocogen_steps.pt', dict(x0_pred=x0p, p_iterates=torch.stack(p_iterates), residual_final=r.detach().clone()))

    # ---- ancestral sampling loop with corrections (the sample_loop_6.pt recipe) ----------------------------------------
    model.eval()
    d6 = DenoisingDiffusion(6, 'cpu')

    def loop(**kw):
        torch.manual_seed(77)
        (x_seq, _), aux = d6.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True,
                                           residual_func=res, eval_residuals=True, **kw)
        return x_seq, aux['residual'].detach().clone()

    out = {}
    for tag, kw in (('xt', dict(N_correction=2, M_correction=3, correction_mode='xt')),
                    ('x0', dict(N_correction=2, M_correction=0, correction_mode='x0'))):
        x_seq, r = loop(**kw)
        M = kw['M_correction']
        # On the CPU `.cpu()` returns the tensor itself, so the reference's trajectory entries of the t = 0 step and of
        # the post-loop corrections all alias one tensor that the in-place corrections keep updating.  The tail (the
        # last two loop states, then one state per post-loop correction) is therefore rebuilt from the loop without
        # post-loop corrections and M explicit residual_correction calls, and checked against the aliased final state.
        if M:
            tail, _ = loop(**dict(kw, M_correction=0))
            tail = [v.clone() for v in tail[-2:]]
            cur = tail[-1].permute(0, 2, 3, 1).reshape(1, 4096, 2).clone()
            for _ in range(M):
                cur, r_m = res.residual_correction(cur)
                tail.append(cur.reshape(1, 64, 64, 2).permute(0, 3, 1, 2).detach().clone())
            assert torch.equal(tail[-1], x_seq[-1]) and torch.equal(r_m, r)
        else:
            tail = [v.clone() for v in x_seq[-2:]]
        out[f'{tag}_x_final'] = x_seq[-1].clone()
        out[f'{tag}_residual'] = r
        out[f'{tag}_tail'] = torch.stack(tail)
        out[f'{tag}_len'] = torch.tensor(len(x_seq))
    torch.manual_seed(77)                                    # the draws: x_T, then one z per step (corrections draw none)
    x_T = torch.randn(1, 2, 64, 64)
    zs = [torch.randn(1, 2, 64, 64) for _ in range(6)]
    MG.save('sample_loop_cocogen.pt', dict(x_T=x_T, noises=torch.stack(zs), **out))


if __name__ == '__main__':
    main()
