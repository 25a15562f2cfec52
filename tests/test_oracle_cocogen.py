"""The oracle's CoCoGen corrections (oracle/pidm_oracle.py) against fixtures produced by the UNMODIFIED reference
(oracle/make_golden.py cocogen): successive residual_correction calls and the sampling loop with corrections."""
import pytest
import torch

from checks import rel
from oracle import pidm_oracle as O


def test_successive_corrections_match_reference(golden):
    gd = golden('cocogen_steps.pt')
    n = gd['p_iterates'].shape[0]
    x, r, p_it = O.cocogen_steps(gd['x0_pred'], n)
    p0 = gd['x0_pred'][:, 0]
    for k in range(n):
        # each correction is tiny (step 1e-6 / max dr/dp): compare the accumulated CHANGE of p, not the field
        d_ref = gd['p_iterates'][k] - p0
        assert d_ref.abs().max() > 0
        assert rel(p_it[k] - p0, d_ref) < 1e-3, (k, rel(p_it[k] - p0, d_ref))
    assert torch.equal(x[:, 1], gd['x0_pred'][:, 1])                   # K is never touched
    assert rel(r, gd['residual_final']) < 1e-5


def test_one_step_equals_pidm_oracle():
    """cocogen_steps(x, 1) is pidm_oracle.cocogen_correction (same Jacobian maximum, same gradient)"""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 2, 64, 64, generator=g, dtype=torch.float64)
    x[:, 1] = x[:, 1].exp()
    xa, ra, _ = O.cocogen_steps(x, 1)
    xb, rb = O.cocogen_correction(x)
    assert torch.equal(xa, xb) and torch.equal(ra, rb)


@pytest.mark.parametrize('tag,N,M', [('xt', 2, 3), ('x0', 2, 0)])
def test_sampling_loop_with_corrections_matches_reference(golden, tag, N, M):
    gd = golden('sample_loop_cocogen.pt')
    cfg = O.unet_config(dim=32, channels=2)
    sd = O.make_test_state_dict(cfg, 0)
    with torch.no_grad():
        seq, r = O.p_sample_loop(sd, cfg, gd['x_T'], list(gd['noises']), O.diffusion_tables(6), 6, N_correction=N,
                                 M_correction=M, correction_mode=tag, trajectory=True)
    assert len(seq) == int(gd[f'{tag}_len']) == 7 + M
    tail = gd[f'{tag}_tail']
    for k in range(tail.shape[0]):
        assert rel(seq[len(seq) - tail.shape[0] + k], tail[k]) < 2e-4, k
    assert rel(seq[-1], gd[f'{tag}_x_final']) < 2e-4
    assert rel(r, gd[f'{tag}_residual']) < 2e-3            # residual amplifies x differences by 1/h^2 (as sample_loop_6)
