"""configs[0] (toy study, main_toy.py): the libpidm-backed `denoising_toy_utils` against the golden fixture produced by
the UNMODIFIED reference module (tests/golden/toy.pt): loss, tracked scalars, gradients in the three
(model_pred_mode, x0_estimation) combinations the driver offers, and the ancestral loop with the reference's draws."""
import pytest
import torch

from checks import rel

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def residual_func(x):
    return torch.sum(x ** 2, dim=1) - 1.0


def ineq_func(x):
    density = torch.sum(torch.abs(x), dim=1)
    return torch.relu(density - 1.0), density


def opt_func(x):
    return x[:, 0]


def build(gd):
    from physicsinformeddiffusionmodels_b200 import denoising_toy_utils as T
    model = T.ConditionalModel(2, 100).to(DEV)
    model.load_state_dict({k[3:]: v for k, v in gd.items() if k.startswith('sd_')})
    return T, model


@pytest.mark.parametrize('tag,mode,ddim', [('x0_mean', 'x0', False), ('x0_sample', 'x0', True), ('eps_sample', 'eps', True)])
def test_toy_loss_matches_reference(golden, monkeypatch, tag, mode, ddim):
    gd = golden('toy.pt')
    T, model = build(gd)
    dd = T.create_diff_dict(100, DEV)
    t_half = gd['t'][:65].to(DEV)                          # the reference draws B//2+1 values and mirrors them (:440-441)
    draws = iter([gd['noise'].to(DEV)] + [torch.zeros(128, 2, device=DEV)] * 4)
    monkeypatch.setattr(torch, 'randint', lambda *a, **k: t_half)
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(draws))
    loss, data_l, res_l, ineq_l, opt_l = T.model_estimation_loss(
        model, gd['x0'].to(DEV), 100, dd, model_pred_mode=mode, residual_func=residual_func, ineq_func=ineq_func,
        opt_func=opt_func, c_data=1.0, c_residual=0.005, c_ineq=0.3, lambda_opt=0.01, use_ddim_x0=ddim,
        reduced_ddim_steps=0)
    monkeypatch.undo()
    assert abs(loss.item() / gd[tag + '_loss'].item() - 1) < 2e-5
    for a, b in zip((data_l, res_l, ineq_l, opt_l), gd[tag + '_tracked'].tolist()):
        assert abs(a - b) < 2e-5 * max(1.0, abs(b)), (a, b)
    loss.backward()
    assert rel(model.lin3.weight.grad, gd[tag + '_grad_lin3']) < 1e-4
    assert rel(model.lin1.lin.weight.grad, gd[tag + '_grad_lin1']) < 1e-4
    assert rel(model.lin2.embed.weight.grad, gd[tag + '_grad_embed2']) < 1e-4


def test_toy_sampling_loop_matches_reference(golden, monkeypatch):
    gd = golden('toy.pt')
    T, model = build(gd)
    model.eval()
    d8 = T.create_diff_dict(8, DEV)
    draws = iter(list(gd['loop_draws'].to(DEV)))
    monkeypatch.setattr(torch, 'randn', lambda *a, **k: next(draws))
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(draws))
    xs, mo, x0e = T.p_sample_loop(model, [64, 2], 8, d8, model_pred_mode='x0', save_output=False, surpress_noise=True)
    monkeypatch.undo()
    assert len(xs) == 9 and not xs[-1].is_cuda
    assert rel(xs[-1], gd['loop_final']) < 1e-4


def test_toy_rejects_cpu_tensors_and_mu_mode(golden):
    gd = golden('toy.pt')
    T, model = build(gd)
    dd = T.create_diff_dict(100, DEV)
    with pytest.raises(RuntimeError):
        T.model_estimation_loss(model.cpu(), gd['x0'], 100, dd, model_pred_mode='x0', residual_func=residual_func)
    with pytest.raises(NotImplementedError):
        T.model_estimation_loss(model.to(DEV), gd['x0'].to(DEV), 100, dd, model_pred_mode='mu', residual_func=residual_func)
