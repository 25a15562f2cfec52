"""Residual-gradient guidance on the CPU: the oracle against one training iteration of the unmodified reference
(oracle/make_golden.py guidance), the guidance no-grad list and the sharded classifier-free mask draw."""
import os

import torch

from checks import rel
from oracle import pidm_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _names(fname):
    with open(os.path.join(GOLDEN, fname)) as f:
        return sorted(k for k in f.read().split() if not k.endswith('rotary_emb.freqs'))


def test_oracle_matches_reference_guidance_step(golden):
    gd = golden('darcy_guidance_step.pt')
    assert 0 < int(gd['null_mask'].sum()) < len(gd['null_mask'])          # both branches of the mask are exercised
    cfg = O.unet_config(dim=32, channels=2)
    sdr = {k: v.clone().requires_grad_('freqs' not in k) for k, v in O.make_test_state_dict(cfg, 0).items()}
    loss, _ = O.darcy_training_loss(sdr, cfg, gd['x0'], gd['t'], gd['noise'], O.diffusion_tables(100),
                                    guidance_null_mask=gd['null_mask'])
    assert abs(loss.item() / gd['loss'].item() - 1) < 2e-5
    loss.backward()
    n = int(gd['grad_sample'])
    worst = {k: rel(O.golden_sample(sdr[k[5:]].grad, n), v) for k, v in gd.items()
             if k.startswith('grad_') and k not in ('grad_norm', 'grad_sample')}
    assert 'grad_emb_conv.0.weight' in worst and 'grad_combine_conv.bias' in worst
    assert max(worst.values()) < 1e-3, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in sdr.values() if p.grad is not None)).item()
    assert abs(gn / gd['grad_norm'].item() - 1) < 1e-4


def test_guidance_no_grad_list_matches_reference():
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    m = Unet3D(dim=32, channels=2)
    ref = _names('params_without_grad_guidance.txt')
    assert sorted(m.unused_parameter_names(guidance=True)) == ref
    default = _names('params_without_grad.txt')
    assert sorted(m.unused_parameter_names()) == default
    assert ref == [k for k in default if not k.startswith(('emb_conv.', 'combine_conv.'))]


def test_sharded_mask_draw_is_a_slice_of_the_global_draw():
    from physicsinformeddiffusionmodels_b200.unet_model import draw_null_mask
    world, B = 4, 16
    torch.manual_seed(3)
    full = draw_null_mask(world * B, 0.1, 'cpu')
    assert 0 < int(full.sum()) < world * B
    for rank in range(world):
        torch.manual_seed(3)
        shard = draw_null_mask(B, 0.1, 'cpu', (rank, world))
        assert torch.equal(shard, full[rank * B:(rank + 1) * B])
    torch.manual_seed(3)
    mine = draw_null_mask(B, 0.1, 'cpu')
    torch.manual_seed(3)
    assert torch.equal(mine, torch.zeros(B).float().uniform_(0, 1) < 0.1)        # reference prob_mask_like
    assert draw_null_mask(B, 1., 'cpu').all() and not draw_null_mask(B, 0., 'cpu').any()
