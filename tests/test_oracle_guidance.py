"""Residual-gradient guidance on the CPU: the guidance no-grad list and the sharded classifier-free mask draw.  The
oracle against one training iteration of the unmodified reference (darcy_guidance_step) is a row of
test_oracle_golden.py."""
import os

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _names(fname):
    with open(os.path.join(GOLDEN, fname)) as f:
        return sorted(k for k in f.read().split() if not k.endswith('rotary_emb.freqs'))


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
