"""Unet3D(padding_mode='circular') on the CPU: the parameter surface against the reference, and the oracle's
padding_mode='circular' (oracle/pidm_oracle.py) against fixtures produced by the UNMODIFIED reference
(oracle/make_golden.py circular)."""
import pytest
import torch
import torch.nn.functional as F

from checks import rel
from oracle import pidm_oracle as O

CIRCULAR = O.unet_config(dim=32, channels=2, padding_mode='circular')


def test_circular_unet_keys_and_seeded_init(golden):
    """reference key list; under seed 0 every tensor is the zeros-mode initial value (six up-sampling keys renamed)"""
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    torch.manual_seed(0)
    sd = Unet3D(dim=32, channels=2, padding_mode='circular').state_dict()
    assert list(sd.keys()) == golden('unet_circular_keys.pt')['keys']
    torch.manual_seed(0)
    sd0 = Unet3D(dim=32, channels=2).state_dict()
    assert [k.replace('.conv_transpose.', '.') for k in sd] == list(sd0.keys()) and len(sd) == 317
    renamed = [k for k in sd if 'conv_transpose' in k]
    assert len(renamed) == 6
    for k, v in sd.items():
        assert torch.equal(v, sd0[k.replace('.conv_transpose.', '.')]), k
    gd = golden('unet_init_seed0.pt')
    for k, v in sd.items():
        ref = gd[k.replace('.conv_transpose.', '.')]
        assert abs(v.double().sum().item() - ref[0].item()) < 1e-9, k


def test_circular_load_state_dict_is_strict():
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    m = Unet3D(dim=32, channels=2, padding_mode='circular')
    m.load_state_dict(O.make_test_state_dict(CIRCULAR, 0), strict=True)
    with pytest.raises(RuntimeError):
        # a zeros checkpoint has the old up-sampling keys
        m.load_state_dict(O.make_test_state_dict(O.unet_config(dim=32, channels=2), 0), strict=True)


def test_circular_conv_specs():
    """every padded spatial convolution is circular except emb_conv[2] (zero-padded in the reference)"""
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    m = Unet3D(dim=32, channels=2, padding_mode='circular')
    circ = [s for s in m._packer.specs if s.circular]
    assert len(circ) == 45
    assert sorted({(s.kind, s.kh, s.stride, s.halo, s.dgrad_halo) for s in circ}) == [
        ('conv', 3, 1, 1, 1), ('conv', 4, 2, 1, 1), ('conv', 7, 1, 3, 3), ('convT', 4, 2, 1, 1)]
    assert not m._spec[id(m.emb_conv[2])].circular
    assert not any(s.circular for s in Unet3D(dim=32, channels=2)._packer.specs)


def test_unknown_padding_mode_raises():
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    with pytest.raises(ValueError):
        Unet3D(dim=32, channels=2, padding_mode='reflect')


def test_periodic_transposed_conv_identity():
    """the reference's circular pad 2 + padding 5 equals circular pad 1 + padding 3 (the engine's form), in fp64"""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 8, 8, 8, generator=g, dtype=torch.float64)
    w = torch.randn(8, 4, 4, 4, generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(F.pad(x, (2,) * 4, mode='circular'), w, stride=2, padding=5)
    assert torch.equal(O.conv_transpose_circular(x, w, None), ref)


def test_circular_oracle_forward_matches_reference(golden):
    gd = golden('unet_circular_fwd.pt')
    cfg = O.unet_config(dim=32, channels=2)
    with torch.no_grad():
        y, taps = O.unet_forward(O.make_test_state_dict(CIRCULAR, 0), CIRCULAR, gd['x'], gd['t'], return_taps=True)
        y0 = O.unet_forward(O.make_test_state_dict(cfg, 0), cfg, gd['x'], gd['t'])
    for k in ('init_conv', 'downs.0.0', 'downs.0.2', 'mid_attn', 'ups.0'):
        assert rel(O.golden_sample(taps[k]), gd['tap_' + k]) < 2e-5, k
    assert rel(y, gd['y']) < 5e-5
    assert rel(y0, gd['y']) > 1e-2                        # the zero-padded network differs


@pytest.mark.parametrize('shift', [(8, 16), (24, 40), (0, 8)])
def test_circular_oracle_rolls_exactly(shift):
    """with periodic padding every layer commutes with a roll by a multiple of 8 pixels (the coarsest level is 8x8)"""
    sd = {k: v.double() for k, v in O.make_test_state_dict(CIRCULAR, 0).items()}
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 2, 64, 64, generator=g, dtype=torch.float64)
    t = torch.tensor([17])
    with torch.no_grad():
        y = O.unet_forward(sd, CIRCULAR, x, t)
        ys = O.unet_forward(sd, CIRCULAR, torch.roll(x, shift, (2, 3)), t)
    assert (ys - torch.roll(y, shift, (2, 3))).abs().max().item() < 1e-10
