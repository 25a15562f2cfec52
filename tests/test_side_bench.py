"""scripts/side_bench.py on the CPU: the byte and flop counts its rates divide by, the halo census of the circular Darcy
U-Net, and that a measurement on a machine without a GPU fails instead of falling back."""
import importlib.util
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, 'scripts', 'side_bench.py')


@pytest.fixture(scope='module')
def side_bench():
    spec = importlib.util.spec_from_file_location('side_bench', SCRIPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_algorithmic_byte_and_flop_counts(side_bench):
    assert side_bench.DARCY_BYTES == {'fwd': 81_920, 'loss': 98_304}
    assert side_bench.GUIDANCE_BYTES == {'abs_residual_grad': 65_536, 'cond_embed_fwd': 294_912}
    assert (side_bench.FACTOR_FLOP, side_bench.FACTOR_BYTES) == (159_744_000, 12_845_056)


def test_halo_census_of_the_circular_darcy_unet(side_bench):
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    model = Unet3D(dim=32, channels=2, padding_mode='circular')
    # 45 forward operands and 44 backward dy per training step, 378 MB written at batch 32 (DESIGN.md §7)
    assert side_bench.halo_census(model, 32, 64) == (45, 44, 378_413_056)


def test_measuring_without_a_gpu_fails():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    out = subprocess.run([sys.executable, SCRIPT, 'periodic'], capture_output=True, text=True, timeout=600, cwd=ROOT,
                         env=env)
    assert out.returncode != 0
    assert 'no CUDA device' in out.stderr, out.stderr[-2000:]
