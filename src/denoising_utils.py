"""Drop-in module name of the reference (`src/denoising_utils.py`): re-exports the engine's implementation so that the
reference's main.py / sample.py run unchanged against this repository."""
from physicsinformeddiffusionmodels_b200.denoising_utils import *  # noqa: F401,F403
