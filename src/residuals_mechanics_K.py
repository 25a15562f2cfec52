"""Drop-in module name of the reference (`src/residuals_mechanics_K.py`): re-exports the engine's implementation so that the
reference's main.py / sample.py run unchanged against this repository."""
from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import *  # noqa: F401,F403
