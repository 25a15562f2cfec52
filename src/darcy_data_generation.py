"""Drop-in module name of the reference (`src/darcy_data_generation.py`): re-exports the engine's implementation, whose
main() writes the reference's four CSV files through the GPU path (seeds seed0 + i instead of pid * time)."""
from physicsinformeddiffusionmodels_b200.darcy_data_generation import *  # noqa: F401,F403
from physicsinformeddiffusionmodels_b200.darcy_data_generation import main

if __name__ == '__main__':
    main()
