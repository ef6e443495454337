"""Entry point with the path bodywork.yaml names (``executable_module_path:
mlops_simulation/stage_1_train_model.py``, bodywork.yaml:9): runs the GPU stage."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bodywork_mlops_demo_b200.stage_1_train_model import run  # noqa: E402

if __name__ == "__main__":
    sys.exit(run())
