"""deepi2p_b200 -- H100-native (sm_90a) inverse-camera-projection registration path of DeepI2P.

Scope (SURVEY.md section 8): the Ceres-backed solver FrustumRegistration.solvePGivenK and the
multi-start loop around it, plus the two CUDA ops of the classifier (index_max, ball_query),
rebuilt as hand-written CUDA behind a C ABI (include/deepi2p_b200.h) and the reference's own
Python extension API (deepi2p_b200/dropin/).  Nothing else of DeepI2P is here.
"""
import os
import sys

__version__ = "0.1.0"

_DROPIN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin")


def install_dropins():
    """Make `import FrustumRegistration`, `import index_max`, `import ball_query` resolve to the
    CUDA implementations (prepends deepi2p_b200/dropin to sys.path)."""
    if _DROPIN_DIR not in sys.path:
        sys.path.insert(0, _DROPIN_DIR)
    return _DROPIN_DIR
