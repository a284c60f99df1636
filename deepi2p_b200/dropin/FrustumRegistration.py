"""Drop-in for the reference's pybind11 module `FrustumRegistration`
(evaluation/frustum_reg/src/registration.cpp:190-213): same module name, same function name,
same keyword names, same return tuple -- backed by the sm_90a batched solver instead of Ceres.

    import deepi2p_b200; deepi2p_b200.install_dropins()
    import FrustumRegistration
    P, final_cost, residuals = FrustumRegistration.solvePGivenK(pc, labels, K, ry, t, H, W, lb, ub, 500, False, True)

`solve` is an alias (BASELINE.json's name for the same call); `solve_batch` / `register_batch`
are the batched entry points that replace the caller's fork-per-solve loop.
"""
from deepi2p_b200.frustum import register_batch, solve_batch, solve_p_given_k  # noqa: F401

__version__ = "b200-1"
__doc__ = "Frustum Registration"


def solvePGivenK(points, labels, K, init_y_angle, init_T, H, W, t_xyz_lower_bound, t_xyz_upper_bound, max_iter,
                 is_debug, is_2d):
    return solve_p_given_k(points, labels, K, init_y_angle, init_T, H, W, t_xyz_lower_bound, t_xyz_upper_bound,
                           max_iter, is_debug, is_2d)


solve = solvePGivenK
