"""CPU: pin the oracle's dynamics Jacobians (autograd of oracle/drm_oracle.py) against the reference's own autograd
Jacobians (tests/golden/make_golden_derivatives.py -> <robot>.deriv.npz), and pin why the forward-dynamics derivatives
must differentiate the articulated-body algorithm itself: the shortcut -H^-1 dtau is exact for symmetric inertias only."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, assert_close, urdf_path
import derivatives_oracle as D
from oracle import drm_oracle as O

DERIV_ROBOTS = ["iiwa7", "panda_no_gripper", "fetch_arm_no_gripper", "2link_robot", "allegro_hand_description_left_small_damping"]


def load_deriv(stem):
    return np.load(os.path.join(GOLDEN_DIR, stem + ".deriv.npz"), allow_pickle=False)


def golden_robot(stem, dtype, g, tag):
    robot = O.load_robot(urdf_path(stem), dtype)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=dtype)
        inertia[0] = robot.inertia[0]
        robot.inertia = inertia
    return robot


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("stem", DERIV_ROBOTS)
def test_oracle_jacobians_match_reference_autograd(stem, dtype, tag):
    g = load_deriv(stem)
    robot = golden_robot(stem, dtype, g, tag)
    q, qd, qdd, f = (torch.tensor(g[k], dtype=dtype) for k in ("q", "qd", "qdd", "f"))
    pre = "" if tag == "sym" else "nonsym."

    def close(got, key):
        ref = g[pre + key]
        assert_close(got.detach().numpy(), ref, rtol=2e-4, atol=2e-5 * max(np.abs(ref).max(), 1e-6), what=pre + key)

    for grav in (0, 1):
        for damp in (0, 1):
            dq, dqd = D.inverse_dynamics_derivatives(robot, q, qd, qdd, bool(grav), bool(damp))
            close(dq, f"id.g{grav}d{damp}.dq")
            close(dqd, f"id.g{grav}d{damp}.dqd")
    for damp in (0, 1):
        dq, dqd, df = D.forward_dynamics_derivatives(robot, q, qd, f, True, bool(damp))
        close(dq, f"fd.g1d{damp}.dq")
        close(dqd, f"fd.g1d{damp}.dqd")
        close(df, f"fd.g1d{damp}.df")


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("stem", ["iiwa7", "allegro_hand_description_left"])
def test_shortcut_holds_for_symmetric_inertias_only(stem):
    """-H^-1 dtau/dx at qdd = FD equals dqdd/dx, and H^-1 equals dqdd/df, when every inertia is symmetric (fp64).  With
    non-symmetric inertias the reference's articulated-body algorithm is not the inverse of its RNEA, and the shortcut's
    dqdd/dq is off by more than 1e-3 relative, while dqdd/df still equals the ABA(q, 0, e_j) columns."""
    dt = torch.float64
    robot = O.load_robot(urdf_path(stem), dt)
    q, qd, _ = O.sample_inputs(robot, 6, seed=5, dtype=dt)
    f = torch.randn(6, robot.n_dofs, generator=torch.Generator().manual_seed(6), dtype=dt)
    for r, symmetric in ((robot, True), (D.perturbed(robot), False)):
        exact = D.forward_dynamics_derivatives(r, q, qd, f, True, True)
        short = D.shortcut_forward_dynamics_derivatives(r, q, qd, f, True, True)
        cols = torch.stack([O.forward_dynamics(r, q, torch.zeros_like(qd), torch.eye(r.n_dofs, dtype=dt)[j].expand_as(f),
                                               False, False) for j in range(r.n_dofs)], dim=2)
        assert _rel(exact[2], cols) < 1e-12
        if symmetric:
            for a, b in zip(short, exact):
                assert _rel(a, b) < 1e-9
        else:
            assert _rel(short[0], exact[0]) > 1e-3
