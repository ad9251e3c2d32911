"""CPU: pin the regressor oracle (tests/regressor_oracle.py): Y . pi reproduces the oracle's inverse dynamics on every
shipped robot, flag combination and symmetric / non-symmetric inertia; the structural zeros are exact; and, mapped to the
URDF parameters by the chain rule, Y is the reference's own autograd Jacobian (tests/golden/make_golden_regressor.py ->
<robot>.regressor.npz)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, URDFS, urdf_path
import derivatives_oracle as D
import regressor_oracle as R
from oracle import drm_oracle as O

dt = torch.float64
FLAGS = [(True, True), (True, False), (False, True), (False, False)]
GOLDEN = ["iiwa7", "panda_no_gripper", "fetch_arm_no_gripper", "2link_robot", "allegro_hand_description_left_small_damping"]


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_regressor_times_parameters_is_the_inverse_dynamics(stem, nonsym):
    robot = O.load_robot(urdf_path(stem), dt)
    if nonsym:
        robot = D.perturbed(robot)
    q, qd, qdd = O.sample_inputs(robot, 9, seed=21, dtype=dt)
    pi = R.table_params(robot)
    for grav, damp in FLAGS:
        Y = R.regressor(robot, q, qd, qdd, grav, damp)
        tau = O.inverse_dynamics(robot, q, qd, qdd, grav, damp)
        got = torch.einsum("bilk,lk->bi", Y, pi)
        scale = torch.einsum("bilk,lk->bi", Y.abs(), pi.abs()).max()
        assert float((got - tau).abs().max()) <= 1e-12 * float(scale), (stem, grav, damp)
        zero = R.structural_zeros(robot, damp)
        assert torch.all(Y[:, zero] == 0), (stem, grav, damp)
        if damp:                                               # damping columns are qd of the link's own dof
            for l in robot.controlled:
                assert torch.equal(Y[:, robot.dof[l], l, 13], qd[:, robot.dof[l]])


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_oracle_matches_reference_autograd(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".regressor.npz"), allow_pickle=False)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"])
        inertia[0] = robot.inertia[0]
        robot.inertia = inertia
    robot = robot.to(dt)
    q, qd, qdd = (torch.tensor(g[k]).to(dt) for k in ("q", "qd", "qdd"))
    pre = "" if tag == "sym" else "nonsym."
    N = len(robot.names)
    for grav, damp in ((1, 1), (0, 0)):
        J = R.urdf_parameter_jacobians(R.regressor(robot, q, qd, qdd, bool(grav), bool(damp)), robot.mass, robot.com)
        for pname, want_of in J.items():
            for link in range(1, N):
                key = f"{pre}g{grav}d{damp}.{pname}.{link}"
                if key not in g:
                    assert pname == "joint_damping" and robot.dof[link] < 0
                    continue
                want, got = torch.tensor(g[key]).to(dt), want_of[:, :, link]
                scale = float(want.abs().max())
                assert float((got - want).abs().max()) <= 1e-4 * max(scale, 1e-3), (key, scale)
