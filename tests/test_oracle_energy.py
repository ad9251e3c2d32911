"""CPU: pin the energy / momentum / centre-of-mass oracle (tests/energy_oracle.py) in fp64: against the reference's own
per-body state (tests/golden/make_golden_energy.py -> <robot>.energy.npz), and against the identities that tie it to the
rest of the oracle -- momentum = H qd, kinetic = 1/2 qd . momentum, J_com = d com / dq, dV/dq = the RNEA gravity torque,
and conservation of energy along the forward dynamics."""
import copy
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, URDFS, urdf_path
import derivatives_oracle as D
import energy_oracle as E
from oracle import drm_oracle as O

dt = torch.float64
GOLDEN = ["iiwa7", "panda_no_gripper", "fetch_arm_no_gripper", "2link_robot", "allegro_hand_description_left_small_damping"]
KEYS = ("kinetic", "potential", "momentum", "com", "com_velocity", "com_jacobian")


def robot_of(stem, nonsym):
    robot = O.load_robot(urdf_path(stem), dt)
    return D.perturbed(robot) if nonsym else robot


def rel_err(got, want):
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_oracle_matches_reference_per_body_state(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".energy.npz"), allow_pickle=False)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"])
        inertia[0] = robot.inertia[0]
        robot.inertia = inertia
    robot = robot.to(dt)
    q, qd = (torch.tensor(g[k]).to(dt) for k in ("q", "qd"))
    pre = "" if tag == "sym" else "nonsym."
    for key, got in zip(KEYS, E.energy_momentum(robot, q, qd)):
        want = torch.tensor(g[pre + key]).to(dt)
        # the goldens are the reference's fp32 evaluation
        assert rel_err(got, want) <= 2e-5, (key, rel_err(got, want))


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_momentum_is_mass_matrix_times_qd_and_kinetic_is_half_qd_momentum(stem, nonsym):
    robot = robot_of(stem, nonsym)
    q, qd, _ = O.sample_inputs(robot, 7, seed=31, dtype=dt)
    kin, _, mom, _, comv, jcom = E.energy_momentum(robot, q, qd)
    H = D.mass_matrix(robot, q)
    want = (H @ qd.unsqueeze(2)).squeeze(2)
    assert rel_err(mom, want) <= 1e-12
    assert rel_err(kin, 0.5 * (qd * mom).sum(-1)) <= 1e-12
    assert rel_err(comv, (jcom @ qd.unsqueeze(2)).squeeze(2)) <= 1e-12


@pytest.mark.parametrize("stem", sorted(URDFS))
def test_com_jacobian_and_gravity_torque_are_derivatives(stem):
    robot = robot_of(stem, False)
    q, _, _ = O.sample_inputs(robot, 5, seed=32, dtype=dt)
    B, n = q.shape
    _, _, _, _, _, jcom = E.energy_momentum(robot, q)
    eps = 1e-6
    d_com, d_pot = [], []
    for k in range(n):
        e = torch.zeros(n, dtype=dt)
        e[k] = eps
        _, vp, _, cp, _, _ = E.energy_momentum(robot, q + e)
        _, vm, _, cm, _, _ = E.energy_momentum(robot, q - e)
        d_com.append((cp - cm) / (2 * eps))
        d_pot.append((vp - vm) / (2 * eps))
    d_com, d_pot = torch.stack(d_com, dim=2), torch.stack(d_pot, dim=1)
    assert rel_err(jcom, d_com) <= 1e-7
    z = torch.zeros_like(q)
    tau_g = O.inverse_dynamics(robot, q, z, z, True, False)
    assert rel_err(d_pot, tau_g) <= 1e-7
    assert rel_err(E.GRAVITY * E.total_mass(robot) * jcom[:, 2], tau_g) <= 1e-12


@pytest.mark.parametrize("stem", sorted(URDFS))
def test_power_balance_along_forward_dynamics(stem):
    """dE/dt = grad_q E . qd + momentum . qdd equals the power qd . f of the applied joint forces (symmetric inertias, no
    damping), with qdd from the oracle's articulated-body algorithm."""
    robot = robot_of(stem, False)
    q, qd, _ = O.sample_inputs(robot, 6, seed=33, dtype=dt)
    f = torch.randn(q.shape, generator=torch.Generator().manual_seed(34), dtype=dt)
    qdd = O.forward_dynamics(robot, q, qd, f, True, False)
    qa = q.clone().requires_grad_(True)
    kin, pot, mom, _, _, _ = E.energy_momentum(robot, qa, qd)
    grad_q, = torch.autograd.grad((kin + pot).sum(), [qa])
    power = (grad_q * qd).sum(-1) + (mom.detach() * qdd).sum(-1)
    want = (qd * f).sum(-1)
    scale = (grad_q.abs() * qd.abs()).sum(-1) + (mom.detach().abs() * qdd.abs()).sum(-1) + want.abs()
    assert float(((power - want).abs() / scale).max()) <= 1e-10


def test_massless_model_gives_zeros():
    robot = copy.copy(O.load_robot(urdf_path("iiwa7"), dt))
    robot.mass = torch.zeros_like(robot.mass)
    q, qd, _ = O.sample_inputs(robot, 4, seed=35, dtype=dt)
    kin, pot, mom, com, comv, jcom = E.energy_momentum(robot, q, qd)
    for t in (pot, com, comv, jcom):
        assert torch.equal(t, torch.zeros_like(t))
    assert bool(torch.isfinite(kin).all() and torch.isfinite(mom).all())
