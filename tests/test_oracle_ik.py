"""CPU: pin tests/ik_oracle.py, the restatement of the inverse-kinematics kernel's algorithm that the GPU tests compare with:
its orientation error against scipy's rotation vectors, one step against the closed form via numpy.linalg, and the
converged fraction of the fp64 solve on reachable targets."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import ik_oracle as IK
from conftest import urdf_path
from oracle import drm_oracle as O


def rotvec(target_quat, quat):
    return IK.orientation_error(torch.tensor(target_quat), torch.tensor(quat)).numpy()


def test_orientation_error_is_the_rotation_vector_of_target_times_inverse():
    rs = Rotation.random(500, random_state=1)
    rt = Rotation.random(500, random_state=2)
    want = (rt * rs.inv()).as_rotvec()
    got = rotvec(rt.as_quat(), rs.as_quat())
    np.testing.assert_allclose(got, want, atol=1e-12)
    # either sign of either quaternion, and a target that is not normalised
    for st, ss in ((-1, 1), (1, -1), (-1, -1), (3.5, 1)):
        np.testing.assert_allclose(rotvec(st * rt.as_quat(), ss * rs.as_quat()), want, atol=1e-12)


def test_orientation_error_near_pi_and_at_zero():
    gen = np.random.default_rng(3)
    axes = gen.normal(size=(200, 3))
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    angles = np.pi - np.concatenate([np.zeros(50), 10.0 ** -gen.uniform(1, 8, 150)])
    rs = Rotation.random(200, random_state=4)
    rt = Rotation.from_rotvec(axes * angles[:, None]) * rs
    got = rotvec(rt.as_quat(), rs.as_quat())
    np.testing.assert_allclose(np.linalg.norm(got, axis=1), angles, atol=1e-9)
    want = (rt * rs.inv()).as_rotvec()
    # at exactly pi the axis sign is a convention: compare up to sign there, exactly elsewhere
    sign = np.where(np.sum(got * want, axis=1) < 0, -1.0, 1.0)
    np.testing.assert_allclose(got[50:], want[50:], atol=1e-7)
    np.testing.assert_allclose(got[:50] * sign[:50, None], want[:50], atol=1e-9)
    same = rs.as_quat()
    assert np.abs(rotvec(same, same)).max() < 1e-15 and np.abs(rotvec(same, -same)).max() < 1e-15
    ident = np.array([[0.0, 0.0, 0.0, 1.0]])                # s = 0: the error is exactly zero, not 0/0
    assert np.all(rotvec(ident, ident) == 0) and np.all(rotvec(ident, -ident) == 0)


def test_one_step_is_the_damped_least_squares_closed_form():
    gen = torch.Generator().manual_seed(5)
    for M in (3, 6):
        J = torch.randn(64, M, 7, generator=gen, dtype=torch.float64)
        J[:8, :, 3:] = 0                                  # rank-deficient rows: damping keeps the system definite
        e = torch.randn(64, M, generator=gen, dtype=torch.float64)
        lam = 10.0 ** (-4 * torch.rand(64, generator=gen, dtype=torch.float64))
        dq, ok = IK.step(J, e, lam)
        assert bool(ok.all())
        Jn, en, ln = J.numpy(), e.numpy(), lam.numpy()
        want = np.stack([Jn[b].T @ np.linalg.solve(Jn[b] @ Jn[b].T + ln[b] * np.eye(M), en[b]) for b in range(64)])
        np.testing.assert_allclose(dq.numpy(), want, rtol=1e-9, atol=1e-12)
    # a failed factorisation rejects the step: no motion
    J = torch.zeros(2, 3, 4, dtype=torch.float64)
    dq, ok = IK.step(J, torch.ones(2, 3, dtype=torch.float64), torch.tensor([-1.0, float("nan")], dtype=torch.float64))
    assert not bool(ok.any()) and bool((dq == 0).all())


def test_solve_state_machine_on_a_two_link_arm():
    """Accepts halve the damping, rejections quadruple it, converged rows stop, limits hold, K = 0 evaluates only."""
    robot = O.load_robot(urdf_path("2link_robot"), torch.float64)
    lo, hi = IK.joint_limits(robot, torch.float64)
    q0, tpos, _ = IK.problem(robot, "endEffector", 64, seed=6)
    q0 = q0.double()
    r0 = IK.solve(robot, q0, "endEffector", tpos, lower=lo, upper=hi, max_iters=0)
    assert torch.equal(r0["q"], q0.clamp(lo, hi)) and bool((r0["damping"] == IK.DAMPING_INIT).all())
    r1 = IK.solve(robot, q0, "endEffector", tpos, lower=lo, upper=hi, max_iters=1)
    lam = r1["damping"]
    assert bool(torch.where(r1["accepted"], lam == IK.DAMPING_INIT / 2, lam == 4 * IK.DAMPING_INIT).all())
    assert bool((r1["pos_err"] <= r0["pos_err"]).all())
    r = IK.solve(robot, q0, "endEffector", tpos, lower=lo, upper=hi, max_iters=50)
    assert float(r["converged"].double().mean()) > 0.9
    assert bool(((r["q"] >= lo) & (r["q"] <= hi)).all())
    conv = r["converged"]
    assert bool((r["pos_err"][conv] <= 1e-4).all())
    # chaining: 50 iterations in one solve equal 50 one-iteration solves that pass q and the damping on
    q, damp = q0, None
    for _ in range(50):
        s = IK.solve(robot, q, "endEffector", tpos, lower=lo, upper=hi, damping=damp, max_iters=1)
        q, damp = s["q"], s["damping"]
    assert torch.equal(q, r["q"]) and torch.equal(damp, r["damping"])


@pytest.mark.parametrize("stem,link,pose", [("iiwa7", "iiwa_link_ee", True), ("panda_no_gripper", "panda_virtual_ee_link", True),
                                            ("iiwa7", "iiwa_link_ee", False)])
def test_fp64_oracle_converges_on_reachable_targets(stem, link, pose):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    lo, hi = IK.joint_limits(robot, torch.float64)
    q0, tpos, tquat = IK.problem(robot, link, 256, seed=0)
    r = IK.solve(robot, q0.double(), link, tpos, tquat if pose else None, lo, hi, max_iters=100)
    frac = float(r["converged"].double().mean())
    print(f"{stem} {'pose' if pose else 'position'}: converged {frac:.3f}")
    assert frac >= 0.9, frac
    conv = r["converged"]
    assert bool((r["pos_err"][conv] <= 1e-4).all()) and bool((r["rot_err"][conv] <= 1e-3).all())
    # the reported errors are those of the returned q
    p, quat = O.forward_kinematics(robot, r["q"], link)
    assert torch.allclose((tpos.double() - p).norm(dim=1), r["pos_err"], atol=1e-12)
    if pose:
        assert torch.allclose(IK.orientation_error(tquat.double(), quat).norm(dim=1), r["rot_err"], atol=1e-12)
