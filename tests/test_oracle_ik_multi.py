"""CPU: pin tests/ik_multi_oracle.py, the restatement of the multi-link inverse-kinematics kernel that the GPU tests compare
with: with one link it is the single-link oracle, its task-space and joint-space steps are the same step, and its stacked
Jacobian and error are the per-link blocks of tests/ik_oracle.py."""
import pytest
import torch

import ik_multi_oracle as IKM
import ik_oracle as IK
from conftest import urdf_path
from oracle import drm_oracle as O

TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]


def robot64(stem):
    return O.load_robot(urdf_path(stem), torch.float64)


@pytest.mark.parametrize("stem,link", [("iiwa7", "iiwa_link_ee"), ("allegro_hand_description_left", "link_7.0_tip"),
                                       ("2link_robot", "endEffector")])
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "position"])
def test_one_link_is_the_single_link_oracle(stem, link, pose):
    robot = robot64(stem)
    lo, hi = IK.joint_limits(robot, torch.float64)
    q0, tpos, tquat = IKM.problem(robot, [link], 64, seed=1)
    q1, tpos1, tquat1 = IK.problem(robot, link, 64, seed=1)
    assert torch.equal(q0, q1) and torch.equal(tpos[0], tpos1) and torch.equal(tquat[0], tquat1)
    multi = IKM.solve(robot, q0.double(), [link], tpos, tquat if pose else None, lo, hi, max_iters=20)
    single = IK.solve(robot, q0.double(), link, tpos[0], tquat[0] if pose else None, lo, hi, max_iters=20)
    M, n_u = (6 if pose else 3), len(IKM.union_dofs(robot, [link]))
    if M <= n_u:            # the same system: the same arithmetic
        assert torch.equal(multi["q"], single["q"]) and torch.equal(multi["damping"], single["damping"])
        assert torch.equal(multi["converged"], single["converged"])
    else:                   # 2link_robot in pose mode: the joint-space form, equal up to rounding
        assert torch.allclose(multi["q"], single["q"], atol=1e-9)
    assert torch.allclose(multi["pos_err"][0], single["pos_err"], atol=1e-12)
    assert torch.allclose(multi["rot_err"][0], single["rot_err"], atol=1e-12)


def test_task_and_joint_space_steps_agree_in_fp64():
    gen = torch.Generator().manual_seed(2)
    for M, n_u in ((12, 16), (24, 16), (9, 9), (24, 23), (6, 2)):
        J = torch.randn(64, M, n_u, generator=gen, dtype=torch.float64)
        J[:8, :, n_u // 2:] = 0                            # rank-deficient rows: the damping keeps both systems definite
        e = torch.randn(64, M, generator=gen, dtype=torch.float64)
        lam = 10.0 ** (-3 * torch.rand(64, generator=gen, dtype=torch.float64))
        a, ok_a = IKM.step(J, e, lam, "task")
        b, ok_b = IKM.step(J, e, lam, "joint")
        assert bool(ok_a.all()) and bool(ok_b.all())
        err = float((a - b).abs().max() / a.abs().max())
        assert err < 1e-11, (M, n_u, err)
        want_space = "task" if M <= n_u else "joint"
        assert torch.equal(IKM.step(J, e, lam)[0], IKM.step(J, e, lam, want_space)[0])
    # a failed factorisation in joint space rejects the step too
    dq, ok = IKM.step(torch.zeros(2, 6, 2, dtype=torch.float64), torch.ones(2, 6, dtype=torch.float64),
                      torch.tensor([-1.0, float("nan")], dtype=torch.float64))
    assert not bool(ok.any()) and bool((dq == 0).all())


@pytest.mark.parametrize("stem,links", [("allegro_hand_description_left", TIPS), ("iiwa7_allegro", TIPS[:2]),
                                        ("jaco", ["j2n6s300_link_finger_tip_1", "j2n6s300_end_effector"])])
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "position"])
def test_stacked_jacobian_and_error_are_the_per_link_blocks(stem, links, pose):
    robot = robot64(stem)
    q0, tpos, tquat = IKM.problem(robot, links, 32, seed=3)
    q, tpos, tquat = q0.double(), tpos.double(), tquat.double()
    J, e, E, perr, rerr = IKM.evaluate(robot, q, links, tpos, tquat if pose else None)
    R = 6 if pose else 3
    assert J.shape == (32, R * len(links), robot.n_dofs) and e.shape == (32, R * len(links))
    Esum = torch.zeros(32, dtype=torch.float64)
    for l, link in enumerate(links):
        p, quat, Jl = IK.pose_and_jacobian(robot, q, link)
        assert torch.equal(J[:, R * l:R * l + R], Jl[:, :R])
        assert torch.equal(e[:, R * l:R * l + 3], tpos[l] - p)
        if pose:
            assert torch.equal(e[:, R * l + 3:R * l + 6], IK.orientation_error(tquat[l], quat))
        Esum = Esum + (e[:, R * l:R * l + R] ** 2).sum(1)
        assert torch.equal(perr[l], e[:, R * l:R * l + 3].norm(dim=1))
    assert torch.allclose(E, Esum, rtol=1e-14, atol=0)
    # columns outside the union of the paths are zero; inside it every column turns some link (a wrist joint whose axis
    # passes through the tip may not move its position)
    U = IKM.union_dofs(robot, links)
    off = [c for c in range(robot.n_dofs) if c not in U]
    assert bool((J[:, :, off] == 0).all())
    if pose:
        assert bool((J[:, :, U].abs().sum((0, 1)) > 0).all())


def test_fp64_solve_moves_shared_joints_and_converges():
    """iiwa7_allegro, two fingertips of different fingers: the arm joints are shared, the other fingers never move."""
    robot = robot64("iiwa7_allegro")
    links = ["link_3.0_tip", "link_7.0_tip"]
    lo, hi = IK.joint_limits(robot, torch.float64)
    q0, tpos, tquat = IKM.problem(robot, links, 128, seed=4)
    r = IKM.solve(robot, q0.double(), links, tpos, tquat, lo, hi, max_iters=100)
    frac = float(r["converged"].double().mean())
    print(f"iiwa7_allegro two tips pose: converged {frac:.3f}")
    assert frac >= 0.7, frac
    conv = r["converged"]
    assert bool((r["pos_err"][:, conv] <= 1e-4).all()) and bool((r["rot_err"][:, conv] <= 1e-3).all())
    U = IKM.union_dofs(robot, links)
    off = [c for c in range(robot.n_dofs) if c not in U]
    assert off and torch.equal(r["q"][:, off], q0.double().clamp(lo, hi)[:, off])
    # the reported errors are those of the returned q
    for l, link in enumerate(links):
        p, _ = O.forward_kinematics(robot, r["q"], link)
        assert torch.allclose((tpos[l].double() - p).norm(dim=1), r["pos_err"][l], atol=1e-12)
