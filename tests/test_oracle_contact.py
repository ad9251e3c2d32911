"""CPU: pin the contact oracle (tests/contact_oracle.py) against the reference's own evaluation
(tests/golden/make_golden_contact.py -> <robot>.contact.npz), a direct KKT solve with the oracle's mass matrix, the
constraint identities, the kinetic energy across impulses and the unsolved rule on redundant constraint sets."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, assert_close, urdf_path
import contact_oracle as C
import derivatives_oracle as D
import osd_oracle as S
from oracle import drm_oracle as O

TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
TRI = ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"]
GOLDEN = ["2link_robot", "iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro", "trifinger_edu"]
# (robot, links, position_only): sets the joints can satisfy, so mu = 0 solves them away from singular configurations.  (Two
# Allegro fingertips in pose mode are not such a set: each finger's last three joints are parallel.)
CASES = [("iiwa7", ["iiwa_link_ee"], False), ("panda_no_gripper", ["panda_virtual_ee_link"], False),
         ("allegro_hand_description_left", TIPS, True), ("trifinger_edu", TRI, True), ("iiwa7_allegro", TIPS, True),
         ("iiwa7_allegro", ["palm_link"], False)]
REDUNDANT = [("iiwa7_allegro", TIPS, False), ("2link_robot", ["endEffector"], False)]
dt = torch.float64


def state(robot, B, seed):
    q, qd, _ = O.sample_inputs(robot, B, seed=seed, dtype=dt)
    f = torch.randn(B, robot.n_dofs, generator=torch.Generator().manual_seed(seed + 1), dtype=dt)
    return q, qd, f


def refs(B, M, seed, scale=1.0):
    return scale * torch.randn(B, M, generator=torch.Generator().manual_seed(seed), dtype=dt)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def kinetic(H, qd):
    return 0.5 * torch.einsum("bi,bij,bj->b", qd, H, qd)


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_oracle_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".contact.npz"), allow_pickle=False)
    robot = O.load_robot(urdf_path(stem), dt)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=dt)
        inertia[0] = robot.inertia[0]
        robot.inertia = inertia
    q, qd, f, a_ref, v_ref = (torch.tensor(g[k], dtype=dt) for k in ("q", "qd", "f", "a_ref", "v_ref"))
    links = [str(s) for s in g["links"]]
    pos, mu = bool(g["position_only"]), float(g["mu"])
    qdd, force, ok, _ = C.contact_dynamics(robot, q, qd, f, links, a_ref, True, False, pos, mu)
    qd_plus, impulse, ok2, _ = C.contact_impulse(robot, q, qd, links, v_ref, pos, mu)
    assert bool(ok.all()) and bool(ok2.all())
    pre = "" if tag == "sym" else "nonsym."
    for name, got in (("qdd", qdd), ("force", force), ("qd_plus", qd_plus), ("impulse", impulse)):
        ref = g[pre + name]
        assert_close(got.numpy(), ref, rtol=1e-3, atol=1e-3 * max(np.abs(ref).max(), 1e-6), what=pre + name)


@pytest.mark.parametrize("stem,links,pos", CASES)
def test_kkt_solve_and_gauss_principle(stem, links, pos):
    """Symmetric inertias: [H -J^T; J mu I] [qdd; lambda] = [H qdd_free; a_ref - Jdot qd], and H (qdd - qdd_free) = J^T lambda."""
    robot = O.load_robot(urdf_path(stem), dt)
    q, qd, f = state(robot, 6, 1)
    J = S.stacked_jacobian(robot, q, links, pos).detach()
    M, n = J.shape[1:]
    a_ref = refs(6, M, 2)
    H = D.mass_matrix(robot, q)
    qdd_free = O.forward_dynamics(robot, q, qd, f, True, True).detach()
    bias = S.bias_acceleration(robot, q, qd, links, pos).detach()
    for mu in (0.0, 1e-2):
        qdd, lam, ok, _ = C.contact_dynamics(robot, q, qd, f, links, a_ref, True, True, pos, mu)
        assert bool(ok.all())
        K = torch.cat([torch.cat([H, -J.transpose(1, 2)], 2), torch.cat([J, mu * torch.eye(M, dtype=dt).expand(6, M, M)], 2)], 1)
        rhs = torch.cat([torch.einsum("bij,bj->bi", H, qdd_free), a_ref - bias], 1)
        x = torch.linalg.solve(K, rhs)
        assert _rel(qdd, x[:, :n]) < 1e-10
        assert _rel(lam, x[:, n:]) < 1e-10
        assert _rel(torch.einsum("bij,bj->bi", H, qdd - qdd_free), torch.einsum("bmn,bm->bn", J, lam)) < 1e-10


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem,links,pos", CASES)
def test_constraint_identities(stem, links, pos, nonsym):
    robot = O.load_robot(urdf_path(stem), dt)
    if nonsym:
        robot = D.perturbed(robot)
    q, qd, f = state(robot, 5, 3)
    J = S.stacked_jacobian(robot, q, links, pos).detach()
    bias = S.bias_acceleration(robot, q, qd, links, pos).detach()
    M = J.shape[1]
    a_ref, v_ref = refs(5, M, 4), refs(5, M, 5, 0.1)
    for mu in (0.0, 0.05):
        qdd, lam, ok, _ = C.contact_dynamics(robot, q, qd, f, links, a_ref, True, False, pos, mu)
        assert bool(ok.all())
        Jqdd = torch.einsum("bmn,bn->bm", J, qdd)       # relative to the terms that cancel: light fingers reach 1e4 m/s^2
        scale = max(float(Jqdd.abs().max()), float(bias.abs().max()), 1.0)
        assert float((Jqdd + bias - (a_ref - mu * lam)).abs().max()) < 1e-10 * scale
        ft = f + torch.einsum("bmn,bm->bn", J, lam)
        assert _rel(O.forward_dynamics(robot, q, qd, ft, True, False), qdd) < 1e-10
        qp, imp, ok, _ = C.contact_impulse(robot, q, qd, links, v_ref, pos, mu)
        assert bool(ok.all())
        assert _rel(torch.einsum("bmn,bn->bm", J, qp), v_ref - mu * imp) < 1e-10


@pytest.mark.parametrize("stem,links,pos", CASES)
def test_impulse_kinetic_energy(stem, links, pos):
    """Inelastic: the kinetic energy does not increase; elastic (v_ref = -J qd, mu = 0): it is unchanged."""
    robot = O.load_robot(urdf_path(stem), dt)
    q, qd, _ = state(robot, 6, 6)
    H = D.mass_matrix(robot, q)
    J = S.stacked_jacobian(robot, q, links, pos).detach()
    T0 = kinetic(H, qd)
    qp, _, ok, _ = C.contact_impulse(robot, q, qd, links, None, pos, 0.0)
    assert bool(ok.all())
    assert bool((kinetic(H, qp) <= T0 * (1 + 1e-12)).all())
    assert float((T0 - kinetic(H, qp)).min()) > 0 or float(J.abs().max()) == 0
    qp, _, ok, _ = C.contact_impulse(robot, q, qd, links, -torch.einsum("bmn,bn->bm", J, qd), pos, 0.0)
    assert bool(ok.all())
    assert float(((kinetic(H, qp) - T0).abs() / T0).max()) < 1e-10


@pytest.mark.parametrize("stem,links,pos", REDUNDANT)
def test_redundant_sets_need_regularisation(stem, links, pos):
    robot = O.load_robot(urdf_path(stem), dt)
    q, qd, f = state(robot, 6, 7)
    qdd, lam, ok, piv = C.contact_dynamics(robot, q, qd, f, links, None, True, False, pos, 0.0)
    assert not bool(ok.any()) and bool(torch.isnan(qdd).all()) and bool(torch.isnan(lam).all())
    assert float(piv.max()) < C.PIVOT_MIN
    qp, imp, ok, _ = C.contact_impulse(robot, q, qd, links, None, pos, 0.0)
    assert not bool(ok.any()) and bool(torch.isnan(qp).all())
    J = S.stacked_jacobian(robot, q, links, pos).detach()
    A = J @ S.force_response(robot, q) @ J.transpose(1, 2)
    mu = 1e-3 * torch.diagonal(A, dim1=1, dim2=2).amax(1)
    qdd, lam, ok, piv = C.contact_dynamics(robot, q, qd, f, links, None, True, False, pos, mu)
    assert bool(ok.all()) and bool(torch.isfinite(qdd).all()) and bool(torch.isfinite(lam).all())
    qp, imp, ok, _ = C.contact_impulse(robot, q, qd, links, None, pos, mu)
    assert bool(ok.all()) and bool(torch.isfinite(qp).all())


def test_solve_pivots_ties_and_unusable_diagonals():
    """The equilibrated elimination on hand-made systems: a permutation that needs pivoting, a tie, a zero diagonal."""
    A = torch.tensor([[[1e-8, 1.0], [1.0, 1.0]], [[1.0, 1.0], [1.0, 1.0]], [[0.0, 1.0], [1.0, 1.0]],
                      [[4.0, 0.0], [0.0, 1e-12]]], dtype=dt)
    A[0, 0, 0] = 1e-8
    b = torch.tensor([[1.0, 2.0], [1.0, 1.0], [1.0, 1.0], [1.0, 1.0]], dtype=dt)
    x, ok, piv = C.equilibrated_solve(A, b)
    assert ok.tolist() == [True, False, False, True]
    assert _rel(x[0], torch.linalg.solve(A[0], b[0])) < 1e-12
    assert _rel(x[3], torch.tensor([0.25, 1e12], dtype=dt)) < 1e-12       # equilibration: 1e-12 is a unit pivot
    assert float(piv[2]) == 0.0 and float(piv[1]) < 1e-15
    assert bool(torch.isnan(x[1]).all()) and bool(torch.isnan(x[2]).all())
