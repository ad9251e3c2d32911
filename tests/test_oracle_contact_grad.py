"""CPU: the adjoint of the contact dynamics and contact impulses (include/drm_b200.h), proven on the fp64 oracle before the
kernels use it (tests/contact_grad_oracle.py).

1. Autograd of the differentiable oracle agrees with central finite differences, for the dynamics and for the impulse,
   with and without a reference (q, qd, f, the reference and link parameters: a mass, a joint offset, a rotation, a
   centre of mass or an inertia entry).
2. The three-stage formula -- transposed solve, forward-dynamics adjoint, kinematic term phi -- reproduces that autograd to
   fp64 rounding: symmetric and non-symmetric inertias, pose and position mode, mu = 0 and mu > 0, M <= n_u and M > n_u."""
import pytest
import torch

import contact_grad_oracle as CG
import derivatives_oracle as D
from conftest import urdf_path
from oracle import drm_oracle as O

FIELDS = ("trans", "rpy", "mass", "com", "inertia", "damping")
TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
# (robot, links, position_only, mu): M <= n_u, and M > n_u (the planar 2-link arm's end-effector pose, 6 > 2, needs mu > 0)
CASES = [("iiwa7", ["iiwa_link_ee"], False, 0.0), ("iiwa7", ["iiwa_link_ee"], False, 0.05),
         ("2link_robot", ["endEffector"], False, 0.3), ("allegro_hand_description_left", TIPS, True, 0.0),
         ("allegro_hand_description_left", TIPS[:2], False, 0.5)]


def robot_of(stem, nonsym):
    r = O.load_robot(urdf_path(stem), torch.float32)
    if nonsym:
        r = D.perturbed(r)
    r = r.to(torch.float64)
    for name in FIELDS:
        getattr(r, name).requires_grad_(True)
    return r


def inputs(robot, B, M, seed):
    q, qd, _ = O.sample_inputs(robot, B, seed=seed, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed + 1)
    f = torch.randn(B, robot.n_dofs, generator=g, dtype=torch.float64)
    ref = 0.3 * torch.randn(B, M, generator=g, dtype=torch.float64)
    g_out = torch.randn(B, robot.n_dofs, generator=g, dtype=torch.float64)
    g_lam = torch.randn(B, M, generator=g, dtype=torch.float64)
    return q, qd, f, ref, g_out, g_lam


def _m(links, pos):
    return (3 if pos else 6) * len(links)


def autograd_dynamics(robot, q, qd, f, ref, g_out, g_lam, links, pos, mu, grav=True, damp=True):
    ins = [t.detach().clone().requires_grad_(True) for t in (q, qd, f, ref)]
    qdd, lam = CG.dynamics(robot, *ins[:3], links, ins[3], grav, damp, pos, mu)
    loss = (g_out * qdd).sum() + (g_lam * lam).sum()
    wrt = ins + [getattr(robot, n) for n in FIELDS]
    return [torch.zeros_like(w) if x is None else x
            for w, x in zip(wrt, torch.autograd.grad(loss, wrt, allow_unused=True))]


def autograd_impulse(robot, q, qd, ref, g_out, g_lam, links, pos, mu):
    ins = [t.detach().clone().requires_grad_(True) for t in (q, qd, ref)]
    qdp, lam = CG.impulse(robot, ins[0], ins[1], links, ins[2], pos, mu)
    loss = (g_out * qdp).sum() + (g_lam * lam).sum()
    wrt = ins + [getattr(robot, n) for n in FIELDS]
    return [torch.zeros_like(w) if x is None else x
            for w, x in zip(wrt, torch.autograd.grad(loss, wrt, allow_unused=True))]


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_oracle_autograd_matches_finite_differences():
    robot = robot_of("iiwa7", True)
    links, pos, mu = ["iiwa_link_ee"], False, 0.0
    q, qd, f, ref, g_out, g_lam = inputs(robot, 3, _m(links, pos), 11)
    grads = autograd_dynamics(robot, q, qd, f, ref, g_out, g_lam, links, pos, mu)

    def loss():
        with torch.no_grad():
            qdd, lam = CG.dynamics(robot, q, qd, f, links, ref, True, True, pos, mu)
            return float((g_out * qdd).sum() + (g_lam * lam).sum())

    h = 1e-6
    for k, t in enumerate((q, qd, f, ref)):
        for idx in [(0, 0), (1, 2), (2, t.shape[1] - 1)]:
            old = float(t[idx])
            t[idx] = old + h; up = loss()
            t[idx] = old - h; dn = loss()
            t[idx] = old
            fd = (up - dn) / (2 * h)
            assert abs(fd - float(grads[k][idx])) <= 1e-5 * max(1.0, abs(fd)), (k, idx, fd, float(grads[k][idx]))
    for name, idx in (("mass", (7,)), ("trans", (4, 1)), ("rpy", (3, 0)), ("com", (6, 2))):
        field = getattr(robot, name)
        want = float(grads[4 + FIELDS.index(name)][idx])
        with torch.no_grad():
            old = float(field[idx])
            field[idx] = old + h; up = loss()
            field[idx] = old - h; dn = loss()
            field[idx] = old
        fd = (up - dn) / (2 * h)
        assert abs(fd - want) <= 1e-5 * max(1.0, abs(fd)), (name, idx, fd, want)


@pytest.mark.parametrize("with_ref", [True, False], ids=["ref", "noref"])
def test_impulse_oracle_autograd_matches_finite_differences(with_ref):
    robot = robot_of("allegro_hand_description_left", True)
    links, pos, mu = TIPS, True, 0.0
    q, qd, _, ref, g_out, g_lam = inputs(robot, 3, _m(links, pos), 13)
    ref = ref if with_ref else None
    grads = autograd_impulse(robot, q, qd, torch.zeros_like(g_lam) if ref is None else ref, g_out, g_lam, links, pos, mu)

    def loss():
        with torch.no_grad():
            qdp, lam = CG.impulse(robot, q, qd, links, ref, pos, mu)
            return float((g_out * qdp).sum() + (g_lam * lam).sum())

    h = 1e-6
    for k, t in enumerate((q, qd) if ref is None else (q, qd, ref)):
        for idx in [(0, 0), (1, 2), (2, t.shape[1] - 1)]:
            old = float(t[idx])
            t[idx] = old + h; up = loss()
            t[idx] = old - h; dn = loss()
            t[idx] = old
            fd = (up - dn) / (2 * h)
            assert abs(fd - float(grads[k][idx])) <= 1e-5 * max(1.0, abs(fd)), (k, idx, fd, float(grads[k][idx]))
    for name, idx in (("mass", (8,)), ("trans", (6, 1)), ("rpy", (3, 0)), ("inertia", (7, 0, 1))):
        field = getattr(robot, name)
        want = float(grads[3 + FIELDS.index(name)][idx])
        with torch.no_grad():
            old = float(field[idx])
            field[idx] = old + h; up = loss()
            field[idx] = old - h; dn = loss()
            field[idx] = old
        fd = (up - dn) / (2 * h)
        assert abs(fd - want) <= 1e-5 * max(1.0, abs(fd)), (name, idx, fd, want)


def test_formula_without_a_reference():
    """accel_ref / velocity_ref = None is the zero reference: the formula's other gradients are unchanged."""
    robot = robot_of("iiwa7", False)
    links, pos, mu = ["iiwa_link_ee"], False, 0.0
    q, qd, f, _, g_out, g_lam = inputs(robot, 4, 6, 9)
    params = [getattr(robot, n) for n in FIELDS]
    a = CG.adjoint_dynamics(robot, q, qd, f, links, g_out, g_lam, None, True, False, pos, mu, params)
    want = autograd_dynamics(robot, q, qd, f, torch.zeros_like(g_lam), g_out, g_lam, links, pos, mu, True, False)
    for got, w in zip([a[0], a[1], a[2], a[3]] + a[4], want):
        assert rel(got, w) < 1e-9
    b = CG.adjoint_impulse(robot, q, qd, links, g_out, g_lam, None, pos, mu, params)
    want = autograd_impulse(robot, q, qd, torch.zeros_like(g_lam), g_out, g_lam, links, pos, mu)
    for got, w in zip([b[0], b[1], b[2]] + b[3], want):
        assert rel(got, w) < 1e-9


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem,links,pos,mu", CASES)
def test_three_stage_formula_reproduces_autograd_dynamics(stem, links, pos, mu, nonsym):
    robot = robot_of(stem, nonsym)
    q, qd, f, ref, g_out, g_lam = inputs(robot, 4, _m(links, pos), 5)
    want = autograd_dynamics(robot, q, qd, f, ref, g_out, g_lam, links, pos, mu)
    params = [getattr(robot, n) for n in FIELDS]
    q_g, qd_g, f_g, ref_g, p_g = CG.adjoint_dynamics(robot, q, qd, f, links, g_out, g_lam, ref, True, True, pos, mu, params)
    for name, got, w in zip(("q", "qd", "f", "accel_ref") + FIELDS, [q_g, qd_g, f_g, ref_g] + p_g, want):
        assert rel(got, w) < 1e-9, f"{name}: {rel(got, w):.2e}"


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem,links,pos,mu", CASES)
def test_three_stage_formula_reproduces_autograd_impulse(stem, links, pos, mu, nonsym):
    robot = robot_of(stem, nonsym)
    q, qd, _, ref, g_out, g_lam = inputs(robot, 4, _m(links, pos), 7)
    want = autograd_impulse(robot, q, qd, ref, g_out, g_lam, links, pos, mu)
    params = [getattr(robot, n) for n in FIELDS]
    q_g, qd_g, ref_g, p_g = CG.adjoint_impulse(robot, q, qd, links, g_out, g_lam, ref, pos, mu, params)
    for name, got, w in zip(("q", "qd", "velocity_ref") + FIELDS, [q_g, qd_g, ref_g] + p_g, want):
        assert rel(got, w) < 1e-9, f"{name}: {rel(got, w):.2e}"
