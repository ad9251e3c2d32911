"""CPU: pin the implicit-gains restatement (tests/implicit_gains_oracle.py) -- the definition of drmb200_pd_rollout with
DRMB200_IMPLICIT_GAINS -- against the dense form (H + h D_impl + diag(h kd + h^2 kp))^-1 (u - nle), against the stability
of the one-joint step maps, against pd_rollout_oracle at kp = kd = 0, and against golden vectors from the reference
(tests/golden/make_golden_implicit_gains_rollout.py)."""
import os

import numpy as np
import pytest
import torch

import implicit_damping_oracle as I
import implicit_gains_oracle as IG
import pd_rollout_oracle as PD
from conftest import GOLDEN_DIR, urdf_path
from oracle import drm_oracle as O

SYMMETRIC = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro", "allegro_hand_description_left"]
PARAM_OF = {"trans": "trans", "rot_angles": "rpy", "mass": "mass", "com": "com", "inertia_mat": "inertia",
            "joint_damping": "damping"}


def dense_inertia(robot, q):
    """H [B, n, n] from the oracle's inverse dynamics: column j = ID(q, 0, e_j) without gravity or damping."""
    B, n = q.shape
    z = torch.zeros_like(q)
    eye = torch.eye(n, dtype=q.dtype)
    return torch.stack([O.inverse_dynamics(robot, q, z, eye[j].expand(B, n), False, False) for j in range(n)], dim=2)


@pytest.mark.parametrize("implicit_damping", [False, True])
@pytest.mark.parametrize("grav", [0, 1])
@pytest.mark.parametrize("stem", SYMMETRIC)
def test_pivot_form_equals_dense_solve(stem, grav, implicit_damping):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    q, qd, qdd = O.sample_inputs(robot, 6, seed=3, dtype=torch.float64)
    u = qdd                                             # any forces
    gen = torch.Generator().manual_seed(7)
    robot.damping = robot.damping + torch.rand(robot.damping.shape, generator=gen, dtype=torch.float64)
    d = I.damping_vector(robot)
    H = dense_inertia(robot, q)
    nle = O.inverse_dynamics(robot, q, qd, torch.zeros_like(q), bool(grav), True)
    for h in (1e-4, 1e-3, 1e-2):
        kp = 10.0 ** torch.empty_like(q).uniform_(0, 5, generator=gen)
        kd = 10.0 ** torch.empty_like(q).uniform_(-2, 2, generator=gen)
        c = h * (kd + h * kp)
        A = H + torch.diag_embed(c) + (h * torch.diag_embed(d.expand_as(q)) if implicit_damping else 0.0)
        want = torch.linalg.solve(A, (u - nle).unsqueeze(2)).squeeze(2)
        got = IG.forward_dynamics(robot, q, qd, u, bool(grav), True, h if implicit_damping else 0.0, c)
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= 1e-10 * max(scale, 1.0), (h, float((got - want).abs().max()), scale)


def test_without_addend_is_the_implicit_damping_oracle_bit_for_bit():
    robot = O.load_robot(urdf_path("iiwa7"), torch.float64)
    q, qd, f = O.sample_inputs(robot, 5, seed=2, dtype=torch.float64)
    for h in (0.0, 1e-3):
        assert torch.equal(IG.forward_dynamics(robot, q, qd, f, True, True, h), I.forward_dynamics(robot, q, qd, f, True, True, h))
        assert torch.equal(IG.forward_dynamics(robot, q, qd, f, True, True, h, torch.zeros_like(q)),
                           I.forward_dynamics(robot, q, qd, f, True, True, h))


def spectral_radius(m):
    return torch.linalg.eigvals(m).abs().max(-1).values


def test_one_joint_step_maps_stability_grid():
    inertia = 2e-3
    h = torch.tensor([1e-4, 1e-3, 1e-2], dtype=torch.float64).view(-1, 1, 1)
    kp = (10.0 ** torch.linspace(-1, 7, 33, dtype=torch.float64)).view(1, -1, 1)
    kd = (10.0 ** torch.linspace(-4, 3, 29, dtype=torch.float64)).view(1, 1, -1)
    ex, im = IG.step_maps(inertia, h, kp, kd)
    r_im, r_ex = spectral_radius(im), spectral_radius(ex)
    assert bool((r_im < 1).all()), float(r_im.max())
    a, b = (h * h * kp / inertia).expand_as(r_ex), (h * kd / inertia).expand_as(r_ex)
    unstable = (b >= 2) | (a + 2 * b >= 4)
    # away from the boundary, where the radius is 1 to rounding: explicit > 1 exactly where the Jury conditions fail
    margin = torch.minimum((b - 2).abs() / 2, (a + 2 * b - 4).abs() / 4)
    away = margin > 1e-6
    assert int(away.sum()) > 0.9 * away.numel()
    assert torch.equal((r_ex > 1)[away], unstable[away])
    # critical damping: h omega < 0.83 is the explicit limit (a + 2b = 4 with b = 2 sqrt(a))
    w = torch.tensor([800.0, 860.0], dtype=torch.float64)
    ex_c, im_c = IG.step_maps(1.0, 1e-3, w * w, 2 * w)
    assert spectral_radius(ex_c).tolist()[0] < 1 < spectral_radius(ex_c).tolist()[1]
    assert bool((spectral_radius(im_c) < 1).all())
    # the implicit map's determinant is 1 / (1 + a + b)
    det = torch.linalg.det(im)
    a, b = h * h * kp / inertia, h * kd / inertia
    assert torch.allclose(det, (1 / (1 + a + b)).expand_as(det), rtol=1e-9, atol=1e-13)


@pytest.mark.parametrize("stem", ["2link_robot", "iiwa7", "allegro_hand_description_left"])
def test_zero_gains_are_pd_rollout_oracle_bit_for_bit(stem):
    for dtype in (torch.float32, torch.float64):
        robot = O.load_robot(urdf_path(stem), dtype)
        q0, qd0, _ = O.sample_inputs(robot, 4, seed=1, dtype=dtype)
        T, n = 6, robot.n_dofs
        gen = torch.Generator().manual_seed(4)
        q_ref = q0 + 0.1 * torch.randn(T, *q0.shape, generator=gen, dtype=dtype)
        qd_ref = torch.randn(T, *q0.shape, generator=gen, dtype=dtype)
        f = 0.5 * torch.randn(T, *q0.shape, generator=gen, dtype=dtype)
        kp = kd = torch.zeros(n, dtype=dtype)
        lim = torch.full((n,), 0.3, dtype=dtype)
        # the Allegro fingers' explicit damping diverges within these steps (qdd non-finite: 0 * qdd is not 0)
        damping = (False,) if stem.startswith("allegro") else (False, True)
        for grav in (False, True):
            for damp in damping:
                for limit in (None, lim):
                    want = PD.pd_rollout(robot, q0, qd0, q_ref, kp, kd, 1e-3, qd_ref, f, limit, grav, damp)
                    got = IG.pd_rollout(robot, q0, qd0, q_ref, kp, kd, 1e-3, qd_ref, f, limit, grav, damp)
                    for x, y in zip(got, want):
                        assert torch.equal(x, y)


def test_saturation_follows_the_predicted_command():
    q = torch.zeros(1, 3, dtype=torch.float64)
    qd = torch.tensor([[1.0, 0.0, 0.0]], dtype=torch.float64)
    q_ref = torch.tensor([[0.0, 1.0, float("nan")]], dtype=torch.float64)
    lim = torch.tensor([5.0, 5.0, 5.0], dtype=torch.float64)
    kp, kd = torch.tensor([1000.0, 4.0, 1.0], dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    u, c, sat = IG.gains_step(q, qd, q_ref, kp, kd, 0.01, effort_limit=lim)
    # joint 0: u-hat = 1000 * -(0 + 0.01) = -10 saturates; joint 1: 4 stays; joint 2: NaN counts as saturated
    assert sat.tolist() == [[True, False, True]]
    assert u[0, 0] == -5.0 and u[0, 1] == 4.0 and bool(torch.isnan(u[0, 2]))
    assert c[0, 0] == 0.0 and c[0, 2] == 0.0 and c[0, 1] == 0.01 * (0.0 + 0.01 * 4.0)


def load(stem):
    return np.load(os.path.join(GOLDEN_DIR, stem + ".implicit_gains_rollout.npz"), allow_pickle=False)


def tags(g):
    """g{gravity}d1{e|i}: explicit or implicit damping (the Allegro models have the implicit tags only)."""
    return sorted({k.split(".")[0] for k in g.files if k.startswith(("g0", "g1"))})

INPUTS = ("q0", "qd0", "q_ref", "qd_ref", "f", "kp", "kd")


def golden_rollout(robot, g, tag, dtype, requires_grad=False):
    ins = [torch.tensor(g[k], dtype=dtype).requires_grad_(requires_grad) for k in INPUTS]
    q0, qd0, q_ref, qd_ref, f, kp, kd = ins
    traj = IG.pd_rollout(robot, q0, qd0, q_ref, kp, kd, float(g["dt"]), qd_ref, f, None, tag.startswith("g1"), True,
                         tag.endswith("i"))
    return ins, traj


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("stem", SYMMETRIC)
def test_rollout_restatement_matches_reference(stem, dtype):
    g = load(stem)
    robot = O.load_robot(urdf_path(stem), dtype)
    assert tags(g) == (["g0d1i", "g1d1i"] if "allegro" in stem else ["g0d1e", "g0d1i", "g1d1e", "g1d1i"])
    for tag in tags(g):
        _, traj = golden_rollout(robot, g, tag, dtype)
        for name, got in zip(("q", "qd", "qdd", "tau"), traj):
            want = g[f"{tag}.{name}"]
            assert np.all(np.isfinite(want))
            scale = np.abs(want).max(axis=2, keepdims=True)
            err = np.abs(got.numpy() - want)
            assert np.all(err <= 1e-3 * scale + 1e-6), (tag, name, float((err / (scale + 1e-6)).max()))


# Family-relative bounds on the gradients: the goldens are the reference's fp32 autograd through a dense solve per step.
GRAD_TOL = {"iiwa7_allegro": 5e-3}


def family_close(got, want, fam, tol, what):
    err = float(np.abs(np.asarray(got, dtype=np.float64) - want).max())
    assert err <= tol * max(fam, 1e-12), f"{what}: |err| {err:.3e} > {tol} x family scale {fam:.3e}"


@pytest.mark.parametrize("stem", SYMMETRIC)
def test_rollout_restatement_gradients_match_reference_autograd(stem):
    g = load(stem)
    dt = torch.float64
    robot = O.load_robot(urdf_path(stem), dt)
    names = ("trans", "rpy", "mass", "com", "inertia", "damping")
    for tag in tags(g):
        for name in names:
            setattr(robot, name, getattr(robot, name).detach().clone().requires_grad_(True))
        ins, traj = golden_rollout(robot, g, tag, dt, requires_grad=True)
        loss = sum((torch.tensor(g[f"G_{k}"], dtype=dt) * v).sum() for k, v in zip(("q", "qd", "qdd", "tau"), traj))
        params = [getattr(robot, name) for name in names]
        grads = torch.autograd.grad(loss, ins + params, allow_unused=True)
        by_name = dict(zip(names, grads[len(ins):]))
        tol = GRAD_TOL.get(stem, 5e-4)
        for t, key in zip(grads[:len(ins)], INPUTS):
            ref = g[f"{tag}.grad.{key}"]
            family_close(t.numpy(), ref, np.abs(ref).max(), tol, f"{tag}.{key}")
        prefix = f"{tag}.grad."
        checked = set()
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in INPUTS:
                continue
            pname, idx = key[len(prefix):].rsplit(".", 1)
            mine = by_name[PARAM_OF[pname]]
            mine = torch.zeros_like(getattr(robot, PARAM_OF[pname])) if mine is None else mine
            ref = g[key]
            fam = max(np.abs(g[k]).max() for k in g.files if k.startswith(prefix + pname + "."))
            mine = mine[int(idx)].reshape(ref.shape).numpy()
            if pname == "inertia_mat":
                # the goldens differentiate H and nle (RNEA), this the articulated-body arithmetic: equal for symmetric
                # inertias, so only the symmetric part of the inertia gradient is defined by both
                mine, ref = mine + mine.T, ref + ref.T
            family_close(mine, ref, 2 * fam if pname == "inertia_mat" else fam, tol, key)
            checked.add(pname)
        assert "joint_damping" in checked
