"""CPU: pin the implicit-damping restatement (tests/implicit_damping_oracle.py) -- the definition of
drmb200_forward_dynamics_implicit_damping and of the rollouts with DRMB200_IMPLICIT_DAMPING -- against the dense form
(H + h D)^-1 (f - nle), against the one-joint contraction it must produce, against the oracle's own forward dynamics at
h = 0, and against golden vectors from the reference (tests/golden/make_golden_implicit_rollout.py)."""
import os

import numpy as np
import pytest
import torch

import implicit_damping_oracle as I
from conftest import GOLDEN_DIR, urdf_path
from oracle import drm_oracle as O

SYMMETRIC = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro", "allegro_hand_description_left"]
GOLDEN_STEMS = SYMMETRIC
PARAM_OF = {"trans": "trans", "rot_angles": "rpy", "mass": "mass", "com": "com", "inertia_mat": "inertia",
            "joint_damping": "damping"}

ONE_JOINT = """<?xml version="1.0"?>
<robot name="one_joint">
  <link name="base"/>
  <joint name="j1" type="revolute">
    <parent link="base"/><child link="l1"/>
    <origin xyz="0 0 0" rpy="0 0 0"/><axis xyz="0 0 1"/>
    <limit lower="-3" upper="3" effort="10" velocity="10"/>
    <dynamics damping="{damping}"/>
  </joint>
  <link name="l1">
    <inertial>
      <origin xyz="{cx} 0 0" rpy="0 0 0"/>
      <mass value="{mass}"/>
      <inertia ixx="0.001" ixy="0" ixz="0" iyy="0.001" iyz="0" izz="{izz}"/>
    </inertial>
  </link>
</robot>
"""


def dense_inertia(robot, q):
    """H [B, n, n] from the oracle's inverse dynamics: column j = ID(q, 0, e_j) without gravity or damping."""
    B, n = q.shape
    z = torch.zeros_like(q)
    eye = torch.eye(n, dtype=q.dtype)
    return torch.stack([O.inverse_dynamics(robot, q, z, eye[j].expand(B, n), False, False) for j in range(n)], dim=2)


@pytest.mark.parametrize("grav", [0, 1])
@pytest.mark.parametrize("stem", SYMMETRIC)
def test_pivot_form_equals_dense_solve(stem, grav):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    q, qd, qdd = O.sample_inputs(robot, 6, seed=3, dtype=torch.float64)
    f = qdd                                             # any forces
    gen = torch.Generator().manual_seed(7)
    robot.damping = robot.damping + torch.rand(robot.damping.shape, generator=gen, dtype=torch.float64)   # every joint damped
    d = I.damping_vector(robot)
    H = dense_inertia(robot, q)
    nle = O.inverse_dynamics(robot, q, qd, torch.zeros_like(q), bool(grav), True)
    for h in (1e-4, 1e-3, 1e-2):
        want = torch.linalg.solve(H + h * torch.diag_embed(d.expand_as(q)), (f - nle).unsqueeze(2)).squeeze(2)
        got = I.forward_dynamics(robot, q, qd, f, bool(grav), True, h)
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= 1e-10 * max(scale, 1.0), (h, float((got - want).abs().max()), scale)


def test_one_joint_velocity_contracts_by_inertia_over_inertia_plus_h_d(tmp_path):
    mass, cx, izz, damping = 0.3, 0.05, 0.002, 4.0
    path = tmp_path / "one_joint.urdf"
    path.write_text(ONE_JOINT.format(mass=mass, cx=cx, izz=izz, damping=damping))
    robot = O.load_robot(str(path), torch.float64)
    c = robot.com[1]                                    # the parameters as loaded (the URDF's values rounded to fp32)
    inertia = float(robot.inertia[1][2, 2] + robot.mass[1] * (c[0] * c[0] + c[1] * c[1]))   # about the joint axis
    damping = float(robot.damping[1])
    for h in (1e-4, 1e-3, 1e-1):                        # h d / I = 0.15 .. 145: explicit Euler diverges above 2
        qd = torch.tensor([[1.0], [-0.5]], dtype=torch.float64)
        q = torch.zeros_like(qd)
        ratio = inertia / (inertia + h * damping)
        for _ in range(20):
            qdd = I.forward_dynamics(robot, q, qd, torch.zeros_like(q), False, True, h)
            nxt = qd + h * qdd
            assert torch.allclose(nxt, ratio * qd, rtol=1e-13, atol=0.0), (h, (nxt / qd).tolist(), ratio)
            q, qd = q + h * nxt, nxt


@pytest.mark.parametrize("stem", ["2link_robot", "iiwa7", "allegro_hand_description_left"])
def test_zero_step_is_the_oracle_bit_for_bit(stem):
    for dtype in (torch.float32, torch.float64):
        robot = O.load_robot(urdf_path(stem), dtype)
        q, qd, qdd = O.sample_inputs(robot, 5, seed=1, dtype=dtype)
        for grav in (False, True):
            for damp in (False, True):
                want = O.forward_dynamics(robot, q, qd, qdd, grav, damp)
                got = I.forward_dynamics(robot, q, qd, qdd, grav, damp, 0.0)
                assert torch.equal(got, want)


def load(stem):
    return np.load(os.path.join(GOLDEN_DIR, stem + ".implicit_rollout.npz"), allow_pickle=False)


def tags(g):
    return sorted({k.split(".")[0] for k in g.files if k.startswith("g")} - {"G_q", "G_qd", "G_qdd"})


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("stem", GOLDEN_STEMS)
def test_rollout_restatement_matches_reference(stem, dtype):
    g = load(stem)
    robot = O.load_robot(urdf_path(stem), dtype)
    q0, qd0, f = (torch.tensor(g[k], dtype=dtype) for k in ("q0", "qd0", "f"))
    assert tags(g) == ["g0d1", "g1d1"]
    for tag in tags(g):
        traj = I.forward_dynamics_rollout(robot, q0, qd0, f, float(g["dt"]), tag == "g1d1")
        for name, got in zip(("q", "qd", "qdd"), traj):
            want = g[f"{tag}.{name}"]
            assert np.all(np.isfinite(want))
            scale = np.abs(want).max(axis=2, keepdims=True)
            err = np.abs(got.numpy() - want)
            assert np.all(err <= 1e-3 * scale + 1e-6), (tag, name, float((err / (scale + 1e-6)).max()))


# Family-relative bounds on the gradients: the goldens are the reference's fp32 autograd through a dense solve per step,
# whose own error reaches 3.4e-3 of the q0 family on the stiff hand-on-arm (iiwa7_allegro) and stays below 3.3e-4 elsewhere.
GRAD_TOL = {"iiwa7_allegro": 5e-3}


def family_close(got, want, fam, tol, what):
    err = float(np.abs(np.asarray(got, dtype=np.float64) - want).max())
    assert err <= tol * max(fam, 1e-12), f"{what}: |err| {err:.3e} > {tol} x family scale {fam:.3e}"


@pytest.mark.parametrize("stem", GOLDEN_STEMS)
def test_rollout_restatement_gradients_match_reference_autograd(stem):
    g = load(stem)
    dt = torch.float64
    robot = O.load_robot(urdf_path(stem), dt)
    names = ("trans", "rpy", "mass", "com", "inertia", "damping")
    for tag in tags(g):
        for name in names:
            setattr(robot, name, getattr(robot, name).detach().clone().requires_grad_(True))
        q0, qd0, f = (torch.tensor(g[k], dtype=dt).requires_grad_(True) for k in ("q0", "qd0", "f"))
        traj = I.forward_dynamics_rollout(robot, q0, qd0, f, float(g["dt"]), tag == "g1d1")
        loss = sum((torch.tensor(g[f"G_{k}"], dtype=dt) * v).sum() for k, v in zip(("q", "qd", "qdd"), traj))
        params = [getattr(robot, name) for name in names]
        grads = torch.autograd.grad(loss, [q0, qd0, f] + params, allow_unused=True)
        by_name = dict(zip(names, grads[3:]))
        tol = GRAD_TOL.get(stem, 5e-4)
        for t, key in zip(grads[:3], ("q0", "qd0", "f")):
            ref = g[f"{tag}.grad.{key}"]
            family_close(t.numpy(), ref, np.abs(ref).max(), tol, f"{tag}.{key}")
        prefix = f"{tag}.grad."
        checked = set()
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in ("q0", "qd0", "f"):
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
