"""CPU: pin the rollout restatement (tests/rollout_oracle.py: semi-implicit Euler over oracle/drm_oracle.py: forward_dynamics)
against golden vectors from the reference's compute_forward_dynamics in the same loop (tests/golden/make_golden_rollout.py):
trajectories in fp32 and fp64, and autograd gradients w.r.t. q0, qd0, f and every link parameter."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, assert_close, urdf_path
from oracle import drm_oracle as O
from rollout_oracle import forward_dynamics_rollout

STEMS = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro"]
PARAM_OF = {"trans": "trans", "rot_angles": "rpy", "mass": "mass", "com": "com", "inertia_mat": "inertia",
            "joint_damping": "damping"}


def load_rollout(stem):
    return np.load(os.path.join(GOLDEN_DIR, stem + ".rollout.npz"), allow_pickle=False)


def flag_tags(g):
    return sorted({k.split(".")[0] for k in g.files if k.startswith("g1d")})


def inputs(g, dtype):
    return tuple(torch.tensor(g[k], dtype=dtype) for k in ("q0", "qd0", "f"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("stem", STEMS)
def test_rollout_trajectories_match_reference(stem, dtype):
    g = load_rollout(stem)
    robot = O.load_robot(urdf_path(stem), dtype)
    q0, qd0, f = inputs(g, dtype)
    dt = float(g["dt"])
    for tag in flag_tags(g):
        q, qd, qdd = forward_dynamics_rollout(robot, q0, qd0, f, dt, True, tag == "g1d1")
        for name, got in (("q", q), ("qd", qd), ("qdd", qdd)):
            want = g[f"{tag}.{name}"]
            assert got.shape == want.shape
            # fp32 evaluation noise of the reference, carried through the steps: normwise per step and configuration
            scale = np.abs(want).max(axis=2, keepdims=True)
            err = np.abs(got.numpy() - want)
            assert np.all(err <= 1e-3 * scale + 1e-6), (tag, name, float((err / (scale + 1e-6)).max()))


@pytest.mark.parametrize("stem", STEMS)
def test_rollout_gradients_match_reference_autograd(stem):
    g = load_rollout(stem)
    dt = torch.float64
    robot = O.load_robot(urdf_path(stem), dt)
    names = ("trans", "rpy", "mass", "com", "inertia", "damping")
    for tag in flag_tags(g):
        for name in names:
            setattr(robot, name, getattr(robot, name).detach().clone().requires_grad_(True))
        q0, qd0, f = (t.requires_grad_(True) for t in inputs(g, dt))
        traj = forward_dynamics_rollout(robot, q0, qd0, f, float(g["dt"]), True, tag == "g1d1")
        loss = sum((torch.tensor(g[f"G_{k}"], dtype=dt) * v).sum() for k, v in zip(("q", "qd", "qdd"), traj))
        params = [getattr(robot, name) for name in names]
        grads = torch.autograd.grad(loss, [q0, qd0, f] + params, allow_unused=True)
        by_name = dict(zip(names, grads[3:]))
        for t, key in zip(grads[:3], ("q0", "qd0", "f")):
            ref = g[f"{tag}.grad.{key}"]
            assert_close(t.numpy(), ref, rtol=2e-3, atol=2e-4 * max(np.abs(ref).max(), 1e-3), what=f"{tag}.{key}")
        prefix = f"{tag}.grad."
        checked = 0
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in ("q0", "qd0", "f"):
                continue
            pname, idx = key[len(prefix):].rsplit(".", 1)
            mine = by_name[PARAM_OF[pname]]
            mine = torch.zeros_like(getattr(robot, PARAM_OF[pname])) if mine is None else mine
            ref = g[key]
            fam = max(np.abs(g[k]).max() for k in g.files if k.startswith(prefix + pname + "."))
            assert_close(mine[int(idx)].reshape(ref.shape).numpy(), ref, rtol=2e-3, atol=2e-4 * max(fam, 1e-6), what=key)
            checked += 1
        assert checked > 0


def test_rollout_of_zero_steps_is_empty():
    robot = O.load_robot(urdf_path("iiwa7"), torch.float64)
    q0, qd0, _ = O.sample_inputs(robot, 3, seed=1, dtype=torch.float64)
    q, qd, qdd = forward_dynamics_rollout(robot, q0, qd0, torch.zeros(0, 3, 7, dtype=torch.float64), 1e-3)
    assert q.shape == qd.shape == qdd.shape == (0, 3, 7)
