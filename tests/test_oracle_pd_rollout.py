"""CPU: pin the PD-rollout restatement (tests/pd_rollout_oracle.py: a PD law around semi-implicit Euler over
oracle/drm_oracle.py: forward_dynamics) against golden vectors from the reference's compute_forward_dynamics in the same
loop (tests/golden/make_golden_pd_rollout.py): trajectories and applied torques in fp32 and fp64, and autograd gradients
w.r.t. q0, qd0, q_ref, qd_ref, f, kp, kd and every link parameter."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, assert_close, urdf_path
from oracle import drm_oracle as O
from pd_rollout_oracle import pd_rollout

STEMS = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro"]
PARAM_OF = {"trans": "trans", "rot_angles": "rpy", "mass": "mass", "com": "com", "inertia_mat": "inertia",
            "joint_damping": "damping"}
INPUTS = ("q0", "qd0", "q_ref", "qd_ref", "f", "kp", "kd")
KEYS = ("q", "qd", "qdd", "tau")


def load(stem):
    return np.load(os.path.join(GOLDEN_DIR, stem + ".pd_rollout.npz"), allow_pickle=False)


def flag_tags(g):
    return sorted({k.split(".")[0] for k in g.files if k.startswith("g1d")})


def run(robot, ins, g, tag):
    return pd_rollout(robot, ins["q0"], ins["qd0"], ins["q_ref"], ins["kp"], ins["kd"], float(g["dt"]), ins["qd_ref"],
                      ins["f"], torch.tensor(g["effort_limit"], dtype=ins["q0"].dtype), True, tag == "g1d1")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("stem", STEMS)
def test_pd_rollout_trajectories_match_reference(stem, dtype):
    g = load(stem)
    robot = O.load_robot(urdf_path(stem), dtype)
    ins = {k: torch.tensor(g[k], dtype=dtype) for k in INPUTS}
    assert 0.05 < float((np.abs(g[f"{flag_tags(g)[0]}.tau"]) >= g["effort_limit"]).mean()) < 0.5   # the limit binds
    for tag in flag_tags(g):
        for name, got in zip(KEYS, run(robot, ins, g, tag)):
            want = g[f"{tag}.{name}"]
            assert got.shape == want.shape
            # fp32 evaluation noise of the reference, carried through the steps: normwise per step and configuration
            scale = np.abs(want).max(axis=2, keepdims=True)
            err = np.abs(got.numpy() - want)
            assert np.all(err <= 1e-3 * scale + 1e-6), (tag, name, float((err / (scale + 1e-6)).max()))


@pytest.mark.parametrize("stem", STEMS)
def test_pd_rollout_gradients_match_reference_autograd(stem):
    g = load(stem)
    dt = torch.float64
    robot = O.load_robot(urdf_path(stem), dt)
    names = ("trans", "rpy", "mass", "com", "inertia", "damping")
    for tag in flag_tags(g):
        for name in names:
            setattr(robot, name, getattr(robot, name).detach().clone().requires_grad_(True))
        ins = {k: torch.tensor(g[k], dtype=dt, requires_grad=True) for k in INPUTS}
        traj = run(robot, ins, g, tag)
        loss = sum((torch.tensor(g[f"G_{k}"], dtype=dt) * v).sum() for k, v in zip(KEYS, traj))
        params = [getattr(robot, name) for name in names]
        grads = torch.autograd.grad(loss, [ins[k] for k in INPUTS] + params, allow_unused=True)
        by_name = dict(zip(names, grads[len(INPUTS):]))
        for t, key in zip(grads, INPUTS):
            ref = g[f"{tag}.grad.{key}"]
            assert_close(t.numpy(), ref, rtol=2e-3, atol=2e-4 * max(np.abs(ref).max(), 1e-3), what=f"{tag}.{key}")
        prefix = f"{tag}.grad."
        checked = 0
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in INPUTS:
                continue
            pname, idx = key[len(prefix):].rsplit(".", 1)
            mine = by_name[PARAM_OF[pname]]
            mine = torch.zeros_like(getattr(robot, PARAM_OF[pname])) if mine is None else mine
            ref = g[key]
            fam = max(np.abs(g[k]).max() for k in g.files if k.startswith(prefix + pname + "."))
            assert_close(mine[int(idx)].reshape(ref.shape).numpy(), ref, rtol=2e-3, atol=2e-4 * max(fam, 1e-6), what=key)
            checked += 1
        assert checked > 0


def test_pd_rollout_with_zero_gains_is_the_open_loop_rollout():
    from rollout_oracle import forward_dynamics_rollout
    robot = O.load_robot(urdf_path("iiwa7"), torch.float64)
    q0, qd0, _ = O.sample_inputs(robot, 3, seed=1, dtype=torch.float64)
    f = torch.randn(5, 3, 7, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    zero = torch.zeros(7, dtype=torch.float64)
    got = pd_rollout(robot, q0, qd0, torch.randn(5, 3, 7, dtype=torch.float64), zero, zero, 1e-3, f=f)
    want = forward_dynamics_rollout(robot, q0, qd0, f, 1e-3)
    for a, b in zip(got[:3], want):
        assert torch.equal(a, b)
    assert torch.equal(got[3], f)
    empty = pd_rollout(robot, q0, qd0, torch.zeros(0, 3, 7, dtype=torch.float64), zero, zero, 1e-3)
    assert all(t.shape == (0, 3, 7) for t in empty)
