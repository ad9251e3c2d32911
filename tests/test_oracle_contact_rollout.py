"""CPU: pin the contact-rollout oracle (tests/contact_rollout_oracle.py) against the reference's own loop
(tests/golden/make_golden_contact_rollout.py -> <robot>.contact_rollout.npz), against the contact oracle step by step, and
on the physics the stabilisation is for: the constraint error decays at omega > 0 and the pose error is the rotation of
R R*^T."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, urdf_path
import contact_oracle as C
import contact_rollout_oracle as CR
from oracle import drm_oracle as O

TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
GOLDEN = ["2link_robot", "iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro", "trifinger_edu"]
dt = torch.float64


def _traj_error(got, want):
    scale = want.abs().amax(-1, keepdim=True).clamp_min(1e-30)
    return float(((got - want).abs() / scale).max())


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_oracle_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".contact_rollout.npz"), allow_pickle=False)
    robot = O.load_robot(urdf_path(stem), dt)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=dt)
        inertia[0] = robot.inertia[0]
        robot.inertia = inertia
    q0, qd0, f = (torch.tensor(g[k], dtype=dt) for k in ("q0", "qd0", "f"))
    links = [str(s) for s in g["links"]]
    pos, mu, step, omega = bool(g["position_only"]), float(g["mu"]), float(g["dt"]), float(g["omega"])
    out = CR.contact_rollout(robot, q0, qd0, f, links, step, omega, include_gravity=True, position_only=pos, mu=mu)
    pre = "" if tag == "sym" else "nonsym."
    # the rows whose every step is well conditioned (smallest scaled pivot >= 500x the threshold): TriFinger's stretched
    # fingers make some rows near-singular at mu = 0, where the reference's plain solve and the oracle's part ways
    rows = out[5] & (out[6] >= 500 * C.PIVOT_MIN) & torch.isfinite(torch.tensor(g[pre + "q"])).all(2).all(0)
    assert int(rows.sum()) >= 2, f"{stem}: only {int(rows.sum())} of 8 rows well conditioned"
    for i, k in enumerate(("q", "qd", "qdd", "force")):
        err = _traj_error(out[i][:, rows], torch.tensor(g[pre + k], dtype=dt)[:, rows])
        # The reference evaluates its pieces in fp32 (as in the contact goldens) and that rounding compounds over the 32
        # steps: measured on these rows, TriFinger qd 1.85e-2, Panda force 1.46e-2, the 2-link force 1.19e-2, TriFinger
        # force 1.01e-2, every other robot and output <= 5.4e-3 (the hands <= 4e-5).  The bound leaves little margin on
        # TriFinger; the kernel's own check against the fp64 oracle (test_contact_rollout_gpu.py) is much tighter.
        assert err < 2e-2, f"{stem} {tag} {k}: {err:.3e}"


def test_zero_omega_is_the_plain_contact_loop():
    robot = O.load_robot(urdf_path("iiwa7"), dt)
    q, qd, _ = O.sample_inputs(robot, 5, seed=1, dtype=dt)
    f = torch.randn(4, 5, 7, generator=torch.Generator().manual_seed(2), dtype=dt)
    out = CR.contact_rollout(robot, q, qd, f, ["iiwa_link_ee"], 1e-3)
    for t in range(4):
        qdd, force, ok, _ = C.contact_dynamics(robot, q, qd, f[t], ["iiwa_link_ee"])
        qd = qd + 1e-3 * qdd
        q = q + 1e-3 * qd
        assert torch.equal(out[0][t], q) and torch.equal(out[3][t], force) and torch.equal(out[4][t], torch.zeros_like(force))


@pytest.mark.parametrize("stem,links,pos", [("iiwa7", ["iiwa_link_ee"], False), ("trifinger_edu",
                         ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"], True)])
def test_stabilisation_pulls_the_links_back_to_their_targets(stem, links, pos):
    """Start off the targets: with omega > 0 the constraint error decays like exp(-omega t) (critically damped), and
    without stabilisation it does not."""
    robot = O.load_robot(urdf_path(stem), dt)
    q, _, _ = O.sample_inputs(robot, 3, seed=4, dtype=dt)
    qd = torch.zeros_like(q)
    tp, tq = CR.poses(robot, q, links)
    tp = tp + 2e-3
    f = torch.zeros(200, 3, robot.n_dofs, dtype=dt)

    def err(qs):
        p, quat = CR.poses(robot, qs, links)
        e = (p - tp).norm(dim=-1).amax(0)
        if not pos:
            e = e + torch.stack([CR.rotvec_error(quat[l], tq[l]).norm(dim=-1) for l in range(len(links))]).amax(0)
        return float(e.max())
    e0 = err(q)
    stab = CR.contact_rollout(robot, q, qd, f, links, 1e-3, 50.0, tp, None if pos else tq, position_only=pos)
    free = CR.contact_rollout(robot, q, qd, f, links, 1e-3, 0.0, tp, None if pos else tq, position_only=pos)
    assert err(stab[0][-1]) < 0.15 * e0            # decays (exactly exp(-10) (1 + 10) ~ 5e-4 only for a linear constraint)
    assert err(free[0][-1]) > 0.5 * e0


def test_rotation_error_is_the_rotation_of_r_times_target_transposed():
    g = torch.Generator().manual_seed(6)
    a = torch.randn(16, 4, generator=g, dtype=dt)
    b = torch.randn(16, 4, generator=g, dtype=dt)
    a, b = a / a.norm(dim=1, keepdim=True), b / b.norm(dim=1, keepdim=True)

    def mat(qu):
        x, y, z, w = qu.unbind(-1)
        return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                            2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                            2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1).view(-1, 3, 3)
    r = CR.rotvec_error(a, -3.0 * b)              # sign and scale of the target do not matter
    theta = r.norm(dim=1, keepdim=True)
    k = r / theta
    K = torch.zeros(16, 3, 3, dtype=dt)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K = K - K.transpose(1, 2)
    Rr = torch.eye(3, dtype=dt) + torch.sin(theta)[..., None] * K + (1 - torch.cos(theta))[..., None] * K @ K
    assert torch.allclose(Rr, mat(a) @ mat(b).transpose(1, 2), atol=1e-12)
    assert bool((theta <= torch.pi + 1e-12).all())
