"""CPU: pin the operational-space oracle (tests/osd_oracle.py) against central differences of the Jacobian, the affinity
identity acceleration(f + J^T F) = acceleration(f) + inv_inertia F, the textbook J H^-1 J^T (symmetric inertias only) and
the reference's own evaluation (tests/golden/make_golden_osd.py -> <robot>.osd.npz)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, assert_close, urdf_path
import derivatives_oracle as D
import osd_oracle as S
from oracle import drm_oracle as O

TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
CASES = [("iiwa7", ["iiwa_link_ee"]), ("allegro_hand_description_left", TIPS), ("iiwa7_allegro", ["link_3.0_tip", "iiwa_link_7"])]
GOLDEN = ["2link_robot", "iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro"]
dt = torch.float64


def state(robot, B, seed):
    q, qd, _ = O.sample_inputs(robot, B, seed=seed, dtype=dt)
    f = torch.randn(B, robot.n_dofs, generator=torch.Generator().manual_seed(seed + 1), dtype=dt)
    return q, qd, f


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("stem,links", CASES)
def test_bias_matches_central_differences(stem, links):
    robot = O.load_robot(urdf_path(stem), dt)
    q, qd, _ = state(robot, 5, 1)
    h = 1e-6
    Jp = S.stacked_jacobian(robot, q + h * qd, links)
    Jm = S.stacked_jacobian(robot, q - h * qd, links)
    fd = torch.einsum("bmn,bn->bm", (Jp - Jm) / (2 * h), qd)
    bias = S.bias_acceleration(robot, q, qd, links)
    assert (bias - fd).abs().max() < 1e-7 * max(1.0, float(fd.abs().max()))
    assert float(bias.abs().max()) > 1e-3


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem,links", CASES)
def test_affinity_identity(stem, links, nonsym):
    robot = O.load_robot(urdf_path(stem), dt)
    if nonsym:
        robot = D.perturbed(robot)
    q, qd, f = state(robot, 4, 2)
    inv, acc, vel, bias = S.operational_space_dynamics(robot, q, qd, f, links, True, True)
    J = S.stacked_jacobian(robot, q, links)
    F = torch.randn(acc.shape, generator=torch.Generator().manual_seed(3), dtype=dt)
    _, acc2, _, _ = S.operational_space_dynamics(robot, q, qd, f + torch.einsum("bmn,bm->bn", J, F), links, True, True)
    assert (acc2 - acc - torch.einsum("bmk,bk->bm", inv, F)).abs().max() < 1e-10 * max(1.0, float(acc.abs().max()))
    assert _rel(vel, torch.einsum("bmn,bn->bm", J, qd)) < 1e-14


@pytest.mark.parametrize("stem,links", CASES)
def test_inverse_inertia_is_j_hinv_jt_for_symmetric_inertias_only(stem, links):
    robot = O.load_robot(urdf_path(stem), dt)
    q, qd, f = state(robot, 4, 4)
    J = S.stacked_jacobian(robot, q, links)
    for r, symmetric in ((robot, True), (D.perturbed(robot), False)):
        inv = S.operational_space_dynamics(r, q, qd, f, links)[0]
        textbook = J @ torch.linalg.inv(D.mass_matrix(r, q)) @ J.transpose(1, 2)
        if symmetric:
            assert _rel(inv, textbook) < 1e-9
            assert _rel(inv, inv.transpose(1, 2)) < 1e-9
        else:
            assert _rel(inv, textbook) > 1e-4


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_oracle_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".osd.npz"), allow_pickle=False)
    robot = O.load_robot(urdf_path(stem), dt)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=dt)
        inertia[0] = robot.inertia[0]
        robot.inertia = inertia
    q, qd, f = (torch.tensor(g[k], dtype=dt) for k in ("q", "qd", "f"))
    links = [str(s) for s in g["links"]]
    got = S.operational_space_dynamics(robot, q, qd, f, links, True, False, bool(g["position_only"]))
    pre = "" if tag == "sym" else "nonsym."
    for k, name in enumerate(("inv_inertia", "acceleration", "velocity", "bias")):
        ref = g[pre + name]
        assert_close(got[k].numpy(), ref, rtol=2e-4, atol=2e-5 * max(np.abs(ref).max(), 1e-6), what=pre + name)
