"""GPU: batches beyond the small-batch tile switch (1 Ki rows per SM, 132 Ki on an H100) take the wide-tile kernel instantiations; every row must
be bit-identical to the same row computed in a small batch (narrow tiles), for FK+Jacobian and RNEA."""
import pytest
import torch

from conftest import urdf_path
import differentiable_robot_model_b200 as drm
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("stem,link", [("iiwa7", "iiwa_link_ee"), ("allegro_hand_description_left", "link_3.0_tip")])
def test_wide_and_narrow_tiles_agree_bitwise(stem, link):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    B = 148 * 1024 + 12345                                     # above the switch, ragged last tile
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, B, seed=1))
    big_fk = m.compute_fk_and_jacobian(q, link)
    big_tau = m.compute_inverse_dynamics(q, qd, qdd)
    idx = torch.randperm(B, device=DEV)[:4001]
    small_fk = m.compute_fk_and_jacobian(q[idx], link)
    small_tau = m.compute_inverse_dynamics(q[idx], qd[idx], qdd[idx])
    for a, b in zip(big_fk, small_fk):
        assert torch.equal(a[idx], b)
    assert torch.equal(big_tau[idx], small_tau)
    assert torch.isfinite(big_tau).all()
