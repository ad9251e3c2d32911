"""GPU: examples/identify_dynamics_iiwa.py identifies the Kuka's inertial parameters and dampings in closed form from
noise-free torques of the same fp32 inverse-dynamics kernel, to a held-out torque NMSE below 1e-6."""
import os
import sys

import pytest

from conftest import REPO

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(REPO, "examples"))


def test_identify_dynamics_iiwa_reaches_a_small_held_out_error():
    import identify_dynamics_iiwa as ex
    held_out = ex.run(n_data=2048)
    print(f"held-out torque NMSE {held_out:.3e}")
    assert held_out < 1e-6
