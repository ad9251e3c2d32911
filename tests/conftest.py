import os
import sys

import numpy as np
import pytest

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

GOLDEN_DIR = os.path.join(REPO, "tests", "golden")
ROBOT_DATA = os.path.join(REPO, "differentiable_robot_model_b200", "robot_data")

# golden file stem -> URDF path relative to robot_data/
URDFS = {
    "2link_robot": "2link_robot.urdf",
    "iiwa7": "kuka_iiwa/urdf/iiwa7.urdf",
    "panda_no_gripper": "panda_description/urdf/panda_no_gripper.urdf",
    "panda": "panda_description/urdf/panda.urdf",
    "allegro_hand_description_left": "allegro/urdf/allegro_hand_description_left.urdf",
    "allegro_hand_description_left_small_damping": "allegro/urdf/allegro_hand_description_left_small_damping.urdf",
    "trifinger_edu": "trifinger_edu_description/trifinger_edu.urdf",
    "jaco_clean": "kinova_description/urdf/jaco_clean.urdf",
    "jaco": "kinova_description/urdf/jaco.urdf",
    "fetch_arm_no_gripper": "fetch_description/urdf/fetch_arm_no_gripper.urdf",
    "fetch_arm_no_gripper_small_damping": "fetch_description/urdf/fetch_arm_no_gripper_small_damping.urdf",
    "iiwa7_allegro": "kuka_iiwa/urdf/iiwa7_allegro.urdf",
}


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")
    # the CPU oracle issues thousands of tiny torch ops: on a 128-core host the default intra-op
    # thread count makes each of them slower, not faster
    import torch
    torch.set_num_threads(min(8, os.cpu_count() or 1))


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need a CUDA device and the built C-ABI library: skip (not fail) where either is missing."""
    import torch
    from differentiable_robot_model_b200 import engine
    reason = None
    if not torch.cuda.is_available():
        reason = "needs a CUDA device"
    elif not os.path.exists(engine.library_path()):
        reason = f"{engine.library_path()} has not been built"
    if reason:
        skip = pytest.mark.skip(reason=reason)
        for item in items:
            if "gpu" in item.keywords:
                item.add_marker(skip)


def urdf_path(stem):
    return os.path.join(ROBOT_DATA, URDFS[stem])


def load_golden(stem):
    return np.load(os.path.join(GOLDEN_DIR, stem + ".npz"), allow_pickle=False)


@pytest.fixture(params=sorted(URDFS))
def robot_stem(request):
    return request.param


def assert_close(actual, expected, rtol=1e-5, atol=1e-6, what=""):
    """The parity metric of SURVEY.md section 8(c): elementwise allclose(rtol, atol) AND normwise
    relative error <= 1e-5 (relaxed by the same atol floor for tiny tensors)."""
    actual = np.asarray(actual, dtype=np.float64)
    expected = np.asarray(expected, dtype=np.float64)
    assert actual.shape == expected.shape, f"{what}: shape {actual.shape} vs {expected.shape}"
    err = np.abs(actual - expected)
    bound = atol + rtol * np.abs(expected)
    worst = np.unravel_index(np.argmax(err - bound), err.shape) if err.size else ()
    assert np.all(err <= bound), (
        f"{what}: max |err|={err.max():.3e} at {worst}: got {actual[worst]:.9g}, want {expected[worst]:.9g}")
    scale = np.abs(expected).max() if expected.size else 0.0
    if scale > 0:
        assert err.max() <= max(10 * rtol * scale, atol), f"{what}: normwise error {err.max() / scale:.3e}"


def canon_quat(q):
    """Sign-canonicalise xyzw quaternions (q == -q): make the largest-magnitude component positive."""
    q = np.asarray(q, dtype=np.float64)
    idx = np.argmax(np.abs(q), axis=-1)
    sign = np.sign(np.take_along_axis(q, idx[..., None], axis=-1))
    return q * sign


LARGE_GOLDEN = {"large_iiwa7": "iiwa7", "large_panda_no_gripper": "panda_no_gripper", "large_allegro_left": "allegro_hand_description_left"}


def quat_branch_margin(R):
    """How far each rotation matrix is from a decision boundary of the reference's get_quaternion branch structure
    (spatial_vector_algebra.py:118-128): min(|trace|, gaps between the diagonal elements the else-branch compares).
    Rows with a clear margin must reproduce the reference's RAW quaternion, sign included."""
    R = np.asarray(R, dtype=np.float64)
    tr = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2]
    d = np.stack([R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]], axis=1)
    gaps = np.minimum(np.abs(d[:, 0] - d[:, 1]), np.minimum(np.abs(d[:, 1] - d[:, 2]), np.abs(d[:, 0] - d[:, 2])))
    return np.where(tr > 0, np.abs(tr), np.minimum(np.abs(tr), gaps))
