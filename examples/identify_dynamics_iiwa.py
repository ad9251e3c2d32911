"""Identify every inertial parameter and damping of a Kuka iiwa from joint torques in closed form (CUDA engine).

The torques are linear in each link's inertial parameters and damping, tau = Y(q, qd, qdd) . pi
(``DifferentiableRobotModel.compute_dynamics_regressor`` / ``inertial_parameters``), so one regressor launch over a batch of
measurements and one linear least-squares solve identify them all: no learning rate, no epochs, no parametrisation
modules (compare ``learn_dynamics_iiwa.py``, which fits three link parameters by gradient descent through the RNEA).

* Training and held-out data come from ``generate_random_inverse_dynamics_data`` (uniform joint states: the sine motion
  of ``learn_dynamics_iiwa.py`` moves every joint in phase and excites too few parameter combinations).
* The nine ``I_o`` columns of each link are reduced to the symmetric form (xx, xy, xz, yy, yz, zz) by adding the
  ``I_o[a, b]`` and ``I_o[b, a]`` columns; with ``mc``, ``m`` and the damping that is 11 parameters per link.  The root's
  columns are zero and are dropped.
* Only base parameters (combinations of the link parameters) are identifiable from joint torques, so the regressor is
  rank-deficient.  The solve is the minimum-norm least-squares solution in fp64 on the GPU, through the SVD
  pseudo-inverse (``torch.linalg.lstsq`` on CUDA only has the full-rank QR driver); singular values below 1e-5 of the
  largest are treated as zero, which for the iiwa separates the 50 identifiable directions from fp32 round-off.
* The identified parameters predict the held-out torques; the score is the variance-normalised mean squared error of
  ``common.nmse``.
"""
import torch

from common import nmse
from differentiable_robot_model_b200 import DifferentiableKUKAiiwa
from differentiable_robot_model_b200.data_utils import generate_random_inverse_dynamics_data

RTOL = 1e-5


def symmetric_columns(Y):
    """[..., 14] regressor columns (I_o 9 | mc 3 | m | damping) -> [..., 11] (Ixx Ixy Ixz Iyy Iyz Izz | mc 3 | m | damping)."""
    I = Y[..., :9]
    sym = torch.stack([I[..., 0], I[..., 1] + I[..., 3], I[..., 2] + I[..., 6], I[..., 4], I[..., 5] + I[..., 7], I[..., 8]], dim=-1)
    return torch.cat([sym, Y[..., 9:]], dim=-1)


def regressor_matrix(robot, data):
    """[B * n, (n_links - 1) * 11] fp64: one row per (sample, joint), the root's columns dropped."""
    Y = robot.compute_dynamics_regressor(data["q"], data["qd"], data["qdd_des"], include_gravity=True, use_damping=True)
    A = symmetric_columns(Y)[:, :, 1:].flatten(2)
    return A.reshape(-1, A.shape[-1]).double()


def run(n_data=4096, device="cuda"):
    truth = DifferentiableKUKAiiwa(device=device)
    train = generate_random_inverse_dynamics_data(truth, n_data).data
    test = generate_random_inverse_dynamics_data(truth, n_data).data
    A = regressor_matrix(truth, train)
    pi_hat = torch.linalg.pinv(A, rtol=RTOL) @ train["tau"].double().reshape(-1)
    rank = int((torch.linalg.svdvals(A) > RTOL * torch.linalg.svdvals(A)[0]).sum())
    prediction = (regressor_matrix(truth, test) @ pi_hat).reshape(test["tau"].shape)
    held_out = float(nmse(prediction, test["tau"].double(), test["tau"].double().var(dim=0)))
    print(f"identified {A.shape[1]} parameters ({rank} identifiable combinations) from {n_data} samples; "
          f"held-out torque NMSE {held_out:.3e}")
    return held_out


if __name__ == "__main__":
    run()
    import learn_dynamics_iiwa
    history = learn_dynamics_iiwa.run()
    print(f"learn_dynamics_iiwa.py (gradient descent on three link parameters): final-epoch training NMSE {history[-1]:.3e}")
