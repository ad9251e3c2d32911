"""Recover the joint origin (trans, rot_angles) of Kuka iiwa link 1 from end-effector positions (CUDA engine).

The experiment of the reference's ``examples/learn_kinematics_of_iiwa.py`` (``run(n_epochs, n_data, device)``, :26):
one FK kernel launch forward, the analytic FK adjoint kernel backward.
"""
import torch

from common import fit_full_batch
from differentiable_robot_model_b200 import DifferentiableKUKAiiwa, DifferentiableRobotModel
from differentiable_robot_model_b200.data_utils import generate_random_forward_kinematics_data
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor

EE = "iiwa_link_ee"


def run(n_epochs=3000, n_data=100, device="cuda"):
    truth = DifferentiableKUKAiiwa(device=device)
    student = DifferentiableRobotModel(truth.urdf_path, "kuka_iiwa", device=device)
    for parameter in ("trans", "rot_angles"):
        student.make_link_param_learnable("iiwa_link_1", parameter, UnconstrainedTensor(dim1=1, dim2=3))
    samples = generate_random_forward_kinematics_data(truth, n_data=n_data, ee_name=EE)

    def position_error():
        predicted, _ = student.compute_forward_kinematics(q=samples["q"], link_name=EE)
        return torch.nn.functional.mse_loss(predicted, samples["ee_pos"])

    history = fit_full_batch(student.parameters(), position_error, n_epochs)
    print("gt trans:", truth._bodies[1].trans())
    student.print_learnable_params()
    return history


if __name__ == "__main__":
    run()
