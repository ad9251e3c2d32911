"""Recover both joint origins of the planar 2-link toy robot from end-effector positions, freezing one of them for a
while on the way (CUDA engine).

The experiment of the reference's ``examples/learn_kinematics_of_toy.py`` (``run(n_epochs, n_data, device)``, :27),
including its freeze at iteration 10 / unfreeze at iteration 100.
"""
import torch

from common import fit_full_batch
from differentiable_robot_model_b200 import DifferentiableRobotModel, DifferentiableTwoLinkRobot
from differentiable_robot_model_b200.data_utils import generate_random_forward_kinematics_data
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor

EE = "endEffector"


def run(n_epochs=3000, n_data=100, device="cuda"):
    truth = DifferentiableTwoLinkRobot(device=device)
    student = DifferentiableRobotModel(truth.urdf_path, name="2link", device=device)
    for link in ("arm1", "arm2"):
        student.make_link_param_learnable(link, "trans", UnconstrainedTensor(dim1=1, dim2=3))
    samples = generate_random_forward_kinematics_data(truth, n_data=n_data, ee_name=EE)

    def position_error():
        predicted, _ = student.compute_forward_kinematics(q=samples["q"], link_name=EE)
        return torch.nn.functional.mse_loss(predicted, samples["ee_pos"])

    def schedule(i):
        if i == 10:
            student.freeze_learnable_link_param(link_name="arm1", parameter_name="trans")
        elif i == 100:
            student.unfreeze_learnable_link_param(link_name="arm1", parameter_name="trans")

    history = fit_full_batch(student.parameters(), position_error, n_epochs, every=500, before_step=schedule)
    print("ground-truth joint origins:", truth._bodies[1].trans(), truth._bodies[2].trans())
    student.print_learnable_params()
    return history


if __name__ == "__main__":
    run()
