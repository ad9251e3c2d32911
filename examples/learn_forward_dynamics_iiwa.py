"""Identify link-1 mass / centre of mass / inertia of a Kuka iiwa from joint accelerations (CUDA engine).

The experiment of the reference's ``examples/learn_forward_dynamics_iiwa.py`` (``run(n_epochs, n_data, device)``, :50).
Every ``compute_forward_dynamics`` call is ONE articulated-body kernel launch and ``backward()`` its analytic adjoint
kernel; the learned ``inertia_mat`` is an unconstrained -- hence non-symmetric -- 3x3, which is why the kernels carry
general 6x6 articulated inertias.
"""
from common import fit_minibatch, nmse
from differentiable_robot_model_b200 import DifferentiableKUKAiiwa, DifferentiableRobotModel
from differentiable_robot_model_b200.data_utils import generate_sine_motion_forward_dynamics_data
from differentiable_robot_model_b200.rigid_body_params import PositiveScalar, UnconstrainedTensor


def run(n_epochs=100, n_data=10000, device="cuda"):
    truth = DifferentiableKUKAiiwa(device=device)
    student = DifferentiableRobotModel(truth.urdf_path, name="kuka_iiwa", device=device)
    student.make_link_param_learnable("iiwa_link_1", "mass", PositiveScalar())
    student.make_link_param_learnable("iiwa_link_1", "com", UnconstrainedTensor(dim1=1, dim2=3))
    student.make_link_param_learnable("iiwa_link_1", "inertia_mat", UnconstrainedTensor(dim1=3, dim2=3))
    data = generate_sine_motion_forward_dynamics_data(truth, n_data=n_data, dt=1.0 / 250.0, freq=0.1)
    variance = data.var()

    def acceleration_error(batch):
        q, qd, qdd, tau = batch
        predicted = student.compute_forward_dynamics(q=q, qd=qd, f=tau, include_gravity=True, use_damping=True)
        return nmse(predicted, qdd, variance)

    history = fit_minibatch(student.parameters(), data, acceleration_error, n_epochs)
    student.print_learnable_params()
    return history


if __name__ == "__main__":
    run()
