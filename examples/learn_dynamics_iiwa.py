"""Identify link-1 mass / inertia and the link-2 joint origin of a Kuka iiwa from joint torques (CUDA engine).

The experiment of the reference's ``examples/learn_dynamics_iiwa.py`` (entry point ``run(n_epochs, n_data, device)``,
:49): ground-truth torques along a sine motion, a copy of the model with three learnable link parameters, Adam on the
variance-normalised torque error.  Here every ``compute_inverse_dynamics`` is one RNEA kernel launch and
``backward()`` one launch of its analytic adjoint.
"""
from common import fit_minibatch, nmse
from differentiable_robot_model_b200 import DifferentiableKUKAiiwa, DifferentiableRobotModel
from differentiable_robot_model_b200.data_utils import generate_sine_motion_inverse_dynamics_data
from differentiable_robot_model_b200.rigid_body_params import PositiveScalar, UnconstrainedTensor

LEARNED = (("iiwa_link_1", "mass", lambda: PositiveScalar()),
           ("iiwa_link_1", "inertia_mat", lambda: UnconstrainedTensor(dim1=3, dim2=3)),
           ("iiwa_link_2", "trans", lambda: UnconstrainedTensor(dim1=1, dim2=3)))


def run(n_epochs=10, n_data=1000, device="cuda"):
    truth = DifferentiableKUKAiiwa(device=device)
    student = DifferentiableRobotModel(truth.urdf_path, name="kuka_iiwa", device=device)
    for link, parameter, make in LEARNED:
        student.make_link_param_learnable(link, parameter, make())
    data = generate_sine_motion_inverse_dynamics_data(truth, n_data=n_data, dt=1.0 / 250.0, freq=0.05)
    variance = data.var()

    def torque_error(batch):
        q, qd, qdd_des, tau = batch
        return nmse(student.compute_inverse_dynamics(q=q, qd=qd, qdd_des=qdd_des, include_gravity=True), tau, variance)

    history = fit_minibatch(student.parameters(), data, torque_error, n_epochs)
    student.print_learnable_params()
    return history


if __name__ == "__main__":
    run()
