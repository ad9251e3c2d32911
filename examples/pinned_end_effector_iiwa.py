"""Hold the Kuka iiwa's end-effector origin on its start position while random joint torques act (CUDA engine).

Every step, ``DifferentiableRobotModel.compute_contact_dynamics`` gives the joint accelerations with the end-effector origin
held by a bilateral position contact (one launch for the whole batch).  Semi-implicit Euler integrates them in Python; the
contact asks for the Baumgarte-stabilised constraint acceleration

    a_ref = -2 omega J qd - omega^2 (p - p0)

so that the drift the integrator introduces decays instead of accumulating.  The arm is redundant for a point (7 joints,
3 constraints), so the torques and gravity move it through the null space while the point stays put.  The same rollout
without the contact shows how far the point would have moved.

The torques are smooth random profiles scaled per joint by the diagonal of the mass matrix at the start, so that every
joint sees accelerations of a few rad/s^2 (the wrist's inertia is a thousandth of the shoulder's); the joints' damping
acts.  Semi-implicit Euler leaves a constraint error of about dt^2 |v|^2 / r per step, which the Baumgarte terms bound
by roughly that over (omega dt)^2: omega dt = 0.2 keeps the drift well below a millimetre.

    python examples/pinned_end_effector_iiwa.py [--batch 16] [--steps 1000] [--dt 1e-3] [--omega 200] [--json]
"""
import argparse
import json

import torch

from differentiable_robot_model_b200 import DifferentiableKUKAiiwa

EE = "iiwa_link_ee"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--dt", type=float, default=1e-3)
    ap.add_argument("--omega", type=float, default=200.0, help="Baumgarte stabilisation rate [1/s]")
    ap.add_argument("--accel", type=float, default=2.0, help="random torque scale [rad/s^2 times each joint's inertia]")
    ap.add_argument("--json", action="store_true", help="print one JSON line with the results")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this example runs the CUDA engine and needs a GPU"

    torch.manual_seed(0)
    robot = DifferentiableKUKAiiwa(device="cuda:0")
    limits = robot.get_joint_limits()
    lo = torch.tensor([l["lower"] for l in limits], device="cuda:0")
    hi = torch.tensor([l["upper"] for l in limits], device="cuda:0")
    B, n, dt, w = args.batch, robot._n_dofs, args.dt, args.omega
    q0 = lo + (hi - lo) * (0.3 + 0.4 * torch.rand(B, n, device="cuda:0"))       # away from the joint limits
    p0 = robot.compute_forward_kinematics(q0, EE)[0]
    # a smooth random torque profile per row: a constant plus two sines, scaled by each joint's inertia
    inertia = torch.diagonal(robot.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2)
    amp = args.accel * inertia * torch.randn(3, B, n, device="cuda:0")
    freq = 2 * torch.pi * (0.5 + 2 * torch.rand(B, n, device="cuda:0"))

    def torques(t):
        return amp[0] + amp[1] * torch.sin(freq * t) + amp[2] * torch.cos(0.7 * freq * t)

    def rollout(pinned):
        q, qd = q0.clone(), torch.zeros(B, n, device="cuda:0")
        drift = torch.zeros(B, device="cuda:0")
        motion = torch.zeros(B, device="cuda:0")
        all_solved = True
        for k in range(args.steps):
            f = torques(k * dt)
            if pinned:
                p, _, J, _ = robot.compute_fk_and_jacobian(q, EE)
                a_ref = -2 * w * torch.einsum("bmn,bn->bm", J, qd) - w * w * (p - p0)
                qdd, _, solved = robot.compute_contact_dynamics(q, qd, f, [EE], a_ref, use_damping=True,
                                                                position_only=True)
                all_solved = all_solved and bool(solved.all())
            else:
                qdd = robot.compute_forward_dynamics(q, qd, f, use_damping=True)
            qd = qd + dt * qdd
            q = q + dt * qd
            drift = torch.maximum(drift, (robot.compute_forward_kinematics(q, EE)[0] - p0).norm(dim=1))
            motion = torch.maximum(motion, (q - q0).norm(dim=1))
        return float(drift.max()), float(motion.max()), all_solved

    drift, motion, solved = rollout(True)
    free_drift, _, _ = rollout(False)
    res = {"batch": B, "steps": args.steps, "dt": dt, "omega": w, "max_drift_m": drift, "joint_motion_rad": motion,
           "free_drift_m": free_drift, "all_solved": solved}
    print(f"pinned: largest drift of the end-effector origin {drift * 1e3:.4f} mm over {args.steps * dt:.2f} s, "
          f"joints moved up to {motion:.3f} rad through the null space (every row solved: {solved})")
    print(f"free:   the same torques without the contact move the point up to {free_drift * 1e3:.1f} mm")
    if args.json:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
