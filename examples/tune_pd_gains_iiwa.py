"""Tune the Kuka iiwa's joint-space PD gains by gradient descent through simulated closed-loop rollouts (CUDA engine).

``DifferentiableRobotModel.compute_pd_controlled_rollout`` simulates the PD loop around a batch of smooth reference
trajectories, all steps in one launch, and is differentiable in the gains.  The cost is the mean squared tracking error
plus a small torque cost.  Each joint's gains are kp = w^2 H_kk and kd = 2 zeta w H_kk, scaled by the diagonal of the mass
matrix at the start; the optimiser tunes log(w^2) and log(2 zeta w) per joint (so they stay positive), from a soft
w = 10 rad/s, zeta = 1 on every joint.  The learning rate bounds how far they move, which keeps dt w and dt 2 zeta w
inside the region where semi-implicit Euler is stable.  The torques are clamped to a limit proportional to each
joint's inertia, so that raising the gains without bound stops paying off.

With ``--implicit-gains`` the rollout takes the PD law at the end-of-step state (stable PD,
``compute_pd_controlled_rollout(..., implicit_gains=True)``), which is stable at every dt for any non-negative gains, and
the tuning starts instead from w = 2000 rad/s, zeta = 1: dt w = 1.95, far past the explicit step's limit of about 0.83
at critical damping, where the default rollout is non-finite.  It runs without the torque limit and at a larger learning
rate: from such gains every joint would start saturated, where the limit passes no gradient, and the torque cost alone
keeps the gains from growing.

    python examples/tune_pd_gains_iiwa.py [--batch 256] [--steps 200] [--iters 100] [--implicit-gains] [--json]
"""
import argparse
import json
import math

import torch

from differentiable_robot_model_b200 import DifferentiableKUKAiiwa


def run(batch=256, steps=200, iters=100, dt=2.0 ** -10, effort_weight=1e-6, lr=0.03, device="cuda:0", log=print,
        implicit_gains=False):
    torch.manual_seed(0)
    robot = DifferentiableKUKAiiwa(device=device)
    limits = robot.get_joint_limits()
    lo = torch.tensor([l["lower"] for l in limits], device=device)
    hi = torch.tensor([l["upper"] for l in limits], device=device)
    n = robot._n_dofs
    q0 = lo + (hi - lo) * (0.3 + 0.4 * torch.rand(batch, n, device=device))
    # references: q0 plus a smooth sine per joint, with their derivative
    amp = 0.2 * torch.rand(batch, n, device=device)
    freq = 2 * torch.pi * (0.5 + torch.rand(batch, n, device=device))
    s = dt * torch.arange(1, steps + 1, device=device).view(steps, 1, 1)
    q_ref = q0 + amp * torch.sin(freq * s)
    qd_ref = amp * freq * torch.cos(freq * s)
    inertia = torch.diagonal(robot.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2).mean(0)
    effort_limit = None if implicit_gains else 2000.0 * inertia
    lr = 0.1 if implicit_gains else lr
    w0 = 2000.0 if implicit_gains else 10.0                                                 # rad/s
    log_kp = torch.full((n,), math.log(w0 ** 2), device=device, requires_grad=True)
    log_kd = torch.full((n,), math.log(2 * 1.0 * w0), device=device, requires_grad=True)    # zeta = 1
    opt = torch.optim.Adam([log_kp, log_kd], lr=lr)
    hist = []
    for it in range(iters):
        opt.zero_grad()
        q, _, _, tau = robot.compute_pd_controlled_rollout(q0, torch.zeros_like(q0), q_ref, log_kp.exp() * inertia,
                                                           log_kd.exp() * inertia, dt,
                                                           qd_ref=qd_ref, effort_limit=effort_limit,
                                                           implicit_gains=implicit_gains)
        tracking = ((q - q_ref) ** 2).mean()
        cost = tracking + effort_weight * (tau ** 2).mean()
        cost.backward()
        opt.step()
        hist.append(float(cost))
        if it % max(iters // 5, 1) == 0 or it == iters - 1:
            log(f"iter {it:4d}: cost {hist[-1]:.3e}, rms tracking error {float(tracking.sqrt()):.4f} rad")
    return hist, log_kp.detach().exp() * inertia, log_kd.detach().exp() * inertia


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--implicit-gains", action="store_true",
                    help="stable PD: the law at the end-of-step state, tuned from w = 2000 rad/s")
    ap.add_argument("--json", action="store_true", help="print one JSON line with the results")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this example runs the CUDA engine and needs a GPU"
    hist, kp, kd = run(args.batch, args.steps, args.iters, implicit_gains=args.implicit_gains)
    print(f"cost {hist[0]:.3e} -> {hist[-1]:.3e}; kp {[round(v, 1) for v in kp.tolist()]}, kd {[round(v, 2) for v in kd.tolist()]}")
    if args.json:
        print(json.dumps({"first_cost": hist[0], "last_cost": hist[-1], "kp": kp.tolist(), "kd": kd.tolist()}))


if __name__ == "__main__":
    main()
