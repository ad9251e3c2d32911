#!/usr/bin/env python
"""Batched inverse kinematics of 65 536 targets: the one-launch Levenberg-Marquardt kernel (compute_inverse_kinematics)
against the same iteration written as an eager torch loop over compute_fk_and_jacobian + torch.linalg.solve + clamp, and,
for position targets, the 200-iteration Adam loop of examples/run_kinematic_trajectory_opt.py.

    python scripts/bench_ik.py [--batch 65536] [--iters 100] [--repeats 5] [--robots iiwa7,panda_no_gripper]

Targets are FK of uniform random joint angles within the limits; starts are those angles + N(0, 0.3^2), clamped.  Prints
one JSON line per (robot, mode) with each path's time (CUDA-event median over --repeats runs after a warm-up run), its
converged fraction (position error <= 1e-4 m and, in pose mode, orientation error <= 1e-3 rad), and the GPU's name and
power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from differentiable_robot_model_b200 import DifferentiableRobotModel  # noqa: E402
from differentiable_robot_model_b200.robot_model import robot_description_folder  # noqa: E402

ROBOTS = {"iiwa7": ("kuka_iiwa/urdf/iiwa7.urdf", "iiwa_link_ee"),
          "panda_no_gripper": ("panda_description/urdf/panda_no_gripper.urdf", "panda_virtual_ee_link")}
POS_TOL, ROT_TOL = 1e-4, 1e-3


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:     # the numbers still stand; say that the card could not be read
        return f"unknown ({exc})"


def timed(fn, repeats):
    out = fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    times.sort()
    return times[len(times) // 2], out


def quat_mul(a, b):
    ax, ay, az, aw = a.unbind(1)
    bx, by, bz, bw = b.unbind(1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                        aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], dim=1)


def errors(pos, quat, tpos, tquat):
    """(e [B, M], pos_err, rot_err): the kernel's error definition in torch."""
    e = tpos - pos
    if tquat is None:
        return e, e.norm(dim=1), torch.zeros_like(e[:, 0])
    qe = quat_mul(tquat, torch.cat([-quat[:, :3], quat[:, 3:]], dim=1))
    qe = torch.where(qe[:, 3:] < 0, -qe, qe)
    s = qe[:, :3].norm(dim=1)
    g = torch.where(s > 0, 2 * torch.atan2(s, qe[:, 3]) / s.clamp_min(1e-30), torch.zeros_like(s))
    e_rot = g[:, None] * qe[:, :3]
    return torch.cat([e, e_rot], dim=1), e.norm(dim=1), e_rot.norm(dim=1)


def eager_lm(m, link, q0, tpos, tquat, lo, hi, iters):
    """The kernel's iteration as an eager torch loop: one FK + Jacobian launch and a batched solve per iteration."""
    tq = None if tquat is None else tquat / tquat.norm(dim=1, keepdim=True)
    q = q0.clamp(lo, hi)
    lam = torch.full((q.shape[0],), 1e-2, device=q.device)
    pos, quat, jl, ja = m.compute_fk_and_jacobian(q, link)
    J = torch.cat([jl, ja], 1) if tq is not None else jl
    e, perr, rerr = errors(pos, quat, tpos, tq)
    E = (e * e).sum(1)
    done = (perr <= POS_TOL) & (rerr <= ROT_TOL)
    eye = torch.eye(J.shape[1], device=q.device)
    for _ in range(iters):
        A = J @ J.transpose(1, 2) + lam[:, None, None] * eye
        y = torch.linalg.solve(A, e.unsqueeze(2))
        qt = (q + (J.transpose(1, 2) @ y).squeeze(2)).clamp(lo, hi)
        pos, quat, jl, ja = m.compute_fk_and_jacobian(qt, link)
        Jt = torch.cat([jl, ja], 1) if tq is not None else jl
        et, pt, rt = errors(pos, quat, tpos, tq)
        Et = (et * et).sum(1)
        acc = (Et < E) & ~done
        rej = ~acc & ~done
        q = torch.where(acc[:, None], qt, q)
        J = torch.where(acc[:, None, None], Jt, J)
        e = torch.where(acc[:, None], et, e)
        E, perr, rerr = torch.where(acc, Et, E), torch.where(acc, pt, perr), torch.where(acc, rt, rerr)
        lam = torch.where(acc, (lam / 2).clamp_min(1e-5), torch.where(rej, (4 * lam).clamp_max(1e5), lam))
        done = done | (acc & (perr <= POS_TOL) & (rerr <= ROT_TOL))
    return done


def adam_example(m, link, q0, tpos, lo, hi, iters=200):
    """examples/run_kinematic_trajectory_opt.py: Adam on the squared position error, clamped at the end."""
    q = q0.clone().requires_grad_(True)
    opt = torch.optim.Adam([q], lr=2e-2)
    for _ in range(iters):
        opt.zero_grad()
        pos, _ = m.compute_forward_kinematics(q, link)
        (pos - tpos).square().sum(dim=1).mean().backward()
        opt.step()
    with torch.no_grad():
        pos, _ = m.compute_forward_kinematics(q.clamp(lo, hi), link)
        return (pos - tpos).norm(dim=1) <= POS_TOL


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--robots", default="iiwa7,panda_no_gripper")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ik.py measures on a CUDA device; none is present")
    card = gpu_info()
    dev = "cuda:0"
    for stem in args.robots.split(","):
        path, link = ROBOTS[stem]
        m = DifferentiableRobotModel(os.path.join(robot_description_folder, path), stem, device=dev)
        lo, hi = m._joint_limit_tensors()
        gen = torch.Generator(device=dev).manual_seed(0)
        goal = lo + (hi - lo) * torch.rand(args.batch, m._n_dofs, device=dev, generator=gen)
        tpos, tquat = m.compute_forward_kinematics(goal, link)
        q0 = (goal + 0.3 * torch.randn(goal.shape, device=dev, generator=gen)).clamp(lo, hi)
        for mode in ("pose", "position"):
            quat = tquat if mode == "pose" else None
            t_k, res = timed(lambda: m.compute_inverse_kinematics(q0, link, tpos, quat, max_iters=args.iters,
                                                                  pos_tol=POS_TOL, rot_tol=ROT_TOL), args.repeats)
            t_e, done = timed(lambda: eager_lm(m, link, q0, tpos, quat, lo, hi, args.iters), max(1, args.repeats // 2))
            line = {"robot": stem, "mode": mode, "batch": args.batch, "max_iters": args.iters,
                    "kernel_ms": t_k * 1e3, "kernel_converged": float(res.converged.float().mean()),
                    "eager_lm_ms": t_e * 1e3, "eager_lm_converged": float(done.float().mean()),
                    "speedup_vs_eager_lm": t_e / t_k}
            if mode == "position":
                t_a, ok = timed(lambda: adam_example(m, link, q0, tpos, lo, hi), 1)
                line.update({"adam200_ms": t_a * 1e3, "adam200_converged": float(ok.float().mean()), "speedup_vs_adam200": t_a / t_k})
            line["gpu"] = card
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
