#!/usr/bin/env python
"""Multi-link inverse kinematics of 65 536 rows: the one-launch kernel (compute_inverse_kinematics_multi) against
  * the same iteration written as an eager torch loop over compute_fk_and_jacobian_multi + torch.linalg.solve + clamp, and
  * for the Allegro hand, whose fingers share no joint, one compute_inverse_kinematics call per fingertip with the joint
    columns of each finger merged (a row counts as converged when every finger's call converged).

    python scripts/bench_ik_multi.py [--batch 65536] [--iters 100] [--repeats 5]

Workloads: the four Allegro fingertips in position mode (12 error rows, 16 joints: the task-space system) and the four
fingertips of iiwa7_allegro in pose mode (24 rows, 23 joints: the joint-space system) and in position mode (12 rows: task
space).  Targets are FK of uniform random joint angles within the limits; starts are those angles + N(0, 0.3^2), clamped.
Prints one JSON line per workload with each path's time (CUDA-event median over --repeats runs after a warm-up run), its
converged fraction (every link's position error <= 1e-4 m and, in pose mode, orientation error <= 1e-3 rad), and the
GPU's name and power limit."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_ik import POS_TOL, ROT_TOL, errors, gpu_info, timed  # noqa: E402
from differentiable_robot_model_b200 import DifferentiableRobotModel  # noqa: E402
from differentiable_robot_model_b200.robot_model import robot_description_folder  # noqa: E402

TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
URDF = {"allegro_hand_description_left": "allegro/urdf/allegro_hand_description_left.urdf",
        "iiwa7_allegro": "kuka_iiwa/urdf/iiwa7_allegro.urdf"}
WORKLOADS = [("allegro_hand_description_left", "position"), ("iiwa7_allegro", "pose"), ("iiwa7_allegro", "position")]


def union_dofs(m, links):
    """The movable joints on the union of the root -> link paths, ascending."""
    t, out = m._topology, set()
    for name in links:
        i = m._name_to_idx_map[name]
        while i > 0:
            if t.axis[i] != 0:
                out.add(int(t.dof[i]))
            i = t.parent[i]
    return sorted(out)


def eager_lm(m, links, q0, tpos, tquat, lo, hi, iters):
    """The kernel's iteration as an eager torch loop: one multi-link FK + Jacobian launch and a batched solve in the
    smaller space per iteration."""
    U = torch.tensor(union_dofs(m, links), device=q0.device)
    tq = None if tquat is None else tquat / tquat.norm(dim=2, keepdim=True)

    def evaluate(q):
        out = m.compute_fk_and_jacobian_multi(q, links)
        Js, es, perr, rerr = [], [], [], []
        for l, name in enumerate(links):
            pos, quat, jl, ja = out[name]
            Js.append(torch.cat([jl, ja], 1) if tq is not None else jl)
            e, pe, re = errors(pos, quat, tpos[l], None if tq is None else tq[l])
            es.append(e); perr.append(pe); rerr.append(re)
        J, e = torch.cat(Js, 1)[:, :, U], torch.cat(es, 1)
        done = ((torch.stack(perr) <= POS_TOL) & (torch.stack(rerr) <= ROT_TOL)).all(0)
        return J, e, (e * e).sum(1), done

    q = q0.clamp(lo, hi)
    lam = torch.full((q.shape[0],), 1e-2, device=q.device)
    J, e, E, done = evaluate(q)
    M, n_u = J.shape[1], J.shape[2]
    eye = torch.eye(min(M, n_u), device=q.device)
    for _ in range(iters):
        Jt_ = J.transpose(1, 2)
        if M <= n_u:
            dq_u = (Jt_ @ torch.linalg.solve(J @ Jt_ + lam[:, None, None] * eye, e.unsqueeze(2))).squeeze(2)
        else:
            dq_u = torch.linalg.solve(Jt_ @ J + lam[:, None, None] * eye, (Jt_ @ e.unsqueeze(2))).squeeze(2)
        dq = torch.zeros_like(q)
        dq[:, U] = dq_u
        qt = (q + dq).clamp(lo, hi)
        Jt, et, Et, dt = evaluate(qt)
        acc = (Et < E) & ~done
        rej = ~acc & ~done
        q = torch.where(acc[:, None], qt, q)
        J = torch.where(acc[:, None, None], Jt, J)
        e = torch.where(acc[:, None], et, e)
        E = torch.where(acc, Et, E)
        lam = torch.where(acc, (lam / 2).clamp_min(1e-5), torch.where(rej, (4 * lam).clamp_max(1e5), lam))
        done = done | (acc & dt)
    return done


def per_finger(m, links, q0, tpos, tquat, iters):
    """One single-link solve per fingertip, joint columns merged (valid when the fingers share no joint)."""
    q, done = q0.clone(), torch.ones(q0.shape[0], dtype=torch.bool, device=q0.device)
    for l, name in enumerate(links):
        res = m.compute_inverse_kinematics(q0, name, tpos[l], None if tquat is None else tquat[l], max_iters=iters,
                                           pos_tol=POS_TOL, rot_tol=ROT_TOL)
        cols = union_dofs(m, [name])
        q[:, cols] = res.q[:, cols]
        done &= res.converged
    return done


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ik_multi.py measures on a CUDA device; none is present")
    card = gpu_info()
    dev = "cuda:0"
    for stem, mode in WORKLOADS:
        m = DifferentiableRobotModel(os.path.join(robot_description_folder, URDF[stem]), stem, device=dev)
        lo, hi = m._joint_limit_tensors()
        gen = torch.Generator(device=dev).manual_seed(0)
        goal = lo + (hi - lo) * torch.rand(args.batch, m._n_dofs, device=dev, generator=gen)
        fk = m.compute_fk_and_jacobian_multi(goal, TIPS)
        tpos = torch.stack([fk[name][0] for name in TIPS])
        tquat = torch.stack([fk[name][1] for name in TIPS]) if mode == "pose" else None
        q0 = (goal + 0.3 * torch.randn(goal.shape, device=dev, generator=gen)).clamp(lo, hi)
        t_k, res = timed(lambda: m.compute_inverse_kinematics_multi(q0, TIPS, tpos, tquat, max_iters=args.iters,
                                                                    pos_tol=POS_TOL, rot_tol=ROT_TOL), args.repeats)
        t_e, done = timed(lambda: eager_lm(m, TIPS, q0, tpos, tquat, lo, hi, args.iters), max(1, args.repeats // 2))
        n_u, M = len(union_dofs(m, TIPS)), (6 if mode == "pose" else 3) * len(TIPS)
        line = {"robot": stem, "links": len(TIPS), "mode": mode, "system": "task" if M <= n_u else "joint",
                "batch": args.batch, "max_iters": args.iters,
                "kernel_ms": t_k * 1e3, "kernel_converged": float(res.converged.float().mean()),
                "eager_lm_ms": t_e * 1e3, "eager_lm_converged": float(done.float().mean()), "speedup_vs_eager_lm": t_e / t_k}
        if stem == "allegro_hand_description_left":
            t_s, ok = timed(lambda: per_finger(m, TIPS, q0, tpos, tquat, args.iters), args.repeats)
            line.update({"per_finger_ms": t_s * 1e3, "per_finger_converged": float(ok.float().mean()),
                         "speedup_vs_per_finger": t_s / t_k})
        line["gpu"] = card
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
