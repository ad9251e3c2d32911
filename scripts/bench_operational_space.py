#!/usr/bin/env python
"""Operational-space dynamics of 65 536 rows: the one-launch kernel (compute_operational_space_dynamics) against the best
composition of existing calls -- multi-link FK + Jacobian, forward-dynamics derivatives (for dqdd_df), forward dynamics
and torch.bmm -- which gives inv_inertia, J qd and J qdd but no Jdot qd.

    python scripts/bench_operational_space.py [--batch 65536] [--iters 20]

Prints one JSON line per case with both times (CUDA-event medians after warm-up), the largest relative difference of
inv_inertia and of J qdd between the two paths, the kernel's algorithmic HBM bytes (q, qd, f in; inv_inertia, acceleration,
velocity, bias out) and an operation count, the achieved rates and the GPU's name and power limit.  The operation count is
an estimate from the kernel's loops: 60 flops per walked link, 250 per link for the articulated-body passes, 70 per link
per extra right-hand-side sweep, and 2 per multiply-add of the two small matrix products."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from differentiable_robot_model_b200 import DifferentiableRobotModel, engine  # noqa: E402
from differentiable_robot_model_b200.robot_model import robot_description_folder  # noqa: E402

TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
CASES = [
    ("iiwa7", "kuka_iiwa/urdf/iiwa7.urdf", ["iiwa_link_ee"], False),
    ("panda_no_gripper", "panda_description/urdf/panda_no_gripper.urdf", ["panda_virtual_ee_link"], False),
    ("allegro", "allegro/urdf/allegro_hand_description_left.urdf", TIPS, True),
    ("iiwa7_allegro", "kuka_iiwa/urdf/iiwa7_allegro.urdf", TIPS, False),
]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:     # the numbers still stand; say that the card could not be read
        return f"unknown ({exc})"


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    times.sort()
    return times[len(times) // 2]


def composition(m, q, qd, f, links, position_only):
    """(inv_inertia, J qdd, J qd) from existing calls."""
    with torch.no_grad():
        fk = m.compute_fk_and_jacobian_multi(q, links)
        J = torch.cat([fk[nm][2] if position_only else torch.cat([fk[nm][2], fk[nm][3]], dim=1) for nm in links], dim=1)
        G = m.compute_forward_dynamics_derivatives(q, qd, f)[2]
        qdd = m.compute_forward_dynamics(q, qd, f)
        inv = torch.bmm(torch.bmm(J, G), J.transpose(1, 2))
        return inv, torch.bmm(J, qdd.unsqueeze(2)).squeeze(2), torch.bmm(J, qd.unsqueeze(2)).squeeze(2)


def counts(m, links, position_only):
    """(HBM bytes, flops) per row, from the model's sizes."""
    n = m._n_dofs
    M = (3 if position_only else 6) * len(links)
    n_links = len(m._bodies)
    path = set()
    for nm in links:
        i = m._name_to_idx_map[nm]
        while i > 0:
            path.add(i)
            i = m._parent_idx[i]
    n_u = sum(1 for i in path if m._bodies[i].joint_idx is not None)
    sweeps = min(M, n_u)
    product = M * M * n_u if M <= n_u else n_u * M * (n_u + M)
    flops = 60 * len(path) + 250 * n_links + 70 * n_links * sweeps + 2 * product + 2 * M * n_u
    return 4 * (3 * n + M * M + 3 * M), flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_operational_space.py measures on a CUDA device; none is present")
    card = gpu_info()
    for stem, rel, links, position_only in CASES:
        m = DifferentiableRobotModel(os.path.join(robot_description_folder, rel), stem, device="cuda:0")
        n, B = m._n_dofs, args.batch
        gen = torch.Generator(device="cuda:0").manual_seed(0)
        q, qd, f = (torch.randn(B, n, device="cuda:0", generator=gen) * s for s in (1.0, 0.5, 1.0))
        kernel = lambda: m.compute_operational_space_dynamics(q, qd, f, links, position_only=position_only)  # noqa: E731
        base = lambda: composition(m, q, qd, f, links, position_only)  # noqa: E731
        t_k = timed(kernel, args.iters)
        t_b = timed(base, args.iters)
        got, want = kernel(), base()
        d_inv = float((got.inv_inertia - want[0]).abs().max() / want[0].abs().max())
        d_acc = float((got.acceleration - got.bias_acceleration - want[1]).abs().max() / want[1].abs().max())
        nbytes, flops = counts(m, links, position_only)
        print(json.dumps({
            "robot": stem, "links": len(links), "position_only": position_only, "M": got.velocity.shape[1], "batch": B,
            "kernel_ms": t_k * 1e3, "composition_ms": t_b * 1e3, "speedup": t_b / t_k,
            "bytes_per_row": nbytes, "flops_per_row_est": flops,
            "kernel_GBps": nbytes * B / t_k / 1e9, "kernel_GFLOPs_est": flops * B / t_k / 1e9,
            "max_rel_diff_inv_inertia": d_inv, "max_rel_diff_J_qdd": d_acc, "gpu": card,
        }), flush=True)


if __name__ == "__main__":
    main()
