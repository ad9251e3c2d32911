#!/usr/bin/env python
"""Contact dynamics of 65 536 rows: the one-launch kernel (compute_contact_dynamics) against the four-step composition of
existing calls it replaces -- operational-space dynamics (J G J^T and J qdd_free + Jdot qd), multi-link FK + Jacobian (J),
a batched torch.linalg.solve of (J G J^T + mu I) lambda = a_ref - J qdd_free - Jdot qd, and forward dynamics at f + J^T lambda.

    python scripts/bench_contact_dynamics.py [--batch 65536] [--iters 20]

Prints one JSON line per case with both times (CUDA-event medians after warm-up), the largest relative difference of qdd
and of lambda between the two paths (over the rows both solve whose equilibrated system has a condition number
below 1e3), the kernel's algorithmic HBM bytes (q, qd, f, a_ref in;
qdd, force, solved out) and an operation count, the achieved rates and the GPU's name and power limit.  The operation count
is bench_operational_space.py's estimate plus one right-hand-side sweep (70 flops per link), M^3 / 1.5 for the elimination
and 2 M n_u each for J^T lambda and the right-hand side."""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))
from differentiable_robot_model_b200 import DifferentiableRobotModel  # noqa: E402
from differentiable_robot_model_b200.robot_model import robot_description_folder  # noqa: E402
import bench_operational_space as OSB  # noqa: E402

TIPS = OSB.TIPS
TRI = ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"]
# (name, URDF, links, position_only, regularization)
CASES = [
    ("iiwa7", "kuka_iiwa/urdf/iiwa7.urdf", ["iiwa_link_ee"], False, 0.0),
    ("panda_no_gripper", "panda_description/urdf/panda_no_gripper.urdf", ["panda_virtual_ee_link"], False, 0.0),
    ("trifinger_edu", "trifinger_edu_description/trifinger_edu.urdf", TRI, True, 0.0),
    ("allegro", "allegro/urdf/allegro_hand_description_left.urdf", TIPS, True, 0.0),
    ("iiwa7_allegro", "kuka_iiwa/urdf/iiwa7_allegro.urdf", TIPS, False, 50.0),
]


def composition(m, q, qd, f, links, position_only, a_ref, mu):
    """(qdd, lambda) from existing calls."""
    with torch.no_grad():
        osd = m.compute_operational_space_dynamics(q, qd, f, links, position_only=position_only)
        fk = m.compute_fk_and_jacobian_multi(q, links)
        J = torch.cat([fk[nm][2] if position_only else torch.cat([fk[nm][2], fk[nm][3]], dim=1) for nm in links], dim=1)
        M = J.shape[1]
        A = osd.inv_inertia + mu * torch.eye(M, device=q.device)
        lam = torch.linalg.solve(A, (a_ref - osd.acceleration).unsqueeze(2))
        qdd = m.compute_forward_dynamics(q, qd, f + torch.bmm(J.transpose(1, 2), lam).squeeze(2))
        return qdd, lam.squeeze(2)


def counts(m, links, position_only):
    """(HBM bytes, flops) per row."""
    n = m._n_dofs
    M = (3 if position_only else 6) * len(links)
    _, osd_flops = OSB.counts(m, links, position_only)
    n_links = len(m._bodies)
    n_u = n      # upper bound for the two small products
    return 4 * (3 * n + M + n + M) + 1, osd_flops + 70 * n_links + (2 * M ** 3) // 3 + 4 * M * n_u


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_contact_dynamics.py measures on a CUDA device; none is present")
    card = OSB.gpu_info()
    for stem, rel, links, position_only, mu in CASES:
        m = DifferentiableRobotModel(os.path.join(robot_description_folder, rel), stem, device="cuda:0")
        n, B = m._n_dofs, args.batch
        M = (3 if position_only else 6) * len(links)
        gen = torch.Generator(device="cuda:0").manual_seed(0)
        q, qd, f = (torch.randn(B, n, device="cuda:0", generator=gen) * s for s in (1.0, 0.5, 1.0))
        a_ref = torch.randn(B, M, device="cuda:0", generator=gen)
        kernel = lambda: m.compute_contact_dynamics(q, qd, f, links, a_ref, position_only=position_only,  # noqa: E731
                                                    regularization=mu)
        base = lambda: composition(m, q, qd, f, links, position_only, a_ref, mu)  # noqa: E731
        t_k = OSB.timed(kernel, args.iters)
        t_b = OSB.timed(base, args.iters)
        got, want = kernel(), base()
        with torch.no_grad():         # rows whose equilibrated system is well conditioned (both paths round in fp32)
            A = m.compute_operational_space_dynamics(q, qd, f, links, position_only=position_only).inv_inertia.double()
            A = A + mu * torch.eye(M, device=A.device, dtype=A.dtype)
            sc = torch.diagonal(A, dim1=1, dim2=2).abs().rsqrt()
            well = torch.linalg.cond(sc[:, :, None] * A * sc[:, None, :]) < 1e3
        rows = got.solved & torch.isfinite(want[0]).all(1) & well
        d_qdd = float((got.qdd[rows] - want[0][rows]).abs().max() / want[0][rows].abs().max())
        d_lam = float((got.force[rows] - want[1][rows]).abs().max() / want[1][rows].abs().max())
        nbytes, flops = counts(m, links, position_only)
        print(json.dumps({
            "robot": stem, "links": len(links), "position_only": position_only, "M": M, "regularization": mu, "batch": B,
            "solved_fraction": float(got.solved.float().mean()), "compared_fraction": float(rows.float().mean()),
            "kernel_ms": t_k * 1e3, "composition_ms": t_b * 1e3, "speedup": t_b / t_k,
            "bytes_per_row": nbytes, "flops_per_row_est": flops,
            "kernel_GBps": nbytes * B / t_k / 1e9, "kernel_GFLOPs_est": flops * B / t_k / 1e9,
            "max_rel_diff_qdd": d_qdd, "max_rel_diff_force": d_lam, "gpu": card,
        }), flush=True)


if __name__ == "__main__":
    main()
