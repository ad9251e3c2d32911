#!/usr/bin/env python
"""The adjoint of the contact dynamics (compute_contact_dynamics(..., differentiable=True), csrc/contact_backward.cu) on the
cases of bench_contact_dynamics.py: the forward alone and forward + backward at --batch rows (CUDA-event medians), against
eager torch autograd of the fp32 oracle composition (tests/contact_grad_oracle.py), which runs on the CPU and is timed at
--oracle-batch rows.

    python scripts/bench_contact_backward.py [--batch 65536] [--iters 20] [--oracle-batch 256]

Prints one JSON line per case: both times, the oracle's time (and its batch), the largest gradient difference to the fp64
oracle on 32 well-conditioned rows (fp64 smallest scaled pivot >= 100x the threshold), relative to each family's largest
entry, the algorithmic HBM bytes per row of the three backward stages plus the forward, and the GPU's name and power limit."""
import argparse
import json
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))
sys.path.insert(0, os.path.join(REPO, "tests"))
from differentiable_robot_model_b200 import DifferentiableRobotModel  # noqa: E402
from differentiable_robot_model_b200.robot_model import robot_description_folder  # noqa: E402
import bench_contact_dynamics as CDB  # noqa: E402
import bench_operational_space as OSB  # noqa: E402
import contact_grad_oracle as CG  # noqa: E402
import contact_oracle as C  # noqa: E402
from oracle import drm_oracle as O  # noqa: E402


def bytes_per_row(n, M):
    """forward: q, qd, f, a_ref in, qdd, force, solved out; backward: stage 1 reads q, qd, f, lambda and both upstreams and
    writes nu, g^, tau_c and the two state copies; the forward-dynamics adjoint reads four rows and writes three; the
    kinematic stage reads q, qd, qdd, tau^, lambda, nu and adds into two rows."""
    fwd = 4 * (3 * n + M + n + M) + 1
    bwd = 4 * ((4 * n + 2 * M) + (4 * n + M) + 7 * n + (4 * n + 2 * M) + 4 * n) + 2
    return fwd, fwd + bwd


def oracle_step(path, q, qd, f, ref, g_out, g_lam, links, pos, mu, dtype):
    robot = O.load_robot(path, torch.float32).to(dtype)
    for name in ("trans", "rpy", "mass", "com", "inertia", "damping"):
        getattr(robot, name).requires_grad_(True)
    ins = [t.to(dtype).clone().requires_grad_(True) for t in (q, qd, f, ref)]
    qdd, lam = CG.dynamics(robot, *ins[:3], links, ins[3], True, False, pos, mu)
    loss = (g_out.to(dtype) * qdd).sum() + (g_lam.to(dtype) * lam).sum()
    wrt = ins + [robot.trans, robot.rpy, robot.mass, robot.com, robot.inertia, robot.damping]
    return [torch.zeros_like(w) if g is None else g for w, g in zip(wrt, torch.autograd.grad(loss, wrt, allow_unused=True))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--oracle-batch", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_contact_backward.py measures on a CUDA device; none is present")
    card = OSB.gpu_info()
    for stem, rel, links, pos, mu in CDB.CASES:
        path = os.path.join(robot_description_folder, rel)
        m = DifferentiableRobotModel(path, stem, device="cuda:0")
        n, B = m._n_dofs, args.batch
        M = (3 if pos else 6) * len(links)
        r32 = O.load_robot(path, torch.float32)
        q, qd, _ = O.sample_inputs(r32.to(torch.float64), B, seed=0, dtype=torch.float32)
        gen = torch.Generator().manual_seed(1)
        f, ref = torch.randn(B, n, generator=gen), 0.3 * torch.randn(B, M, generator=gen)
        g_out, g_lam = torch.randn(B, n, generator=gen), torch.randn(B, M, generator=gen)
        dq, dqd, df, dref, dgo, dgl = (t.to("cuda:0") for t in (q, qd, f, ref, g_out, g_lam))
        x = [t.clone().requires_grad_(True) for t in (dq, dqd, df, dref)]

        def forward():
            return m.compute_contact_dynamics(dq, dqd, df, links, dref, position_only=pos, regularization=mu)

        def forward_backward():
            out = m.compute_contact_dynamics(*x[:3], links, x[3], position_only=pos, regularization=mu, differentiable=True)
            return torch.autograd.grad([out.qdd, out.force], x, [dgo, dgl])

        t_f = OSB.timed(forward, args.iters)
        t_fb = OSB.timed(forward_backward, args.iters)

        # eager fp32 oracle autograd on the CPU, at a smaller batch
        Bo = min(args.oracle_batch, B)
        t0 = time.perf_counter()
        oracle_step(path, q[:Bo], qd[:Bo], f[:Bo], ref[:Bo], g_out[:Bo], g_lam[:Bo], links, pos, mu, torch.float32)
        t_o = time.perf_counter() - t0

        # accuracy on 32 well-conditioned rows: the kernel against the fp64 oracle, upstream zero elsewhere
        k = 256
        _, _, ok64, piv = C.contact_dynamics(r32.to(torch.float64), q[:k].double(), qd[:k].double(), f[:k].double(), links,
                                             ref[:k].double(), True, False, pos, mu)
        rows = torch.nonzero(ok64 & (piv >= 100 * C.PIVOT_MIN)).flatten()[:32]
        sel = [t[rows] for t in (q, qd, f, ref, g_out, g_lam)]
        y = [t.to("cuda:0").requires_grad_(True) for t in sel[:4]]
        out = m.compute_contact_dynamics(*y[:3], links, y[3], position_only=pos, regularization=mu, differentiable=True)
        got = torch.autograd.grad([out.qdd, out.force], y, [sel[4].to("cuda:0"), sel[5].to("cuda:0")])
        want = oracle_step(path, *sel, links, pos, mu, torch.float64)
        diff = max(float((g.double().cpu() - w).abs().max() / w.abs().max().clamp_min(1e-30)) for g, w in zip(got, want[:4]))
        fwd_bytes, total_bytes = bytes_per_row(n, M)
        print(json.dumps({
            "robot": stem, "links": len(links), "position_only": pos, "M": M, "regularization": mu, "batch": B,
            "forward_ms": t_f * 1e3, "forward_backward_ms": t_fb * 1e3, "backward_share": (t_fb - t_f) / t_fb,
            "oracle_fp32_cpu_autograd_ms": t_o * 1e3, "oracle_batch": Bo,
            "max_rel_grad_diff_fp64_inputs": diff, "compared_rows": int(len(rows)),
            "bytes_per_row_forward": fwd_bytes, "bytes_per_row_forward_backward": total_bytes,
            "forward_backward_GBps": total_bytes * B / t_fb / 1e9, "gpu": card,
        }), flush=True)


if __name__ == "__main__":
    main()
