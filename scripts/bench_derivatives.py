#!/usr/bin/env python
"""Dynamics Jacobians of 65 536 configurations: the one-launch kernels against n one-hot torch.autograd.grad calls
through the analytic adjoint kernels (the path a user had before compute_*_dynamics_derivatives).

    python scripts/bench_derivatives.py [--batch 65536] [--iters 20] [--robots iiwa7,panda_no_gripper]

Prints one JSON line per (robot, quantity) with configurations/s of both paths, the kernel's achieved output bandwidth
(algorithmic output bytes 8n^2 for inverse dynamics, 12n^2 for forward dynamics, over the kernel time), the largest
difference between the two paths, and the GPU's name and power limit.  Times are CUDA-event medians after warm-up."""
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

URDFS = {"iiwa7": "kuka_iiwa/urdf/iiwa7.urdf", "panda_no_gripper": "panda_description/urdf/panda_no_gripper.urdf"}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
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


def autograd_jacobians(fn, xs):
    """n one-hot reverse passes: row i of every configuration's Jacobian w.r.t. each of xs."""
    xs = [x.clone().requires_grad_(True) for x in xs]
    y = fn(*xs)
    B, n = y.shape
    outs = [torch.empty(B, n, n, device=y.device) for _ in xs]
    for i in range(n):
        g = torch.zeros_like(y)
        g[:, i] = 1
        grads = torch.autograd.grad(y, xs, g, retain_graph=i + 1 < n)
        for o, gr in zip(outs, grads):
            o[:, i, :] = gr
    return outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--robots", default="iiwa7,panda_no_gripper")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_derivatives.py measures on a CUDA device; none is present")
    card = gpu_info()
    for stem in args.robots.split(","):
        m = DifferentiableRobotModel(os.path.join(robot_description_folder, URDFS[stem]), stem, device="cuda:0")
        n, B = m._n_dofs, args.batch
        gen = torch.Generator(device="cuda:0").manual_seed(0)
        q, qd, x3 = (torch.randn(B, n, device="cuda:0", generator=gen) * s for s in (1.0, 0.5, 1.0))
        cases = [
            ("inverse_dynamics", 8, lambda: m.compute_inverse_dynamics_derivatives(q, qd, x3),
             lambda: autograd_jacobians(lambda a, b: m.compute_inverse_dynamics(a, b, x3), [q, qd])),
            ("forward_dynamics", 12, lambda: m.compute_forward_dynamics_derivatives(q, qd, x3),
             lambda: autograd_jacobians(lambda a, b, c: m.compute_forward_dynamics(a, b, c), [q, qd, x3])),
        ]
        for what, bytes_per_n2, kernel, baseline in cases:
            t_k = timed(kernel, args.iters)
            t_b = timed(baseline, max(3, args.iters // 4))
            got, want = kernel(), baseline()
            diff = max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(got, want))
            print(json.dumps({
                "robot": stem, "quantity": f"{what}_derivatives", "batch": B, "n_dofs": n,
                "kernel_configs_per_s": B / t_k, "autograd_configs_per_s": B / t_b, "speedup": t_b / t_k,
                "kernel_ms": t_k * 1e3, "autograd_ms": t_b * 1e3,
                "output_bytes_per_config": bytes_per_n2 * n * n, "kernel_output_GBps": bytes_per_n2 * n * n * B / t_k / 1e9,
                "max_rel_diff_vs_autograd": diff, "gpu": card,
            }), flush=True)


if __name__ == "__main__":
    main()
