#!/usr/bin/env python
"""The joint-torque regressor (compute_dynamics_regressor, one launch) on 65 536 configurations of the Kuka, the Panda and
the Allegro hand and on 2^18 configurations of the Kuka, and what it replaces at a small batch: one
torch.autograd.functional.jacobian of the inverse dynamics with respect to the link table per configuration.

    python scripts/bench_regressor.py [--iters 50] [--repeats 5] [--small 64]

Prints one JSON line per case: microseconds per launch (CUDA events around `iters` back-to-back launches after warm-up,
median of `repeats`), configurations per second, the algorithmic HBM bytes (q, qd, qdd in: 12 n B; Y out: 56 n L B per
configuration) per second and their fraction of the H100 SXM's 3.35 TB/s data-sheet bandwidth, and the GPU's name and
power limit read in the same run.  A last line times the per-configuration autograd Jacobian against the kernel at the same
small batch and reports the largest relative difference between the two."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from differentiable_robot_model_b200 import DifferentiableRobotModel, engine  # noqa: E402
from differentiable_robot_model_b200.robot_model import robot_description_folder  # noqa: E402

HBM_PEAK = 3.35e12
CASES = [
    ("iiwa7", "kuka_iiwa/urdf/iiwa7.urdf", 65536),
    ("panda_no_gripper", "panda_description/urdf/panda_no_gripper.urdf", 65536),
    ("allegro", "allegro/urdf/allegro_hand_description_left.urdf", 65536),
    ("iiwa7", "kuka_iiwa/urdf/iiwa7.urdf", 1 << 18),
]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:     # the numbers still stand; say that the card could not be read
        return f"unknown ({exc})"


def per_launch(fn, iters, repeats):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3 / iters)
    times.sort()
    return times[len(times) // 2]


def model(rel, stem):
    return DifferentiableRobotModel(os.path.join(robot_description_folder, rel), stem, device="cuda:0")


def state(n, B):
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    return [torch.randn(B, n, device="cuda:0", generator=gen) * s for s in (1.0, 0.5, 1.0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--small", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_regressor.py measures on a CUDA device; none is present")
    card = gpu_info()
    for stem, rel, B in CASES:
        m = model(rel, stem)
        n, L = m._n_dofs, len(m._bodies)
        q, qd, qdd = state(n, B)
        table = m._link_table().detach()
        Y = torch.empty(B, n, L, 14, device="cuda:0")
        t = per_launch(lambda: engine.dynamics_regressor_raw(m._topology, table, q, qd, qdd, 3, out=Y), args.iters, args.repeats)
        nbytes = 12 * n + 56 * n * L
        print(json.dumps({
            "robot": stem, "n_dofs": n, "n_links": L, "batch": B, "us_per_launch": t * 1e6, "configs_per_s": B / t,
            "bytes_per_config": nbytes, "GBps": nbytes * B / t / 1e9, "fraction_of_3.35TBps": nbytes * B / t / HBM_PEAK,
            "gpu": card,
        }), flush=True)

    # the alternative: autograd Jacobian of the inverse dynamics w.r.t. the table, one configuration at a time
    m = model(CASES[0][1], "iiwa7")
    n, B = m._n_dofs, args.small
    q, qd, qdd = state(n, B)
    table = m._link_table().detach()

    def autograd_rows():
        rows = []
        for b in range(B):
            J = torch.autograd.functional.jacobian(
                lambda t: engine.InverseDynamicsFunction.apply(t, q[b:b + 1], qd[b:b + 1], qdd[b:b + 1], m._topology, 3), table)
            rows.append(J[0, :, :, 12:26])
        return torch.stack(rows)

    want = autograd_rows()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        autograd_rows()
    torch.cuda.synchronize()
    t_auto = (time.perf_counter() - t0) / 3
    got = engine.dynamics_regressor_raw(m._topology, table, q, qd, qdd, 3)
    t_k = per_launch(lambda: engine.dynamics_regressor_raw(m._topology, table, q, qd, qdd, 3), args.iters, args.repeats)
    print(json.dumps({
        "robot": "iiwa7", "batch": B, "autograd_jacobian_per_row_ms_total": t_auto * 1e3, "kernel_us_per_launch": t_k * 1e6,
        "speedup": t_auto / t_k, "max_rel_diff": float((got - want).abs().max() / want.abs().max()), "gpu": card,
    }), flush=True)


if __name__ == "__main__":
    main()
