#!/usr/bin/env python
"""Energy, generalized momentum and centre of mass (compute_energy_and_momentum, one launch) on 65 536 configurations of the
Kuka, the Panda, the Allegro hand and the Kuka with the Allegro hand, against what a user composes today from the engine's
other kernels: kinematic_state (poses and velocities of every link) plus torch ops for the energies, the CoM and its
velocity; the mass-matrix kernel and a bmm for the momentum; and compute_fk_and_jacobian_multi over the massive links in
groups of 8 for the CoM Jacobian.

    python scripts/bench_energy_momentum.py [--batch 65536] [--iters 50] [--repeats 5]

Prints one JSON line per robot: microseconds per call of the kernel and of the composition (CUDA events around `iters`
back-to-back calls after warm-up, median of `repeats`), the speedup, the algorithmic HBM bytes per configuration of the
kernel (q, qd in: 8 n B; the six outputs: 4 (8 + 4 n) B) and their rate, the largest per-output relative difference between
the two paths, and the GPU's name and power limit read in the same run."""
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

CASES = [
    ("iiwa7", "kuka_iiwa/urdf/iiwa7.urdf"),
    ("panda", "panda_description/urdf/panda.urdf"),
    ("allegro", "allegro/urdf/allegro_hand_description_left.urdf"),
    ("iiwa7_allegro", "kuka_iiwa/urdf/iiwa7_allegro.urdf"),
]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:     # the numbers still stand; say that the card could not be read
        return f"unknown ({exc})"


def per_call(fn, iters, repeats):
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


def composition(m, table, q, qd, links):
    """The six quantities from the engine's other kernels plus torch ops (same order as energy_momentum_raw)."""
    topo, N = m._topology, len(m._bodies)
    mass, mc, Io = table[:, 24], table[:, 21:24], table[:, 12:21].reshape(N, 3, 3)
    M = mass.sum()
    poses, _, vels = engine.kinematic_state_raw(topo, table, q, qd)
    R = poses[:, :9].reshape(N, 3, 3, -1).permute(3, 0, 1, 2)
    p = poses[:, 9:12].permute(2, 0, 1)
    w, v = vels[:, :3].permute(2, 0, 1), vels[:, 3:].permute(2, 0, 1)
    Rmc = (R @ mc.unsqueeze(2)).squeeze(-1)
    h = (mass[:, None] * p + Rmc).sum(1)
    f_lin = mass[:, None] * v - torch.cross(mc.expand_as(w), w, dim=-1)
    f_ang = (Io @ w.unsqueeze(-1)).squeeze(-1) + torch.cross(mc.expand_as(v), v, dim=-1)
    kinetic = 0.5 * ((v * f_lin).sum(-1) + (w * f_ang).sum(-1)).sum(1)
    potential = 9.81 * h[:, 2]
    com = h / M
    com_velocity = (R @ f_lin.unsqueeze(-1)).squeeze(-1).sum(1) / M
    momentum = torch.bmm(engine.mass_matrix_raw(topo, table, q), qd.unsqueeze(2)).squeeze(2)
    jcom = torch.zeros(q.shape[0], 3, q.shape[1], device=q.device)
    for g in range(0, len(links), 8):
        group = links[g:g + 8]
        _, _, jl, ja = engine.fk_jacobian_multi_raw(topo, group, table, q, want_pos=False, want_quat=False)
        for e, l in enumerate(group):
            jcom += mass[l] * jl[e] + torch.cross(ja[e], Rmc[:, l, :, None].expand_as(ja[e]), dim=1)
    return kinetic, potential, momentum, com, com_velocity, jcom / M


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_energy_momentum.py measures on a CUDA device; none is present")
    card = gpu_info()
    B = args.batch
    for stem, rel in CASES:
        m = DifferentiableRobotModel(os.path.join(robot_description_folder, rel), stem, device="cuda:0")
        n = m._n_dofs
        table = m._link_table().detach()
        links = [l for l in range(1, len(m._bodies)) if bool((table[l, 21:25] != 0).any())]
        gen = torch.Generator(device="cuda:0").manual_seed(0)
        q, qd = (torch.randn(B, n, device="cuda:0", generator=gen) * s for s in (1.0, 0.5))
        got = engine.energy_momentum_raw(m._topology, table, q, qd)
        want = composition(m, table, q, qd, links)
        diff = max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(got, want))
        t_k = per_call(lambda: engine.energy_momentum_raw(m._topology, table, q, qd), args.iters, args.repeats)
        t_c = per_call(lambda: composition(m, table, q, qd, links), args.iters, args.repeats)
        nbytes = 8 * n + 4 * (8 + 4 * n)
        print(json.dumps({
            "robot": stem, "n_dofs": n, "n_links": len(m._bodies), "batch": B, "kernel_us": t_k * 1e6,
            "composition_us": t_c * 1e6, "speedup": t_c / t_k, "bytes_per_config": nbytes, "kernel_GBps": nbytes * B / t_k / 1e9,
            "composition_launch_groups": (len(links) + 7) // 8, "max_rel_diff": diff, "gpu": card,
        }), flush=True)


if __name__ == "__main__":
    main()
