#!/usr/bin/env python
"""What implicit joint damping costs in the one-launch rollouts: the explicit-damping kernel (use_damping=True) against the
implicit one (implicit_damping=True, the pivot d + dt * damping) at the same inputs, forward only, CUDA events, the two
alternated in rounds within one run.

    python scripts/bench_implicit_damping.py [--iters 20] [--rounds 3]

Cases (gravity + damping, dt = 1 ms):
  * Kuka iiwa open-loop rollout (f small and random) and PD rollout (per-row gains, reference velocities, a torque limit)
    at (B, T) = (4096, 256) and (65 536, 64);
  * the Allegro hand's four fingertips held (position) in the contact rollout at (4096, 256), omega = 200 /s, from rest;
    the explicit step diverges on these fingers, so beside the times it reports the share of rows that stay finite and
    solved at every step, for both.
Prints one JSON line per case with the median over rounds of the mean ms per call, the implicit / explicit ratio, the
card's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import differentiable_robot_model_b200 as drm  # noqa: E402

DEV = "cuda:0"
DT = 1e-3
TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:     # the numbers still stand; say that the card could not be read
        return f"unknown ({exc})"


def event_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def start_state(m, batch, gen):
    limits = m.get_joint_limits()
    lo = torch.tensor([l["lower"] for l in limits], device=DEV)
    hi = torch.tensor([l["upper"] for l in limits], device=DEV)
    return lo + (hi - lo) * (0.3 + 0.4 * torch.rand(batch, m._n_dofs, device=DEV, generator=gen))


def kuka_cases(m, batch, steps):
    n = m._n_dofs
    gen = torch.Generator(device=DEV).manual_seed(0)
    q0 = start_state(m, batch, gen)
    qd0 = torch.zeros_like(q0)
    f = 0.05 * torch.randn(steps, batch, n, device=DEV, generator=gen)
    s = DT * torch.arange(1, steps + 1, device=DEV).view(steps, 1, 1)
    freq = 2 * torch.pi * (0.5 + torch.rand(batch, n, device=DEV, generator=gen))
    q_ref, qd_ref = q0 + 0.1 * torch.sin(freq * s), 0.1 * freq * torch.cos(freq * s)
    H = torch.diagonal(m.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2)
    kp, kd, lim = 400.0 * H, 40.0 * H, 20.0 * H.mean(0)

    def open_loop(implicit):
        return lambda: m.compute_forward_dynamics_rollout(q0, qd0, f, DT, True, True, implicit_damping=implicit)

    def pd(implicit):
        return lambda: m.compute_pd_controlled_rollout(q0, qd0, q_ref, kp, kd, DT, qd_ref=qd_ref, effort_limit=lim,
                                                       use_damping=True, implicit_damping=implicit)

    return {f"kuka_open_loop_B{batch}_T{steps}": open_loop, f"kuka_pd_B{batch}_T{steps}": pd}


def allegro_case(batch, steps):
    m = drm.DifferentiableRobotModel(os.path.join(REPO, "differentiable_robot_model_b200", "robot_data", "allegro",
                                                  "urdf", "allegro_hand_description_left.urdf"), "allegro", device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(1)
    q0 = start_state(m, batch, gen)
    qd0 = torch.zeros_like(q0)
    f = torch.zeros(steps, batch, m._n_dofs, device=DEV)

    def contact(implicit):
        return lambda: m.compute_contact_rollout(q0, qd0, f, TIPS, DT, stabilization=0.2 / DT, use_damping=True,
                                                 position_only=True, implicit_damping=implicit)

    def finite_and_solved(implicit):
        out = contact(implicit)()
        ok = out.solved & torch.isfinite(out.q).all(2).all(0) & torch.isfinite(out.qd).all(2).all(0)
        return float(ok.float().mean())

    return {f"allegro_4tips_contact_B{batch}_T{steps}": contact}, finite_and_solved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = gpu_info()
    kuka = drm.DifferentiableKUKAiiwa(device=DEV)
    cases = {}
    with torch.no_grad():
        for batch, steps in ((4096, 256), (65536, 64)):
            cases.update(kuka_cases(kuka, batch, steps))
        contact, finite_and_solved = allegro_case(4096, 256)
        cases.update(contact)
        for name, make in cases.items():
            fns = {"explicit": make(False), "implicit": make(True)}
            times = {k: [] for k in fns}
            for _ in range(args.rounds):               # alternated: both see the same clocks and neighbours
                for k, fn in fns.items():
                    times[k].append(event_ms(fn, args.iters))
            med = {k: statistics.median(v) for k, v in times.items()}
            row = {"case": name, "explicit_ms": round(med["explicit"], 4), "implicit_ms": round(med["implicit"], 4),
                   "implicit_over_explicit": round(med["implicit"] / med["explicit"], 4),
                   "explicit_ms_rounds": [round(x, 4) for x in times["explicit"]],
                   "implicit_ms_rounds": [round(x, 4) for x in times["implicit"]], "gpu": card}
            if name.startswith("allegro"):
                row["finite_and_solved_explicit"] = finite_and_solved(False)
                row["finite_and_solved_implicit"] = finite_and_solved(True)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
