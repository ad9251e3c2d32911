#!/usr/bin/env python
"""What implicit PD gains (stable PD) cost in the one-launch PD rollout: the explicit PD step against the implicit-gains
one (implicit_gains=True, the pivot + dt (kd + dt kp)) at the same inputs, forward and forward + backward, CUDA events,
the two alternated in rounds within one run.

    python scripts/bench_implicit_gains.py [--iters 20] [--rounds 3]

Cases (gravity + damping, dt = 1 ms; per-row gains kp = 400 H_kk, kd = 40 H_kk (w = 20 rad/s), reference velocities and
a torque limit):
  * Kuka iiwa at (B, T) = (4096, 256) and (65 536, 64), forward; forward + backward w.r.t. kp, kd at (4096, 64);
  * the Allegro hand at (4096, 256), forward, with implicit damping (its fingers need it at this step);
  * stiff gains, Kuka at w = 2000 rad/s, zeta = 1 and the Allegro hand at kd = 1.5 x 2 H_kk / dt (w = 400 rad/s): the
    share of rows that stay finite and the RMS tracking error at the last step, for both steps.
Prints one JSON line per case with the median over rounds of the mean ms per call, the implicit / explicit ratio, the
card's name and power limit."""
import argparse
import json
import os
import statistics
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import differentiable_robot_model_b200 as drm  # noqa: E402
from bench_implicit_damping import event_ms, gpu_info, start_state  # noqa: E402

DEV = "cuda:0"
DT = 1e-3


def allegro():
    return drm.DifferentiableRobotModel(os.path.join(REPO, "differentiable_robot_model_b200", "robot_data", "allegro", "urdf",
                                                     "allegro_hand_description_left.urdf"), "allegro", device=DEV)


def pd_inputs(m, batch, steps, seed=0):
    n = m._n_dofs
    gen = torch.Generator(device=DEV).manual_seed(seed)
    q0 = start_state(m, batch, gen)
    qd0 = torch.zeros_like(q0)
    s = DT * torch.arange(1, steps + 1, device=DEV).view(steps, 1, 1)
    freq = 2 * torch.pi * (0.5 + torch.rand(batch, n, device=DEV, generator=gen))
    q_ref, qd_ref = q0 + 0.1 * torch.sin(freq * s), 0.1 * freq * torch.cos(freq * s)
    H = torch.diagonal(m.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2)
    return q0, qd0, q_ref, qd_ref, H


def timed_cases(kuka, hand):
    cases = {}
    for batch, steps in ((4096, 256), (65536, 64)):
        q0, qd0, q_ref, qd_ref, H = pd_inputs(kuka, batch, steps)
        kp, kd, lim = 400.0 * H, 40.0 * H, 20.0 * H.mean(0)

        def fwd(gains, a=(q0, qd0, q_ref, qd_ref, kp, kd, lim)):
            return lambda: kuka.compute_pd_controlled_rollout(a[0], a[1], a[2], a[4], a[5], DT, qd_ref=a[3], effort_limit=a[6],
                                                              use_damping=True, implicit_gains=gains)
        cases[f"kuka_pd_fwd_B{batch}_T{steps}"] = fwd
    q0, qd0, q_ref, qd_ref, H = pd_inputs(kuka, 4096, 64)
    kp, kd, lim = (400.0 * H).requires_grad_(True), (40.0 * H).requires_grad_(True), 20.0 * H.mean(0)

    def fwd_bwd(gains, a=(q0, qd0, q_ref, qd_ref, kp, kd, lim)):
        def call():
            out = kuka.compute_pd_controlled_rollout(a[0], a[1], a[2], a[4], a[5], DT, qd_ref=a[3], effort_limit=a[6],
                                                     use_damping=True, implicit_gains=gains)
            torch.autograd.grad((out.q - a[2]).square().sum() + 1e-6 * out.tau.square().sum(), (a[4], a[5]))
        return call
    cases["kuka_pd_fwd_bwd_B4096_T64"] = fwd_bwd
    q0, qd0, q_ref, qd_ref, H = pd_inputs(hand, 4096, 256)
    hkp, hkd, hlim = 400.0 * H, 40.0 * H, 20.0 * H.mean(0)

    def hand_fwd(gains, a=(q0, qd0, q_ref, qd_ref, hkp, hkd, hlim)):
        return lambda: hand.compute_pd_controlled_rollout(a[0], a[1], a[2], a[4], a[5], DT, qd_ref=a[3], effort_limit=a[6],
                                                          use_damping=True, implicit_damping=True, implicit_gains=gains)
    cases["allegro_pd_fwd_B4096_T256"] = hand_fwd
    return cases


def stiff_rows(m, name, batch, steps, omega, zeta=None, kd_over=None):
    q0, qd0, _, _, H = pd_inputs(m, batch, steps, seed=2)
    kp = omega * omega * H
    kd = 2 * zeta * omega * H if kd_over is None else kd_over * 2 * H / DT
    target = q0 + 0.1
    q_ref = target.expand(steps, -1, -1).contiguous()
    row = {"case": name, "omega": omega, "zeta": zeta, "kd_over_2H_per_dt": kd_over, "B": batch, "T": steps}
    for gains in (False, True):
        out = m.compute_pd_controlled_rollout(q0, qd0, q_ref, kp, kd, DT, include_gravity=False, implicit_gains=gains)
        finite = torch.isfinite(out.q).all(2).all(0) & torch.isfinite(out.qd).all(2).all(0)
        err = (out.q[-1] - target)[finite]
        key = "implicit" if gains else "explicit"
        row[f"finite_rows_{key}"] = float(finite.float().mean())
        row[f"rms_tracking_error_{key}"] = float(err.square().mean().sqrt()) if err.numel() else None
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = gpu_info()
    kuka, hand = drm.DifferentiableKUKAiiwa(device=DEV), allegro()
    with torch.no_grad():
        cases = timed_cases(kuka, hand)
    for name, make in cases.items():
        fns = {"explicit": make(False), "implicit": make(True)}
        times = {k: [] for k in fns}
        grad = torch.enable_grad() if "bwd" in name else torch.no_grad()
        with grad:
            for _ in range(args.rounds):               # alternated: both see the same clocks and neighbours
                for k, fn in fns.items():
                    times[k].append(event_ms(fn, args.iters))
        med = {k: statistics.median(v) for k, v in times.items()}
        print(json.dumps({"case": name, "explicit_ms": round(med["explicit"], 4), "implicit_ms": round(med["implicit"], 4),
                          "implicit_over_explicit": round(med["implicit"] / med["explicit"], 4),
                          "explicit_ms_rounds": [round(x, 4) for x in times["explicit"]],
                          "implicit_ms_rounds": [round(x, 4) for x in times["implicit"]], "gpu": card}), flush=True)
    with torch.no_grad():
        for row in (stiff_rows(kuka, "kuka_stiff", 4096, 400, 2000.0, zeta=1.0),
                    stiff_rows(hand, "allegro_stiff", 4096, 400, 400.0, kd_over=1.5)):
            row["gpu"] = card
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
