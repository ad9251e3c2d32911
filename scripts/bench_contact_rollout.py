#!/usr/bin/env python
"""Contact-constrained rollouts (dt = 1 ms, gravity, Baumgarte rate omega = 200 /s, smooth random torques as in
examples/pinned_end_effector_iiwa.py): the one-launch kernel (compute_contact_rollout) against the stepwise torch loop it
replaces (compute_contact_dynamics with a torch Baumgarte term from compute_fk_and_jacobian_multi, then the integrate),
eager and replayed from a CUDA graph.

    python scripts/bench_contact_rollout.py [--iters 5] [--cases kuka_pos,kuka_pose,trifinger,allegro]

Cases: Kuka end effector position (the example's case), Kuka end effector pose, TriFinger's three tips (position),
Allegro's four tips (position).  The joints' damping acts on the Kuka and TriFinger, not on Allegro: the integrate
treats damping explicitly, which is stable only for dt below about 2 I / d, and with Allegro's finger damping (3-8 N m s/rad
on links of a few grams) every row diverges within ten steps at dt = 1 ms (and at 0.1 ms).  Sizes (B, T): (16, 1000), the example's; (4096, 256); (65 536, 64).  Prints one JSON
line per (case, B, T): ms per call (CUDA events, mean after warm-up), configuration-steps per second, the largest drift
of the held links from their targets of kernel and loop (on the rows every step of both solved; the
fraction the kernel solved is printed), the fraction of rows whose final state is finite, whether the two agree bit for bit at omega = 0 (checked on the
first 256 rows and 16 steps), the algorithmic HBM bytes per configuration-step (f in, q / qd / qdd out: 16n; force out:
4M) and the GPU's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import differentiable_robot_model_b200 as drm  # noqa: E402
from differentiable_robot_model_b200.robot_model import robot_description_folder  # noqa: E402

DEV = "cuda:0"
SIZES = [(16, 1000), (4096, 256), (65536, 64)]
OMEGA, DT = 200.0, 1e-3
TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
CASES = {
    # name: (URDF, held links, position only, joint damping on)
    "kuka_pos": ("kuka_iiwa/urdf/iiwa7.urdf", ["iiwa_link_ee"], True, True),
    "kuka_pose": ("kuka_iiwa/urdf/iiwa7.urdf", ["iiwa_link_ee"], False, True),
    "trifinger": ("trifinger_edu_description/trifinger_edu.urdf",
                  ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"], True, True),
    "allegro": ("allegro/urdf/allegro_hand_description_left.urdf", TIPS, True, False),
}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:     # the numbers still stand; say that the card could not be read
        return f"unknown ({exc})"


def event_ms(fn, iters, graphed, warmup=2):
    if graphed:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        run = g.replay
    else:
        run = fn
    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def rotvec(quat, target):
    """rotation vector of R R*^T from xyzw quaternions [B, 4], the shorter way round (torch, on the device)."""
    ax, ay, az, aw = quat.unbind(-1)
    bx, by, bz, bw = (-target[:, 0], -target[:, 1], -target[:, 2], target[:, 3])
    qe = torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                      aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)
    qe = torch.where(qe[:, 3:] < 0, -qe, qe)
    s = qe[:, :3].norm(dim=-1, keepdim=True)
    return torch.where(s > 0, 2 * torch.atan2(s, qe[:, 3:]) / s.clamp_min(1e-30), torch.zeros_like(s)) * qe[:, :3]


def make_loop(m, names, pos, damp, omega, q0, qd0, f):
    """The stepwise loop; returns (fn, result holder)."""
    multi = m.compute_fk_and_jacobian_multi(q0, names)
    tp = [multi[n][0].clone() for n in names]
    tq = [multi[n][1].clone() for n in names]
    out = {}

    def fn():
        q, qd = q0, qd0
        qs = []
        for t in range(f.shape[0]):
            a_ref = None
            if omega:
                mm = m.compute_fk_and_jacobian_multi(q, names)
                e, v = [], []
                for l, n in enumerate(names):
                    p, quat, jl, ja = mm[n]
                    e.append(p - tp[l])
                    v.append(torch.einsum("bmn,bn->bm", jl, qd))
                    if not pos:
                        e.append(rotvec(quat, tq[l]))
                        v.append(torch.einsum("bmn,bn->bm", ja, qd))
                a_ref = -(2 * omega) * torch.cat(v, 1) - (omega * omega) * torch.cat(e, 1)
            r = m.compute_contact_dynamics(q, qd, f[t], names, a_ref, use_damping=damp, position_only=pos)
            qd = qd + DT * r.qdd
            q = q + DT * qd
            qs.append(q)
        out["q"] = qs
    return fn, out


def max_drift(m, names, qs, q0, rows):
    """The largest distance of a held link from its start position over the rows `rows` (those every step solved)."""
    if not bool(rows.any()):
        return float("nan")
    p0 = m.compute_fk_and_jacobian_multi(q0[rows], names)
    worst = 0.0
    for q in qs:
        mm = m.compute_fk_and_jacobian_multi(q[rows], names)
        worst = max(worst, max(float((mm[n][0] - p0[n][0]).norm(dim=1).max()) for n in names))
    return worst


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--sizes", default=",".join(f"{b}x{t}" for b, t in SIZES))
    args = ap.parse_args()
    card = gpu_info()
    torch.manual_seed(0)
    for case in args.cases.split(","):
        rel, names, pos, damp = CASES[case]
        m = drm.DifferentiableRobotModel(os.path.join(robot_description_folder, rel), case, device=DEV)
        n = m._n_dofs
        M = (3 if pos else 6) * len(names)
        lim = m.get_joint_limits()
        lo = torch.tensor([l["lower"] for l in lim], device=DEV)
        hi = torch.tensor([l["upper"] for l in lim], device=DEV)
        for size in args.sizes.split(","):
            B, T = (int(x) for x in size.split("x"))
            q0 = lo + (hi - lo) * (0.3 + 0.4 * torch.rand(B, n, device=DEV))
            qd0 = torch.zeros_like(q0)
            inertia = torch.diagonal(m.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2)
            amp = 2.0 * inertia * torch.randn(3, B, n, device=DEV)
            freq = 2 * torch.pi * (0.5 + 2 * torch.rand(B, n, device=DEV))
            ts = (torch.arange(T, device=DEV, dtype=torch.float32) * DT).view(T, 1, 1)
            f = amp[0] + amp[1] * torch.sin(freq * ts) + amp[2] * torch.cos(0.7 * freq * ts)

            def kernel():
                return m.compute_contact_rollout(q0, qd0, f, names, DT, stabilization=OMEGA, use_damping=damp,
                                                 position_only=pos)
            res = kernel()
            k_ms = event_ms(kernel, args.iters, False)
            k_graph_ms = event_ms(kernel, args.iters, True)
            loop_fn, held = make_loop(m, names, pos, damp, OMEGA, q0, qd0, f)
            l_iters = max(1, args.iters // 2)
            l_ms = event_ms(loop_fn, l_iters, False, warmup=1)
            lg_ms = event_ms(loop_fn, l_iters, True, warmup=1)
            loop_fn()
            rows = res.solved & torch.stack([torch.isfinite(q).all(1) for q in held["q"]]).all(0)
            kd = max_drift(m, names, res.q, q0, rows)
            ld = max_drift(m, names, held["q"], q0, rows)
            # bit identity at omega = 0 on a slice
            b, t = min(B, 256), min(T, 16)
            z = m.compute_contact_rollout(q0[:b], qd0[:b], f[:t, :b].contiguous(), names, DT, use_damping=damp,
                                          position_only=pos)
            zf, zh = make_loop(m, names, pos, damp, 0.0, q0[:b], qd0[:b], f[:t, :b])
            zf()
            bitwise = all(torch.equal(a.view(torch.int32), w.view(torch.int32)) for a, w in zip(z.q, zh["q"]))
            rec = {"case": case, "B": B, "T": T, "n": n, "M": M, "damping": damp, "kernel_ms": round(k_ms, 3),
                   "kernel_graph_ms": round(k_graph_ms, 3), "loop_ms": round(l_ms, 3), "loop_graph_ms": round(lg_ms, 3),
                   "kernel_config_steps_per_s": B * T / (k_ms * 1e-3),
                   "loop_graph_config_steps_per_s": B * T / (lg_ms * 1e-3),
                   "speedup_vs_graphed_loop": round(lg_ms / k_ms, 2), "kernel_max_drift_m": kd, "loop_max_drift_m": ld,
                   "solved_fraction": float(res.solved.float().mean()),
                   "finite_fraction": float(torch.isfinite(res.q[-1]).all(1).float().mean()), "bitwise_at_omega0": bitwise,
                   "hbm_bytes_per_config_step": 16 * n + 4 * M, "gpu": card}
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
