#!/usr/bin/env python
"""PD-controlled rollouts of the Kuka iiwa (gravity + damping, dt = 1 ms, per-row gains, reference velocities, a torque
limit, no feed-forward): the one-launch kernel (compute_pd_controlled_rollout) against the open-loop rollout kernel at
the same sizes (what the feedback costs) and against the stepwise Python loop it replaces
(`u = kp * (q_ref - q) + kd * (qd_ref - qd); u = clamp(u, -lim, lim)`, compute_forward_dynamics, the integrate), eager and
replayed from a CUDA graph.  Forward alone, and forward + backward (gradients of the gains, the references and the
inertial parameters of every link, through one fused flat parameter).

    python scripts/bench_pd_rollout.py [--iters 10]

Prints one JSON line per (B, T) in (4096, 256), (65 536, 64) with every time (CUDA events, mean per call after
warm-up), configuration-steps per second, the algorithmic HBM bytes per configuration-step (forward: q_ref, qd_ref in,
q / qd / qdd / tau out = 24n; the open-loop rollout 16n) and the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import differentiable_robot_model_b200 as drm  # noqa: E402
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar, UnconstrainedTensor  # noqa: E402

DEV = "cuda:0"
SIZES = [(4096, 256), (65536, 64)]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:     # the numbers still stand; say that the card could not be read
        return f"unknown ({exc})"


def event_ms(fn, iters, graphed, warmup=3):
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


def model():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    for i in range(1, 8):                                  # the system-identification setting: inertial parameters learnable
        b = m._bodies[i]
        m.make_link_param_learnable(b.name, "mass", UnconstrainedScalar(init_val=b.inertia.mass().detach().clone()))
        m.make_link_param_learnable(b.name, "com", UnconstrainedTensor(1, 3, init_tensor=b.inertia.com().detach().clone()))
        m.make_link_param_learnable(b.name, "inertia_mat", UnconstrainedTensor(
            3, 3, init_tensor=b.inertia.inertia_mat().detach().clone().reshape(3, 3)))
    m.fuse_learnable_parameters()
    return m


def bench(m, batch, steps, iters):
    n, dt = m._n_dofs, 1e-3
    gen = torch.Generator(device=DEV).manual_seed(0)
    limits = m.get_joint_limits()
    lo = torch.tensor([l["lower"] for l in limits], device=DEV)
    hi = torch.tensor([l["upper"] for l in limits], device=DEV)
    q0 = lo + (hi - lo) * (0.3 + 0.4 * torch.rand(batch, n, device=DEV, generator=gen))
    qd0 = torch.zeros_like(q0)
    s = dt * torch.arange(1, steps + 1, device=DEV).view(steps, 1, 1)
    freq = 2 * torch.pi * (0.5 + torch.rand(batch, n, device=DEV, generator=gen))
    q_ref = q0 + 0.1 * torch.sin(freq * s)
    qd_ref = 0.1 * freq * torch.cos(freq * s)
    with torch.no_grad():
        H = torch.diagonal(m.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2)
    kp, kd = 400.0 * H, 40.0 * H                           # w = 20 rad/s, zeta = 1 per row
    lim = 20.0 * H.mean(0)                                # binds on part of the (step, row) entries
    f_open = 0.05 * torch.randn(steps, batch, n, device=DEV, generator=gen)
    G = torch.randn(steps, batch, n, device=DEV, generator=gen)
    flat = m.fused_link_params.flat
    kpa, kda, qra = (t.clone().requires_grad_(True) for t in (kp, kd, q_ref))
    fa = f_open.clone().requires_grad_(True)

    def pd_kernel(kp_, kd_, qr_):
        return m.compute_pd_controlled_rollout(q0, qd0, qr_, kp_, kd_, dt, qd_ref=qd_ref, effort_limit=lim,
                                               include_gravity=True, use_damping=True)

    def pd_loop(kp_, kd_, qr_):
        q, qd = q0, qd0
        outs = ([], [], [], [])
        for t in range(steps):
            u = torch.clamp(kp_ * (qr_[t] - q) + kd_ * (qd_ref[t] - qd), -lim, lim)
            qdd = m.compute_forward_dynamics(q, qd, u, True, True)
            qd = qd + dt * qdd
            q = q + dt * qd
            for lst, v in zip(outs, (q, qd, qdd, u)):
                lst.append(v)
        return tuple(torch.stack(lst) for lst in outs)

    def open_loop(ff):
        return m.compute_forward_dynamics_rollout(q0, qd0, ff, dt, True, True)

    def fwd(impl, *args):
        def run():
            with torch.no_grad():
                impl(*args)
        return run

    def fwd_bwd(impl, *args):
        def run():
            flat.grad = None
            for t in args:
                t.grad = None
            sum((v * G).sum() for v in impl(*args)).backward()
        return run

    cs = batch * steps
    res = {"batch": batch, "steps": steps, "dt": dt, "configuration_steps": cs, "gpu": gpu_info(),
           "algorithmic_bytes_per_configuration_step": {"pd_forward": 24 * n, "open_loop_forward": 16 * n}}
    cases = [("pd_kernel_forward", fwd(pd_kernel, kp, kd, q_ref), ("eager",)),
             ("open_loop_forward", fwd(open_loop, f_open), ("eager",)),
             ("pd_loop_forward", fwd(pd_loop, kp, kd, q_ref), ("eager", "graphed")),
             ("pd_kernel_forward_backward", fwd_bwd(pd_kernel, kpa, kda, qra), ("eager", "graphed")),
             ("open_loop_forward_backward", fwd_bwd(open_loop, fa), ("eager", "graphed")),
             ("pd_loop_forward_backward", fwd_bwd(pd_loop, kpa, kda, qra), ("eager", "graphed"))]
    for name, fn, modes in cases:
        for mode in modes:
            try:
                ms = event_ms(fn, iters, graphed=(mode == "graphed"))
            except Exception as exc:                                    # report, do not hide
                res[f"{name}_{mode}_error"] = repr(exc)[:300]
                continue
            res[f"{name}_{mode}_ms"] = round(ms, 4)
            res[f"{name}_{mode}_configuration_steps_per_s"] = cs / ms * 1e3
    with torch.no_grad():
        a, b = pd_kernel(kp, kd, q_ref), pd_loop(kp, kd, q_ref)
    res["kernel_equals_loop"] = all(torch.equal(x, y) for x, y in zip(a, b))
    res["limit_binds_fraction"] = float((a.tau.abs() == lim).float().mean())
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark times CUDA kernels and needs a GPU"
    m = model()
    for batch, steps in SIZES:
        print(json.dumps(bench(m, batch, steps, args.iters)), flush=True)


if __name__ == "__main__":
    main()
