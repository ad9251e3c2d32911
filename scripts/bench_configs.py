#!/usr/bin/env python
"""Secondary measurements for the other BASELINE.json configs (NOT the contract bench; see bench.py):

  config 3  Franka Panda RNEA (gravity + damping), batch 65 536 and 2^21
  config 4  Allegro hand FK + Jacobian of one fingertip, per-GPU shard 32 768 and 2^21
  config 5  Kuka iiwa FK+Jacobian + RNEA forward, then backward with mass / com / inertia_mat of links 1..7
            learnable, per-GPU shard 131 072

CUDA-event timing on the launching stream, >= 5 warm-up iterations, inputs rotated over buffer sets
larger than L2.  Prints one JSON object; copy it to profiles/ to have it judged.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import differentiable_robot_model_b200 as drm  # noqa: E402
from differentiable_robot_model_b200 import engine  # noqa: E402
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar, UnconstrainedTensor  # noqa: E402
from oracle import drm_oracle as O  # noqa: E402

DEV = torch.device("cuda", 0)
PEAK = 3350.0                 # H100 SXM data-sheet HBM3 bandwidth (GB/s) unless MEASURED_PEAKS.json gives a measured one
try:
    PEAK = float(json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass


def timed(fn, iters, warmup=5, inflight=4, n_sets=8):
    """ms per call.  Small launches (iters >= 100) are replayed from a CUDA graph with `inflight` independent
    calls in flight on parallel branches (like bench.py); big ones are launched back to back."""
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if iters < 100:
        e0.record()
        for i in range(iters):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters
    stream = torch.cuda.Stream()
    inflight = min(inflight, n_sets)
    side = [torch.cuda.Stream() for _ in range(inflight - 1)]
    nodes = 128
    with torch.cuda.stream(stream):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            fork = torch.cuda.Event()
            fork.record(stream)
            for s in side:
                s.wait_event(fork)
            for i in range(nodes):
                if i % inflight == 0:
                    fn(i)
                else:
                    with torch.cuda.stream(side[i % inflight - 1]):
                        fn(i)
            for s in side:
                j = torch.cuda.Event()
                j.record(s)
                stream.wait_event(j)
        g.replay()
        stream.synchronize()
        reps = max(1, iters // nodes) * 8
        e0.record(stream)
        for _ in range(reps):
            g.replay()
        e1.record(stream)
        stream.synchronize()
    return e0.elapsed_time(e1) / (reps * nodes)


def rotate_count(bytes_per_set):
    return max(2, int(300e6 // max(bytes_per_set, 1)) + 1)


def bench_rnea(stem_cls, batch):
    m = stem_cls(device=DEV)
    robot = O.load_robot(m.urdf_path, torch.float32)
    n = robot.n_dofs
    R = rotate_count(batch * 16 * n)
    sets = [tuple(t.to(DEV) for t in O.sample_inputs(robot, batch, seed=r)) for r in range(min(R, 8))]
    outs = [torch.empty(batch, n, device=DEV) for _ in sets]
    table, topo = m._link_table(), m._topology
    folded = engine.fold_link_table(topo, table)          # what model.compute_inverse_dynamics does for a constant model
    ms = timed(lambda i: engine.inverse_dynamics_raw(topo, table, *sets[i % len(sets)], 3, out=outs[i % len(sets)], folded=folded),
               200 if batch <= (1 << 17) else 20)
    ms_in_kernel = timed(lambda i: engine.inverse_dynamics_raw(topo, table, *sets[i % len(sets)], 3, out=outs[i % len(sets)]),
                         200 if batch <= (1 << 17) else 20)
    by = 16 * n
    res = {"batch": batch, "ms": ms, "configs_per_s": batch / ms * 1e3, "algorithmic_bytes_per_config": by,
           "achieved_GBps": batch * by / ms / 1e6, "hbm_frac": batch * by / ms / 1e6 / PEAK,
           "table": "folded once (drmb200_fold_link_table)" if folded is not None else "as given",
           "configs_per_s_folding_in_the_kernel": batch / ms_in_kernel * 1e3}
    if batch <= 65536 and engine.lib().drmb200_set_option is not None and os.environ.get("DRMB200_SKIP_CPU") is None:
        # CPU beside it, same box: scalar C port on all cores and the torch port (bounded samples)
        import time
        from oracle.c_oracle import CRobot
        cr = CRobot(robot)
        nq, nqd, nqdd = (t.cpu().numpy() for t in sets[0])
        cr.inverse_dynamics(nq[:4096], nqd[:4096], nqdd[:4096])
        t0 = time.perf_counter()
        cr.inverse_dynamics(nq, nqd, nqdd)
        res["cpu_c_port_configs_per_s"] = batch / (time.perf_counter() - t0)
        res["cpu_c_port_cores"] = os.cpu_count()
        cq = [t[:4096].cpu() for t in sets[0]]
        torch.set_num_threads(8)
        with torch.no_grad():
            O.inverse_dynamics(robot, *cq)
            t0 = time.perf_counter()
            for _ in range(3):
                O.inverse_dynamics(robot, *cq)
        res["cpu_torch_port_configs_per_s"] = 3 * 4096 / (time.perf_counter() - t0)
        res["cpu_torch_port_threads"] = 8
    return res


def bench_forward_dynamics(stem_cls, batch):
    """Articulated-body kernel (forward) and its adjoint kernel (input gradients / input + table gradients)."""
    import ctypes
    m = stem_cls(device=DEV)
    robot = O.load_robot(m.urdf_path, torch.float32)
    n = robot.n_dofs
    sets = [tuple(t.to(DEV) for t in O.sample_inputs(robot, batch, seed=r)) for r in range(min(rotate_count(batch * 16 * n), 8))]
    fs = [torch.randn(batch, n, device=DEV) for _ in sets]
    outs = [torch.empty(batch, n, device=DEV) for _ in sets]
    table, topo = m._link_table(), m._topology
    K = len(sets)
    ms = timed(lambda i: engine.forward_dynamics_raw(topo, table, sets[i % K][0], sets[i % K][1], fs[i % K], 3, out=outs[i % K]),
               200 if batch <= (1 << 17) else 20)
    res = {"batch": batch, "forward_ms": ms, "forward_configs_per_s": batch / ms * 1e3, "algorithmic_bytes_per_config": 16 * n,
           "forward_achieved_GBps": batch * 16 * n / ms / 1e6}
    g = torch.randn(batch, n, device=DEV)
    qg, qdg, fg, tg = torch.empty_like(g), torch.empty_like(g), torch.empty_like(g), torch.zeros_like(table)
    lib, P, S = engine.lib(), engine._ptr, engine._stream
    ws = torch.empty(int(lib.drmb200_forward_dynamics_backward_workspace_bytes(ctypes.byref(topo), batch)) // 4 + 1, device=DEV)

    def bwd(with_table):
        rc = lib.drmb200_forward_dynamics_backward(ctypes.byref(topo), P(table), P(sets[0][0]), P(sets[0][1]), P(fs[0]), batch, 3,
                                                   P(g), P(qg), P(qdg), P(fg), P(tg) if with_table else None, P(ws), S())
        assert rc == 0

    for name, wt in (("backward_inputs_ms", False), ("backward_inputs_and_table_ms", True)):
        res[name] = timed(lambda i: bwd(wt), 10)
    if batch <= 65536:
        # CPU baseline beside it: the torch port of the reference's articulated-body algorithm (oracle), bounded sample
        import time
        rows = 4096
        cq, cqd, cf = sets[0][0][:rows].cpu(), sets[0][1][:rows].cpu(), fs[0][:rows].cpu()
        best = 0.0
        for threads in (8, 32, os.cpu_count() or 8):
            torch.set_num_threads(threads)
            with torch.no_grad():
                O.forward_dynamics(robot, cq, cqd, cf, True, True)
                t0 = time.perf_counter()
                for _ in range(3):
                    O.forward_dynamics(robot, cq, cqd, cf, True, True)
                rate = 3 * rows / (time.perf_counter() - t0)
            if rate > best:
                best, res["cpu_port_threads"] = rate, threads
        res["cpu_port_configs_per_s"] = best
        res["cpu_port_sample"] = f"{rows} rows x 3 calls, torch CPU port of robot_model.py:488-624"
        # and the scalar C restatement on all host cores (oracle/drm_oracle.c, pthreads over the batch)
        from oracle.c_oracle import CRobot
        cr = CRobot(robot)
        nq, nqd, nf = (t.cpu().numpy() for t in (sets[0][0], sets[0][1], fs[0]))
        cr.forward_dynamics(nq[:4096], nqd[:4096], nf[:4096], True, True)
        t0 = time.perf_counter()
        cr.forward_dynamics(nq, nqd, nf, True, True)
        res["cpu_c_port_configs_per_s"] = batch / (time.perf_counter() - t0)
        res["cpu_c_port_cores"] = os.cpu_count()
    return res


def bench_kinematic_state(stem_cls, batch):
    """All-links pose (+ quaternion) (+ velocity) kernel and the pose-only FK of one link."""
    m = stem_cls(device=DEV)
    robot = O.load_robot(m.urdf_path, torch.float32)
    n, N = robot.n_dofs, len(robot.names)
    q, qd, _ = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=0))
    table, topo = m._link_table(), m._topology
    res = {"batch": batch, "n_links": N}
    for name, kw, by in (("poses", dict(qd=None, want_poses=True, want_quats=False), 4 * n + 48 * N),
                         ("poses_quats", dict(qd=None, want_poses=True, want_quats=True), 4 * n + 64 * N),
                         ("poses_vels", dict(qd=qd, want_poses=True, want_quats=False), 8 * n + 72 * N)):
        ms = timed(lambda i: engine.kinematic_state_raw(topo, table, q, **kw), 20)
        res[name] = {"ms": ms, "configs_per_s": batch / ms * 1e3, "algorithmic_bytes_per_config": by,
                     "achieved_GBps": batch * by / ms / 1e6, "hbm_frac": batch * by / ms / 1e6 / PEAK}
    ee = m._name_to_idx_map[robot.names[-1]]
    out = (torch.empty(batch, 3, device=DEV), torch.empty(batch, 4, device=DEV), None, None)
    ms = timed(lambda i: engine.fk_jacobian_raw(topo, ee, table, q, want_jac=False, out=out), 20)
    by = 4 * n + 28
    res["fk_pose_only"] = {"ms": ms, "configs_per_s": batch / ms * 1e3, "algorithmic_bytes_per_config": by,
                           "achieved_GBps": batch * by / ms / 1e6, "hbm_frac": batch * by / ms / 1e6 / PEAK}
    return res


def bench_mass_matrix(stem_cls, batch):
    """One-launch mass-matrix kernel vs the reference's construction through the RNEA kernel ((n + 1) x batch stacked)."""
    m = stem_cls(device=DEV)
    robot = O.load_robot(m.urdf_path, torch.float32)
    n = robot.n_dofs
    q = O.sample_inputs(robot, batch, seed=0)[0].to(DEV)
    table, topo = m._link_table(), m._topology
    out = torch.empty(batch, n, n, device=DEV)
    ms = timed(lambda i: engine.mass_matrix_raw(topo, table, q, out=out), 200 if batch <= (1 << 17) else 20)
    with torch.no_grad():
        ms_stacked = timed(lambda i: m.compute_lagrangian_inertia_matrix_stacked(q), 20)
    by = 4 * n + 4 * n * n
    return {"batch": batch, "kernel_ms": ms, "configs_per_s": batch / ms * 1e3, "algorithmic_bytes_per_config": by,
            "achieved_GBps": batch * by / ms / 1e6, "stacked_rnea_ms": ms_stacked}


def bench_fk(model, link, batch):
    robot = O.load_robot(model.urdf_path if hasattr(model, "urdf_path") else model._urdf_path, torch.float32)
    n = robot.n_dofs
    by = 28 * n + 28
    R = min(rotate_count(batch * by), 8)
    qs = [O.sample_inputs(robot, batch, seed=r)[0].to(DEV) for r in range(R)]
    outs = [(torch.empty(batch, 3, device=DEV), torch.empty(batch, 4, device=DEV), torch.empty(batch, 3, n, device=DEV),
             torch.empty(batch, 3, n, device=DEV)) for _ in range(R)]
    table, topo, ee = model._link_table(), model._topology, model._name_to_idx_map[link]
    ms = timed(lambda i: engine.fk_jacobian_raw(topo, ee, table, qs[i % R], out=outs[i % R]),
               200 if batch <= (1 << 17) else 20)
    return {"batch": batch, "link": link, "ms": ms, "configs_per_s": batch / ms * 1e3,
            "algorithmic_bytes_per_config": by, "achieved_GBps": batch * by / ms / 1e6,
            "hbm_frac": batch * by / ms / 1e6 / PEAK}


def bench_fk_multi(model, links, batch):
    """config 4 fused: (pos, quat, J_lin, J_ang) of several links from ONE tree-walk launch (csrc/fk_tree.cu)."""
    robot = O.load_robot(model.urdf_path if hasattr(model, "urdf_path") else model._urdf_path, torch.float32)
    n, E = robot.n_dofs, len(links)
    by = 4 * n + E * (28 + 24 * n)
    R = min(rotate_count(batch * by), 8)
    qs = [O.sample_inputs(robot, batch, seed=r)[0].to(DEV) for r in range(R)]
    outs = [(torch.empty(E, batch, 3, device=DEV), torch.empty(E, batch, 4, device=DEV), torch.empty(E, batch, 3, n, device=DEV),
             torch.empty(E, batch, 3, n, device=DEV)) for _ in range(R)]
    table, topo = model._link_table(), model._topology
    ees = [model._name_to_idx_map[l] for l in links]
    ms = timed(lambda i: engine.fk_jacobian_multi_raw(topo, ees, table, qs[i % R], out=outs[i % R]),
               200 if batch <= (1 << 17) else 20)
    return {"batch": batch, "links": links, "ms": ms, "configs_per_s": batch / ms * 1e3,
            "algorithmic_bytes_per_config": by, "achieved_GBps": batch * by / ms / 1e6,
            "hbm_frac": batch * by / ms / 1e6 / PEAK}


def bench_backward_kernels(batch):
    """Raw launches of the analytic adjoint kernels (Kuka): FK/Jacobian backward, full RNEA backward, inertial-only."""
    import ctypes
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    robot = O.load_robot(m.urdf_path, torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=0))
    table, topo, ee = m._link_table(), m._topology, m._name_to_idx_map["iiwa_link_ee"]
    g_pos, g_quat = torch.randn(batch, 3, device=DEV), torch.randn(batch, 4, device=DEV)
    g_jl, g_ja = torch.randn(batch, 3, 7, device=DEV), torch.randn(batch, 3, 7, device=DEV)
    g_tau = torch.randn(batch, 7, device=DEV)
    qg, tg = torch.empty_like(q), torch.zeros_like(table)
    ws = engine._workspace(topo, batch, DEV)
    lib, P, S = engine.lib(), engine._ptr, engine._stream
    out = {"batch": batch}

    def fk_bwd(with_table):
        rc = lib.drmb200_fk_jacobian_backward(ctypes.byref(topo), ee, P(table), P(q), batch, P(g_pos), P(g_quat), P(g_jl),
                                              P(g_ja), P(qg), P(tg) if with_table else None, P(ws), S())
        assert rc == 0

    qdg, qddg = torch.empty_like(q), torch.empty_like(q)

    def id_bwd(flags, inputs, with_table=True):
        rc = lib.drmb200_inverse_dynamics_backward(ctypes.byref(topo), P(table), P(q), P(qd), P(qdd), batch, flags, P(g_tau),
                                                   P(qg) if inputs else None, P(qdg) if inputs else None,
                                                   P(qddg) if inputs else None, P(tg) if with_table else None, P(ws), S())
        assert rc == 0

    for name, fn, by in (("fk_jacobian_backward_q_only", lambda i: fk_bwd(False), 28 + 28 + 168 + 28),
                         ("fk_jacobian_backward_q_and_table", lambda i: fk_bwd(True), 28 + 28 + 168 + 28),
                         ("rnea_backward_full", lambda i: id_bwd(3, True), 28 * 7),
                         ("rnea_backward_inputs_only", lambda i: id_bwd(3, True, False), 28 * 7),
                         ("rnea_backward_full_tree_kernel", lambda i: id_bwd(3, True), 28 * 7),
                         ("rnea_backward_inputs_only_tree_kernel", lambda i: id_bwd(3, True, False), 28 * 7),
                         ("rnea_backward_inertial_only", lambda i: id_bwd(3 | 4, False), 16 * 7)):
        engine.set_option("rnea_bwd_chain", 0 if name.endswith("tree_kernel") else 1)
        ms = timed(fn, 20)
        out[name] = {"ms": ms, "configs_per_s": batch / ms * 1e3, "algorithmic_bytes_per_config": by,
                     "achieved_GBps": batch * by / ms / 1e6}
    return out


def bench_train_step(batch, fused=False):
    """config 5 on one shard: FK+Jacobian + RNEA forward, scalar loss, backward to 21 inertial tensors.
    fused: model.fuse_learnable_parameters() (one flat Parameter, one table launch) + Adam(fused=True)."""
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    for i in range(1, 8):
        b = m._bodies[i]
        m.make_link_param_learnable(b.name, "mass", UnconstrainedScalar(init_val=b.inertia.mass().detach().clone()))
        m.make_link_param_learnable(b.name, "com", UnconstrainedTensor(1, 3, init_tensor=b.inertia.com().detach().clone()))
        m.make_link_param_learnable(b.name, "inertia_mat", UnconstrainedTensor(
            3, 3, init_tensor=b.inertia.inertia_mat().detach().clone().reshape(3, 3)))
    if fused:
        m.fuse_learnable_parameters()
    robot = O.load_robot(m.urdf_path, torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=0))
    target = torch.randn(batch, 7, device=DEV)

    def step(_):
        for p in m.parameters():
            p.grad = None
        with m.shared_link_table():
            pos, quat, jl, ja = m.compute_fk_and_jacobian(q, "iiwa_link_ee")
            tau = m.compute_inverse_dynamics(q, qd, qdd)
        loss = (tau - target).square().mean() + pos.square().mean()
        loss.backward()

    ms = timed(step, 20)
    res = {"batch": batch, "fused_parameters": fused, "ms_fwd_bwd": ms, "configs_per_s": batch / ms * 1e3,
           "algorithmic_bytes_per_config": 420, "achieved_GBps": batch * 420 / ms / 1e6,
           "note": "includes the differentiable table build (~40 small torch kernels) and the torch loss ops"}

    # the same step (plus the Adam update) captured ONCE in a CUDA graph and replayed: the host-side autograd / module
    # overhead that dominates the eager step disappears, what remains is the kernels
    try:
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True, fused=fused)

        def full_step():
            opt.zero_grad(set_to_none=False)
            with m.shared_link_table():
                pos, quat, jl, ja = m.compute_fk_and_jacobian(q, "iiwa_link_ee")
                tau = m.compute_inverse_dynamics(q, qd, qdd)
            loss = (tau - target).square().mean() + pos.square().mean()
            loss.backward()
            opt.step()
            return loss

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                full_step()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loss = full_step()
        for _ in range(3):
            graph.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
        gms = e0.elapsed_time(e1) / 50
        res["graphed_step_ms_fwd_bwd_adam"] = gms
        res["graphed_configs_per_s"] = batch / gms * 1e3
        res["graphed_final_loss"] = float(loss)
    except Exception as exc:                                    # report, do not hide
        res["graphed_error"] = repr(exc)[:300]
    return res


def main():
    out = {"peak_GBps": PEAK, "gpu": torch.cuda.get_device_name(0)}
    if os.environ.get("BENCH_ONLY") == "config5":
        out["config5_kuka_train_step"] = [bench_train_step(131072, fused=False), bench_train_step(131072, fused=True)]
        print(json.dumps(out))
        return
    if os.environ.get("BENCH_ONLY") == "backward":
        out["kuka_backward_kernels"] = [bench_backward_kernels(b) for b in (131072, 1 << 20)]
        print(json.dumps(out))
        return
    if os.environ.get("BENCH_ONLY") == "rnea":
        os.environ["DRMB200_SKIP_CPU"] = "1"
        out["config3_panda_rnea"] = [bench_rnea(drm.DifferentiableFrankaPanda, b) for b in (65536, 1 << 21)]
        out["kuka_rnea"] = [bench_rnea(drm.DifferentiableKUKAiiwa, b) for b in (65536, 1 << 21)]
        print(json.dumps(out))
        return
    if os.environ.get("BENCH_ONLY") == "config4":
        allegro = drm.DifferentiableRobotModel(os.path.join(drm.robot_model.robot_description_folder,
                                                            "allegro/urdf/allegro_hand_description_left.urdf"), device=DEV)
        allegro.urdf_path = os.path.join(drm.robot_model.robot_description_folder, "allegro/urdf/allegro_hand_description_left.urdf")
        tips = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
        out["config4_allegro_fk_jac"] = [bench_fk(allegro, "link_15.0_tip", b) for b in (32768, 1 << 21)]
        out["config4_allegro_fk_jac_tree_kernel_one_tip"] = [bench_fk_multi(allegro, tips[3:], b) for b in (32768, 1 << 21)]
        out["config4_allegro_fk_jac_fused_4_tips"] = [bench_fk_multi(allegro, tips, b) for b in (32768, 1 << 20)]
        print(json.dumps(out))
        return
    out["config3_panda_rnea"] = [bench_rnea(drm.DifferentiableFrankaPanda, b) for b in (65536, 1 << 21)]
    out["kuka_rnea"] = [bench_rnea(drm.DifferentiableKUKAiiwa, b) for b in (65536, 1 << 21)]
    engine.set_option("rnea_packed", 0)
    out["kuka_rnea_scalar_arithmetic"] = [bench_rnea(drm.DifferentiableKUKAiiwa, b) for b in (65536, 1 << 21)]
    engine.set_option("rnea_packed", 1)
    allegro = drm.DifferentiableRobotModel(os.path.join(drm.robot_model.robot_description_folder,
                                                        "allegro/urdf/allegro_hand_description_left.urdf"), device=DEV)
    allegro.urdf_path = allegro._urdf_model and os.path.join(drm.robot_model.robot_description_folder,
                                                             "allegro/urdf/allegro_hand_description_left.urdf")
    out["config4_allegro_fk_jac"] = [bench_fk(allegro, "link_15.0_tip", b) for b in (32768, 1 << 21)]
    tips = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
    out["config4_allegro_fk_jac_tree_kernel_one_tip"] = [bench_fk_multi(allegro, tips[3:], b) for b in (32768, 1 << 21)]
    out["config4_allegro_fk_jac_fused_4_tips"] = [bench_fk_multi(allegro, tips, b) for b in (32768, 1 << 20)]
    out["config5_kuka_train_step"] = [bench_train_step(131072, fused=False), bench_train_step(131072, fused=True)]
    out["kuka_backward_kernels"] = [bench_backward_kernels(131072)]
    out["kuka_mass_matrix"] = [bench_mass_matrix(drm.DifferentiableKUKAiiwa, b) for b in (65536, 1 << 20)]
    out["kuka_kinematic_state"] = [bench_kinematic_state(drm.DifferentiableKUKAiiwa, 1 << 20)]
    out["kuka_forward_dynamics"] =[bench_forward_dynamics(drm.DifferentiableKUKAiiwa, b) for b in (65536, 1 << 20)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
