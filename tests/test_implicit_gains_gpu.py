"""GPU: implicit PD gains (stable PD, DRMB200_IMPLICIT_GAINS) in the one-launch PD rollout and its adjoint:

  * zero gains give the explicit PD rollout bit for bit, on every shipped URDF and synthetic topology, with and without a
    limit, under explicit and implicit damping; one T-step launch is bit-identical to T chained one-step launches, per-row
    and shared gains, ragged and unaligned tiles, on every tile rung (a mirror of the launch rule picks the cases);
  * accuracy against the fp64 restatement (tests/implicit_gains_oracle.py) and the reference's goldens
    (tests/golden/*.implicit_gains_rollout.npz), values and gradients;
  * physics: the RNEA kernel closes each step, the applied torque is the PD law at the end-of-step state, the saturation
    mask follows its rule, stiff gains that make the explicit step diverge stay stable and converge, and gradient descent
    on the gains from such a start lowers the cost;
  * the contract: launch counts, CUDA graphs, double backward, argument refusals in Python and at the C ABI.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
import implicit_damping_oracle as I
import implicit_gains_oracle as IG
import synthetic_robots as SR
from conftest import GOLDEN_DIR, URDFS, urdf_path
from differentiable_robot_model_b200 import engine
from oracle import drm_oracle as O
from test_backward_gpu import cuda, learnable_model
from test_implicit_damping_gpu import _grads, compare_by_kind, compare_with_oracle, nonsym_robot, pd_case
from test_pd_rollout_topologies_gpu import SMEM_CAP, STATIC_SMEM, TWO_CTAS, family_inputs, pd_floats, program, select
from test_rollout_gpu import bits, family_close, misaligned
from test_synthetic_topologies_gpu import get

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = 1e-3
EINVAL = -1
SYMMETRIC = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro", "allegro_hand_description_left"]
SYNTHETIC = {k: v for k, v in SR.families().items() if sum(v.doc()[1][1:]) > 0}
KEYS = ("q", "qd", "qdd", "tau")
DAMPING = {"explicit": dict(use_damping=True), "implicit": dict(use_damping=True, implicit_damping=True)}


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_implicit_gains"))


def run(m, x, kp=None, kd=None, dt=DT, **kw):
    """compute_pd_controlled_rollout on the case tuple x = (q0, qd0, q_ref, qd_ref, f, kp, kd, lim); kw: qd_ref / f /
    effort_limit overrides (None drops them) and the model flags."""
    q0, qd0, q_ref, qd_ref, f, kp0, kd0, lim = x
    opt = dict(qd_ref=qd_ref, f=f, effort_limit=lim)
    opt.update(kw)
    return m.compute_pd_controlled_rollout(q0, qd0, q_ref, kp0 if kp is None else kp, kd0 if kd is None else kd, dt, **opt)


def chained(m, x, kp, kd, **kw):
    """T chained one-step launches of the rollout run() makes."""
    q0, qd0, q_ref, qd_ref, f, _, _, lim = x
    opt = dict(qd_ref=qd_ref, f=f, effort_limit=lim)
    opt.update(kw)
    q, qd = q0, qd0
    outs = ([], [], [], [])
    for t in range(q_ref.shape[0]):
        step = {k: (v[t:t + 1] if k in ("qd_ref", "f") and v is not None else v) for k, v in opt.items()}
        o = m.compute_pd_controlled_rollout(q, qd, q_ref[t:t + 1], kp, kd, DT, **step)
        q, qd = o.q[0], o.qd[0]
        for lst, v in zip(outs, o):
            lst.append(v[0])
    return tuple(torch.stack(lst) for lst in outs)


def same(got, want, what, tau_where_finite=False):
    for name, a, b in zip(KEYS, got, want):
        if name == "tau" and tau_where_finite:
            ok = torch.isfinite(want[2])                # tau = u - 0 * qdd is NaN where the explicit qdd is not finite
            a, b = a[ok], b[ok]
        assert torch.equal(bits(a), bits(b)), (what, name)


# ---------------------------------------------------------------------------------------------------------------------
# 1. bit-identity: zero gains, chained steps, every rung
# ---------------------------------------------------------------------------------------------------------------------
def zero_gains_identity(m, x, what):
    z = torch.zeros_like(x[5])
    for mode, kw in DAMPING.items():
        for lim in (None, x[7]):
            got = run(m, x, z, z, effort_limit=lim, implicit_gains=True, **kw)
            want = run(m, x, z, z, effort_limit=lim, **kw)
            same(got, want, (what, mode, lim is not None), tau_where_finite=True)


@pytest.mark.parametrize("stem", sorted(URDFS))
def test_zero_gains_are_bit_identical_to_the_explicit_pd_rollout(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    with torch.no_grad():
        for batch in (5, 65, 20000):
            zero_gains_identity(m, pd_case(m, stem, batch, 3, seed=batch), (stem, batch))


@pytest.mark.parametrize("name", sorted(SYNTHETIC))
def test_zero_gains_on_synthetic_topologies_are_bit_identical(name, model_dir):
    path = SR.build(SYNTHETIC[name], model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    robot = O.load_robot(path, torch.float32)
    with torch.no_grad():
        zero_gains_identity(m, pd_case(m, robot, 40, 2, seed=2, unit_gains=True), name)


@pytest.mark.parametrize("stem", sorted(URDFS))
def test_one_launch_is_bit_identical_to_chained_one_step_launches(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    with torch.no_grad():
        x = pd_case(m, stem, 65, 4, seed=7)
        kp, kd = x[5], x[6]
        layouts = {"per_row": (kp, kd), "shared": (kp.mean(0), kd.mean(0)), "mixed": (kp, kd.mean(0))}
        for lname, (a, b) in layouts.items():
            for mode, kw in DAMPING.items():
                for opt in ({}, {"qd_ref": None, "f": None, "effort_limit": None}):
                    got = run(m, x, a, b, implicit_gains=True, **kw, **opt)
                    want = chained(m, x, a, b, implicit_gains=True, **kw, **opt)
                    same(got, want, (stem, lname, mode, sorted(opt)))
        # unaligned bases and a batch that leaves a ragged last tile
        got = run(m, x, kp, kd, implicit_gains=True, use_damping=True)
        q0, qd0, q_ref, qd_ref, f, _, _, lim = x
        y = (misaligned(q0), qd0, q_ref, qd_ref, misaligned(f), kp, kd, lim)
        same(run(m, y, misaligned(kp), kd, implicit_gains=True, use_damping=True), got, (stem, "misaligned"))


def gains_floats(T, n, n_links, n_slots, n_in, per_row):
    """PDRolloutSmem(..., gains = true).total_floats: the explicit layout plus the [T, n] pivot addends."""
    return pd_floats(T, n, n_links, n_slots, n_in, per_row) + T * n


def gains_tile(prog, batch, n_in, per_row, sms):
    """launch_rollout's choice for the implicit-gains kernels: (tile, dynamic + static bytes); tile None = ELIMIT."""
    def need(T):
        return 4 * gains_floats(T, *prog, n_in, per_row)
    T = 64 if -(-batch // 64) >= sms and need(64) <= TWO_CTAS else 32
    if need(T) + STATIC_SMEM > SMEM_CAP:
        T = 16
    return (T if need(T) + STATIC_SMEM <= SMEM_CAP else None), need(T) + STATIC_SMEM


def sm_count():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def test_the_mirror_fits_the_63_dof_chain_at_16_rows():
    lib = engine.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    for t in (64, 32, 16):
        for imp in (0, 1):
            sym = f"_ZN3drm32pd_rollout_implicit_gains_kernelILi{t}ELb{imp}EEEvNS_11TreeProgramENS_11FoldProgramENS_13PDRolloutArgsE"
            attr = (ctypes.c_size_t * 64)()
            assert cudart.cudaFuncGetAttributes(attr, ctypes.cast(getattr(lib, sym), ctypes.c_void_p)) == 0, sym
            assert attr[0] == STATIC_SMEM, (sym, attr[0])
    # 63 DoFs, 64 links, per-row gains and all three streams: 243 072 B at 32 rows, 125 248 B at 16 (4 032 B more)
    need32, need16 = 4 * gains_floats(32, 63, 64, 0, 3, True), 4 * gains_floats(16, 63, 64, 0, 3, True)
    print(f"63-DoF chain, per-row gains, 3 streams: {need32} B at 32 rows, {need16} B at 16 rows (+ {STATIC_SMEM} static)")
    assert need16 - 4 * pd_floats(16, 63, 64, 0, 3, True) == 4032
    assert need32 + STATIC_SMEM > SMEM_CAP >= need16 + STATIC_SMEM
    assert gains_tile((63, 64, 0), 67, 3, True, sm_count())[0] == 16


# rung -> (family, gains per row, qd_ref and f given, batch; None: 64 rows for every SM plus a ragged row)
RUNGS = {64: ("D_fixed", False, False, None), 32: ("D_fixed", True, True, 67), 16: ("F_chain64", True, True, 67)}


def tuple_of(x):
    return (x["q0"], x["qd0"], x["q_ref"], x["qd_ref"], x["f"], x["kp"], x["kd"], x["lim"])


@pytest.mark.parametrize("rung", sorted(RUNGS))
def test_every_rung_runs_the_mirror_tile_and_matches_chained_steps(rung, model_dir):
    name, per_row, streams, batch = RUNGS[rung]
    M = get(name, model_dir)
    batch = batch or 64 * sm_count() + 1
    x = select(family_inputs(M, batch, 4, seed=rung), per_row, streams, streams, True)
    n_in = 1 + (x["qd_ref"] is not None) + (x["f"] is not None)
    assert gains_tile(program(M), batch, n_in, per_row, sm_count())[0] == rung
    if rung == 16:                   # 64 and 32 rows exceed the limit here: a launch that succeeds ran the 16-row kernel
        assert 4 * gains_floats(32, *program(M), n_in, per_row) + STATIC_SMEM > SMEM_CAP
    x = tuple_of(x)
    # which instantiation runs is not read back with torch.profiler here: a profiling session in this process made
    # test_pd_rollout_topologies_gpu's profiled rung check, which runs later, see no kernel events at all
    with torch.no_grad():
        got = run(M.m, x, implicit_gains=True, use_damping=True)
        want = chained(M.m, x, x[5], x[6], implicit_gains=True, use_damping=True)
    same(got, want, (name, rung))


# ---------------------------------------------------------------------------------------------------------------------
# 2. accuracy against the fp64 restatement and the reference
# ---------------------------------------------------------------------------------------------------------------------
def oracle_rollout(robot, x, mode, dtype):
    c = [None if v is None else v.detach().cpu().to(dtype) for v in x]
    q0, qd0, q_ref, qd_ref, f, kp, kd, lim = c
    return IG.pd_rollout(robot, q0, qd0, q_ref, kp, kd, DT, qd_ref, f, lim, True, True, mode == "implicit")


@pytest.mark.parametrize("nonsym", [False, True])
@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "trifinger_edu", "allegro_hand_description_left"])
def test_rollout_matches_fp64_restatement(stem, nonsym):
    robot = nonsym_robot(stem) if nonsym else O.load_robot(urdf_path(stem), torch.float64)
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    table = O.link_table(robot.to(torch.float32)).float().to(DEV).contiguous()
    x = pd_case(m, stem, 128, 8, seed=13)
    x = x[:5] + (50 * x[5], 5 * x[6], x[7])                   # stiffer: w = 141 rad/s, zeta = 0.71
    # the Allegro fingers' explicit damping diverges at this step whatever the gains: implicit damping only there
    for mode in ("implicit",) if stem.startswith("allegro") else tuple(DAMPING):
        flags = engine.GRAVITY | engine.DAMPING | engine.IMPLICIT_GAINS | (engine.IMPLICIT_DAMPING if mode == "implicit" else 0)
        with torch.no_grad():
            got = engine.pd_rollout_raw(m._topology, table, x[0], x[1], x[2], x[5], x[6], DT, flags, x[3], x[4], x[7])
        want = oracle_rollout(robot, x, mode, torch.float64)
        o32 = oracle_rollout(robot.to(torch.float32), x, mode, torch.float32)
        for k, g, w, w32 in zip(KEYS, got, want, o32):
            scale = w.abs().amax(-1, keepdim=True).clamp_min(1e-6)
            err = float(((g.cpu().double() - w).abs() / scale).max())
            e32 = float(((w32.double() - w).abs() / scale).max())
            print(f"{stem} nonsym={nonsym} {mode} {k}: {err:.2e} vs fp64 (fp32 restatement {e32:.2e})")
            assert err <= max(8 * e32, 1e-5), (mode, k, err, e32)


def gains_grads_case(stem, mode, per_row=True, steps=6, batch=64):
    m, params = learnable_model(stem)
    with torch.no_grad():
        q0, qd0, q_ref, qd_ref, f, kp, kd, lim = pd_case(m, stem, batch, steps, seed=21)
    kp, kd = 50 * kp, 5 * kd
    if not per_row:
        kp, kd = kp.mean(0), kd.mean(0)
    ins = (q0, qd0, q_ref, qd_ref, f, kp, kd)
    kw = dict(DAMPING[mode], implicit_gains=True)

    def fused(mm, *a):
        return tuple(mm.compute_pd_controlled_rollout(a[0], a[1], a[2], a[5], a[6], DT, qd_ref=a[3], f=a[4], effort_limit=lim,
                                                      **kw))

    def loop(mm, *a):
        return chained(mm, (a[0], a[1], a[2], a[3], a[4], None, None, lim), a[5], a[6], **kw)

    return m, params, ins, lim, fused, loop


@pytest.mark.parametrize("stem,mode,per_row", [("iiwa7", "explicit", True), ("iiwa7", "implicit", False),
                                               ("allegro_hand_description_left", "implicit", True),
                                               ("trifinger_edu", "explicit", False)])
def test_pd_rollout_gradients_match_chained_steps_and_fp64_oracle(stem, mode, per_row):
    m, params, ins, lim, fused_fn, loop_fn = gains_grads_case(stem, mode, per_row)
    steps, batch, n = ins[2].shape
    gen = torch.Generator().manual_seed(22)
    G = [torch.randn(steps, batch, n, generator=gen) for _ in range(4)]
    Gd = [x.to(DEV) for x in G]
    fused = _grads(m, params, fused_fn, ins, Gd)
    loop = _grads(m, params, loop_fn, ins, Gd)
    compare_by_kind(fused, loop, params, len(ins), 1e-4, "chained")
    lim64 = lim.cpu().double()

    def oracle_loss(r, *a):
        out = IG.pd_rollout(r, a[0], a[1], a[2], a[5], a[6], DT, a[3], a[4], lim64, True, True, mode == "implicit")
        return sum((w.double() * v).sum() for w, v in zip(G, out))

    worst = compare_with_oracle(stem, fused, oracle_loss, ins, params)
    print(f"{stem} {mode} per_row={per_row}: worst family-relative gradient error vs fp64 oracle {worst:.2e}")


# the goldens' own family-relative distance from the fp64 restatement (tests/test_oracle_implicit_gains.py) is the floor
GOLDEN_TOL = {"iiwa7_allegro": 5e-3}


@pytest.mark.parametrize("stem", SYMMETRIC)
def test_rollout_matches_reference_trajectories_and_gradients(stem):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".implicit_gains_rollout.npz"), allow_pickle=False)
    dt = float(g["dt"])
    tol = GOLDEN_TOL.get(stem, 5e-4)
    const = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    names = ("q0", "qd0", "q_ref", "qd_ref", "f", "kp", "kd")
    for tag in sorted({k.split(".")[0] for k in g.files if k.startswith(("g0", "g1"))}):
        kw = dict(include_gravity=tag.startswith("g1"), use_damping=True, implicit_damping=tag.endswith("i"),
                  implicit_gains=True)
        with torch.no_grad():
            a = [cuda(g[k]) for k in names]
            traj = const.compute_pd_controlled_rollout(a[0], a[1], a[2], a[5], a[6], dt, qd_ref=a[3], f=a[4], **kw)
        for name, got in zip(KEYS, traj):
            want = g[f"{tag}.{name}"]
            scale = np.abs(want).max(axis=2, keepdims=True)
            rel = (np.abs(got.cpu().numpy() - want) / (scale + 1e-6)).max()
            assert rel < 2e-3, (tag, name, rel)
        m, params = learnable_model(stem)
        a = [cuda(g[k], True) for k in names]
        traj = m.compute_pd_controlled_rollout(a[0], a[1], a[2], a[5], a[6], dt, qd_ref=a[3], f=a[4], **kw)
        sum((cuda(g[f"G_{k}"]) * v).sum() for k, v in zip(KEYS, traj)).backward()
        prefix = f"{tag}.grad."
        worst = 0.0
        for key, t in zip(names, a):
            worst = max(worst, family_close(t.grad.cpu().numpy(), g[prefix + key], tol, f"{tag}.{key}"))
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in names:
                continue
            pname, idx = key[len(prefix):].rsplit(".", 1)
            p = params[(int(idx), pname)]
            got = (torch.zeros_like(p) if p.grad is None else p.grad).cpu().numpy().reshape(g[key].shape)
            want = g[key]
            if pname == "inertia_mat":       # the goldens differentiate H and nle: only the symmetric part is shared
                got, want = got + got.T, want + want.T
            fam = max(np.abs(g[k]).max() for k in g.files if k.startswith(prefix + pname + "."))
            fam = 2 * fam if pname == "inertia_mat" else fam
            err = np.abs(got.reshape(-1) - want.reshape(-1)).max()
            assert err <= tol * max(fam, 1e-30), (key, err, fam)
            worst = max(worst, err / max(fam, 1e-30))
        print(f"{stem} {tag}: worst family-relative gradient error vs reference {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. physics
# ---------------------------------------------------------------------------------------------------------------------
def states_before(x, out):
    return torch.cat([x[0][None], out.q[:-1]]), torch.cat([x[1][None], out.qd[:-1]])


def predicted_command(x, qs, qds, kp, kd):
    """u-hat of every step, rounded as the kernel rounds it (each torch operation is one rounded fp32 operation)."""
    q_ref, qd_ref, f = x[2], x[3], x[4]
    qp = qs + DT * qds
    return (f + kp * (q_ref - qp)) + kd * (qd_ref - qds)


@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "trifinger_edu", "allegro_hand_description_left"])
def test_inverse_dynamics_closes_each_step_and_tau_is_the_end_of_step_law(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    x = pd_case(m, stem, 512, 6, seed=51)
    kp, kd = 50 * x[5], 5 * x[6]
    d = I.damping_vector(O.load_robot(urdf_path(stem), torch.float32)).to(DEV)
    # damping: none, explicit (not on the Allegro fingers, which it makes diverge at this step) and implicit, where
    # H qdd + nle = tau - dt D qdd
    modes = {"none": {}, "implicit": DAMPING["implicit"]}
    if not stem.startswith("allegro"):
        modes["explicit"] = DAMPING["explicit"]
    with torch.no_grad():
        for grav in (True, False):
            for mode, kw in modes.items():
                out = run(m, x, kp, kd, implicit_gains=True, include_gravity=grav, **kw)
                qs, qds = states_before(x, out)
                u = predicted_command(x, qs, qds, kp, kd)
                for t in range(x[2].shape[0]):
                    tau = m.compute_inverse_dynamics(qs[t], qds[t], out.qdd[t], grav, use_damping=mode != "none")
                    if mode == "implicit":
                        tau = tau + DT * d * out.qdd[t]
                    scale = (tau.abs() + out.tau[t].abs()).amax(1, keepdim=True).clamp_min(1e-3)
                    err = float(((tau - out.tau[t]).abs() / scale).max())
                    assert err < 2e-3, (grav, mode, t, err)
                    # unsaturated joints: the PD law at the end-of-step state
                    sat = ~((u[t] >= -x[7]) & (u[t] <= x[7]))
                    law = (x[4][t] + kp * (x[2][t] - out.q[t])) + kd * (x[3][t] - out.qd[t])
                    terms = (x[4][t].abs() + (kp * (x[2][t] - out.q[t])).abs() + (kd * (x[3][t] - out.qd[t])).abs())
                    rel = ((out.tau[t] - law).abs() / terms.amax(1, keepdim=True).clamp_min(1e-6))[~sat]
                    assert float(rel.max()) < 1e-4, (grav, mode, t, float(rel.max()))


def test_saturation_mask_follows_its_rule_and_blocks_gradients():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    x = pd_case(m, "iiwa7", 300, 5, seed=61)
    kp, kd = 50 * x[5], 5 * x[6]
    lim = x[7]
    ins = [t.detach().clone().requires_grad_(True) for t in (x[2], x[3], x[4])]
    out = m.compute_pd_controlled_rollout(x[0], x[1], ins[0], kp, kd, DT, qd_ref=ins[1], f=ins[2], effort_limit=lim,
                                          implicit_gains=True)
    with torch.no_grad():
        qs, qds = states_before(x, out)
        u = predicted_command(x, qs, qds, kp, kd)
        sat = ~((u >= -lim) & (u <= lim))
        share = float(sat.float().mean())
        print(f"saturated share of the entries: {share:.3f}")
        assert 0.05 < share < 0.95
        assert torch.equal(out.tau[sat], torch.clamp(u, -lim, lim)[sat])
        assert bool((out.tau[~sat] != u[~sat]).any())               # the pivot term moved the unsaturated ones
    (out.q.sum() + out.tau.sum()).backward()
    for t in ins:
        assert bool((t.grad[sat] == 0).all())
        assert bool((t.grad[~sat] != 0).any())


def stiff_case(stem, batch, omega, zeta, kd_over=None):
    """Per-row gains kp = omega^2 H_kk, kd = 2 zeta omega H_kk (kd_over: kd = kd_over * 2 H_kk / dt instead, above the
    explicit step's limit b < 2 for any kp)."""
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q0, _, _ = O.sample_inputs(robot, batch, seed=71)
    q0 = q0.to(DEV)
    with torch.no_grad():
        H = torch.diagonal(m.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2)
    kp = omega * omega * H
    kd = 2 * zeta * omega * H if kd_over is None else kd_over * 2 * H / DT
    return m, q0, kp, kd


@pytest.mark.parametrize("stem,omega,zeta,kd_over", [("iiwa7", 2000.0, 1.0, None),
                                                     ("allegro_hand_description_left", 400.0, None, 1.5)])
def test_stiff_gains_diverge_explicitly_and_converge_implicitly(stem, omega, zeta, kd_over):
    m, q0, kp, kd = stiff_case(stem, 256, omega, zeta, kd_over)
    T = 400
    target = q0 + 0.1
    q_ref = target.expand(T, -1, -1).contiguous()
    qd0 = torch.zeros_like(q0)
    with torch.no_grad():
        ex = m.compute_pd_controlled_rollout(q0, qd0, q_ref, kp, kd, DT, include_gravity=False)
        im = m.compute_pd_controlled_rollout(q0, qd0, q_ref, kp, kd, DT, include_gravity=False, implicit_gains=True)
    ex_err = (ex.q - target).abs().amax(2)
    bad = ~torch.isfinite(ex_err[-1]) | (ex_err[-1] > ex_err[0])
    im_err = (im.q - target).abs().amax(2)
    what = f"omega = {omega} rad/s, " + (f"zeta = {zeta}" if kd_over is None else f"kd = {kd_over} x 2 H_kk / dt")
    print(f"{stem}, {what}, dt = {DT}, T = {T}: explicit non-finite or growing on {int(bad.sum())} of {bad.numel()} rows; "
          f"implicit max |q - q_ref| {float(im_err[0].max()):.3g} -> {float(im_err[-1].max()):.3g}, "
          f"final max |qd| {float(im.qd[-1].abs().max()):.3g}")
    assert bool(bad.all())
    assert bool(torch.isfinite(im.q).all() and torch.isfinite(im.qd).all())
    assert float(im_err[-1].max()) < 1e-3


def test_gradient_descent_on_stiff_gains_lowers_the_cost():
    # identify moderate gains (omega = 100 rad/s, zeta = 0.5) from their trajectories, starting from gains the explicit
    # step cannot run (omega = 2000 rad/s, zeta = 1)
    m, q0, kp, kd = stiff_case("iiwa7", 64, 2000.0, 1.0)
    _, _, kp_true, kd_true = stiff_case("iiwa7", 64, 100.0, 0.5)
    T = 60
    t = torch.arange(1, T + 1, device=DEV, dtype=torch.float32)[:, None, None] * DT
    q_ref = q0 + 0.3 * torch.sin(2 * torch.pi * 2.0 * t)
    qd0 = torch.zeros_like(q0)
    with torch.no_grad():
        target = m.compute_pd_controlled_rollout(q0, qd0, q_ref, kp_true.mean(0), kd_true.mean(0), DT,
                                                 implicit_gains=True).q
        explicit = m.compute_pd_controlled_rollout(q0, qd0, q_ref, kp.mean(0), kd.mean(0), DT).q
    assert not bool(torch.isfinite(explicit).all())
    log_kp = torch.log(kp.mean(0)).clone().requires_grad_(True)
    log_kd = torch.log(kd.mean(0)).clone().requires_grad_(True)
    opt = torch.optim.Adam([log_kp, log_kd], lr=0.2)
    costs = []
    for _ in range(15):
        opt.zero_grad()
        out = m.compute_pd_controlled_rollout(q0, qd0, q_ref, log_kp.exp(), log_kd.exp(), DT, implicit_gains=True)
        cost = ((out.q - target) ** 2).mean()
        cost.backward()
        assert torch.isfinite(log_kp.grad).all() and torch.isfinite(log_kd.grad).all()
        opt.step()
        costs.append(float(cost))
    print(f"identifying Kuka gains from a stiff start through the implicit-gains rollout: cost {costs[0]:.4g} -> "
          f"{costs[-1]:.4g} in {len(costs)} Adam steps")
    assert costs[-1] < 0.5 * costs[0]


# ---------------------------------------------------------------------------------------------------------------------
# 4. the contract
# ---------------------------------------------------------------------------------------------------------------------
def test_launch_counts_graph_capture_and_double_backward():
    const = drm.DifferentiableKUKAiiwa(device=DEV)
    x = pd_case(const, "iiwa7", 1000, 25, seed=3)
    T = x[2].shape[0]
    run(const, x, implicit_gains=True)
    before = engine.launch_count()
    with torch.no_grad():
        run(const, x, implicit_gains=True, use_damping=True, implicit_damping=True)
    assert engine.launch_count() - before == 1
    kp = x[5].clone().requires_grad_(True)
    out = run(const, x, kp, implicit_gains=True)
    before = engine.launch_count()
    (out.q.sum() + out.tau.sum()).backward()
    assert engine.launch_count() - before == 2 * T + 1                  # no table gradient: no reduction
    m, params = learnable_model("iiwa7")
    with torch.no_grad():
        run(m, x, implicit_gains=True)
    out = run(m, x, kp, implicit_gains=True)
    before = engine.launch_count()
    (out.q.sum() + out.tau.sum()).backward()
    assert engine.launch_count() - before <= 2 * T + 2 + 4              # 2T + 2, the rest the table build's backward
    # double backward raises
    a = x[0][:8].clone().requires_grad_(True)
    o = const.compute_pd_controlled_rollout(a, x[1][:8], x[2][:3, :8], x[5][:8], x[6][:8], DT, implicit_gains=True)
    (g,) = torch.autograd.grad(o.q.sum(), a, create_graph=True)
    with pytest.raises(RuntimeError, match="second-order"):
        g.sum().backward()
    # forward and backward captured in one CUDA graph
    m.fuse_learnable_parameters()
    flat = m.fused_link_params.flat
    y = pd_case(const, "iiwa7", 777, 9, seed=9)
    G = torch.randn(9, 777, 7, generator=torch.Generator().manual_seed(3)).to(DEV)
    kpa = y[5].clone().requires_grad_(True)

    def step():
        o = run(m, y, kpa, implicit_gains=True, use_damping=True, implicit_damping=True)
        ((o.q + o.qd + o.tau) * G).sum().backward()
        return o.q

    flat.grad, kpa.grad = None, None
    eager = [step().detach().clone(), flat.grad.clone(), kpa.grad.clone()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            flat.grad, kpa.grad = None, None
            step()
    torch.cuda.current_stream().wait_stream(side)
    flat.grad = torch.zeros_like(flat)
    kpa.grad = torch.zeros_like(kpa)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        q = step()
    flat.grad.zero_()
    kpa.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(q, eager[0]) and torch.equal(flat.grad, eager[1]) and torch.equal(kpa.grad, eager[2])


def test_argument_refusals():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    x = pd_case(m, "iiwa7", 4, 3, seed=1)
    q0, qd0, f = x[0], x[1], x[4]
    kp = torch.ones(7, device=DEV)
    for bad in (0.0, -1e-3, float("inf"), float("nan")):
        with pytest.raises(AssertionError):
            m.compute_pd_controlled_rollout(q0, qd0, x[2], kp, kp, bad, implicit_gains=True)
    lib, topo, table = engine.lib(), ctypes.byref(m._topology), m._link_table().detach()
    out = torch.empty(3, 4, 7, device=DEV)
    P = engine._ptr
    s = engine._stream()
    ws = torch.empty(1 << 22, device=DEV)
    links = (ctypes.c_int32 * 1)(m._topology.n_links - 1)
    solved = torch.empty(4, dtype=torch.uint8, device=DEV)
    GAINS = engine.IMPLICIT_GAINS
    before = engine.launch_count()
    # the other rollouts refuse the flag
    for flags in (engine.GRAVITY | GAINS, engine.GRAVITY | engine.DAMPING | engine.IMPLICIT_DAMPING | GAINS):
        c = ctypes.c_float(DT)
        rcs = [
            lib.drmb200_forward_dynamics_rollout(topo, P(table), P(q0), P(qd0), P(f), 4, 3, c, flags, P(out), P(out), None, s),
            lib.drmb200_forward_dynamics_rollout_backward(topo, P(table), P(q0), P(qd0), P(f), 4, 3, c, flags, P(out), P(out),
                                                          P(f), None, None, P(out[0]), None, None, None, P(ws), s),
            lib.drmb200_contact_rollout(topo, 1, links, P(table), P(q0), P(qd0), P(f), None, None, 4, 3, c, flags, 1, 0.0, 0.0,
                                        P(out), P(out), None, None, None, P(solved), s),
        ]
        assert rcs == [EINVAL] * len(rcs), (flags, rcs)
    # the PD rollout needs a finite dt > 0 with it
    for dt in (0.0, -1e-3, float("nan"), float("inf")):
        c = ctypes.c_float(dt)
        rcs = [
            lib.drmb200_pd_rollout(topo, P(table), P(q0), P(qd0), P(f), None, None, P(kp), P(kp), 0, None, 4, 3, c,
                                   engine.GRAVITY | GAINS, P(out), P(out), None, P(out), s),
            lib.drmb200_pd_rollout_backward(topo, P(table), P(q0), P(qd0), P(f), None, None, P(kp), P(kp), 0, None, 4, 3, c,
                                            engine.GRAVITY | GAINS, P(out), P(out), P(out), P(f), None, None, None, P(out[0]),
                                            None, None, None, None, None, None, None, P(ws), s),
        ]
        assert rcs == [EINVAL] * len(rcs), (dt, rcs)
    assert engine.launch_count() == before
    # and runs with it
    rc = lib.drmb200_pd_rollout(topo, P(table), P(q0), P(qd0), P(f), None, None, P(kp), P(kp), 0, None, 4, 3,
                                ctypes.c_float(DT), engine.GRAVITY | GAINS, P(out), P(out), None, P(out), s)
    assert rc == 0


def test_gain_tuning_example_from_gains_the_explicit_step_cannot_run():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import tune_pd_gains_iiwa as ex
    hist, kp, kd = ex.run(batch=128, steps=100, iters=40, log=lambda *_: None, implicit_gains=True)
    print(f"tune_pd_gains_iiwa --implicit-gains, from w = 2000 rad/s: cost {hist[0]:.4g} -> {hist[-1]:.4g}")
    assert np.isfinite(hist).all() and hist[-1] < 0.5 * hist[0], (hist[0], hist[-1])
    assert bool((kp > 0).all() and (kd > 0).all())
