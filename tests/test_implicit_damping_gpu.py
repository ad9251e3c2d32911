"""GPU: implicit joint damping (DRMB200_IMPLICIT_DAMPING, drmb200_forward_dynamics_implicit_damping) in the single-step
forward dynamics, its adjoint and the three rollouts:

  * bit-identity of each rollout with the stepwise torch loop around compute_forward_dynamics(..., implicit_damping_dt=dt),
    on every shipped URDF and synthetic topology, both staging paths, every tile rung and every PD input layout;
  * accuracy against the fp64 restatement (tests/implicit_damping_oracle.py), symmetric and non-symmetric inertias, and
    against the reference's goldens (tests/golden/*.implicit_rollout.npz), values and gradients;
  * physics: the RNEA kernel closes each step, the damped Allegro models stay finite where the explicit step diverges,
    the held Allegro fingertips stay put, and a perturbed damping is recovered from trajectories;
  * the contract: launch counts, CUDA graphs, double backward, argument refusals in Python and at the C ABI.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
import implicit_damping_oracle as I
import synthetic_robots as SR
import test_operational_space_gpu as OSDT
from conftest import GOLDEN_DIR, URDFS, urdf_path
from differentiable_robot_model_b200 import engine
from oracle import drm_oracle as O
from test_backward_gpu import _ORACLE_PARAM, cuda, learnable_model
from test_rollout_gpu import bits, family_close, inputs, misaligned

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = 1e-3
EINVAL = -1
SYMMETRIC = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro", "allegro_hand_description_left"]
SYNTHETIC = {k: v for k, v in SR.families().items() if sum(v.doc()[1][1:]) > 0}


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_implicit"))


def stepwise(m, q0, qd0, f, dt, grav):
    q, qd = q0, qd0
    outs = ([], [], [])
    for t in range(f.shape[0]):
        qdd = m.compute_forward_dynamics(q, qd, f[t], grav, True, implicit_damping_dt=dt)
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, v in zip(outs, (q, qd, qdd)):
            lst.append(v)
    return tuple(torch.stack(lst) for lst in outs)


def pd_stepwise(m, q0, qd0, q_ref, kp, kd, dt, qd_ref=None, f=None, lim=None, grav=True):
    q, qd = q0, qd0
    outs = ([], [], [], [])
    for t in range(q_ref.shape[0]):
        ff = torch.zeros_like(q) if f is None else f[t]
        vr = torch.zeros_like(q) if qd_ref is None else qd_ref[t]
        u = ff + kp * (q_ref[t] - q) + kd * (vr - qd)
        if lim is not None:
            u = torch.clamp(u, -lim, lim)
        qdd = m.compute_forward_dynamics(q, qd, u, grav, True, implicit_damping_dt=dt)
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, v in zip(outs, (q, qd, qdd, u)):
            lst.append(v)
    return tuple(torch.stack(lst) for lst in outs)


def same(got, want, what):
    for name, a, b in zip(("q", "qd", "qdd", "tau"), got, want):
        assert torch.equal(bits(a), bits(b)), (what, name)


# ---------------------------------------------------------------------------------------------------------------------
# 1. bit-identity with the stepwise loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_rollout_is_bit_identical_to_the_stepwise_loop(stem):
    models = {"constant": drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV), "learnable": learnable_model(stem)[0]}
    with torch.no_grad():
        for kind, m in models.items():
            for batch, steps in ((1, 7), (63, 5), (65, 9)):
                q0, qd0, f = inputs(stem, batch, steps, seed=batch + steps)
                for grav in (True, False):
                    got = m.compute_forward_dynamics_rollout(q0, qd0, f, DT, grav, True, implicit_damping=True)
                    same(got, stepwise(m, q0, qd0, f, DT, grav), (kind, batch, steps, grav))
        m = models["constant"]
        for batch in (65, 20000):            # 20000 rows fill every SM: the 64-row tile where the model fits it
            q0, qd0, f = inputs(stem, batch, 4, seed=3)
            want = stepwise(m, q0, qd0, f, DT, True)
            for args in ((q0, qd0, f), (misaligned(q0), qd0, f), (q0, qd0, misaligned(f))):
                same(m.compute_forward_dynamics_rollout(*args, DT, True, True, implicit_damping=True), want, batch)


def pd_case(m, stem_or_robot, batch, steps, seed, unit_gains=False):
    """PD inputs: per-row gains kp = w^2 H_kk(q0), kd = 2 w H_kk(q0) at w = 20 rad/s (unit_gains: H_kk taken as 0.01, for
    the synthetic models whose mass-matrix kernel refuses them), a limit that binds for part of the entries."""
    robot = stem_or_robot if isinstance(stem_or_robot, O.Robot) else O.load_robot(urdf_path(stem_or_robot), torch.float32)
    q0, qd0, _ = O.sample_inputs(robot, batch, seed=seed, vel_scale=0.02)
    q0, qd0 = q0.to(DEV), qd0.clamp(-1, 1).to(DEV)
    n = q0.shape[1]
    gen = torch.Generator().manual_seed(seed)
    q_ref = (q0.cpu() + 0.1 * torch.randn(steps, batch, n, generator=gen)).to(DEV)
    qd_ref = (0.2 * torch.randn(steps, batch, n, generator=gen)).to(DEV)
    f = (0.05 * torch.randn(steps, batch, n, generator=gen)).to(DEV)
    if unit_gains:
        H = torch.full_like(q0, 0.01)
    else:
        with torch.no_grad():
            H = torch.diagonal(m.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2).clamp_min(1e-6)
    kp, kd = 400.0 * H, 40.0 * H
    lim = (8.0 * H.mean(0)).clone()
    lim[0] = float("inf")
    return q0, qd0, q_ref, qd_ref, f, kp, kd, lim


def pd_bit_identity(m, case, what):
    q0, qd0, q_ref, qd_ref, f, kp, kd, lim = case
    layouts = {"per_row": (kp, kd), "shared": (kp.mean(0), kd.mean(0)), "mixed": (kp, kd.mean(0))}
    for name, (a, b) in layouts.items():
        for opt in ({}, {"qd_ref": qd_ref}, {"f": f}, {"qd_ref": qd_ref, "f": f, "lim": lim}):
            got = m.compute_pd_controlled_rollout(q0, qd0, q_ref, a, b, DT, qd_ref=opt.get("qd_ref"), f=opt.get("f"),
                                                  effort_limit=opt.get("lim"), use_damping=True, implicit_damping=True)
            want = pd_stepwise(m, q0, qd0, q_ref, a, b, DT, opt.get("qd_ref"), opt.get("f"), opt.get("lim"))
            same(got, want, (what, name, sorted(opt)))


@pytest.mark.parametrize("stem", sorted(URDFS))
def test_pd_rollout_is_bit_identical_to_the_stepwise_loop(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    with torch.no_grad():
        for batch in (5, 65, 20000):
            pd_bit_identity(m, pd_case(m, stem, batch, 3, seed=batch), (stem, batch))
        q0, qd0, q_ref, qd_ref, f, kp, kd, lim = pd_case(m, stem, 65, 3, seed=4)
        got = m.compute_pd_controlled_rollout(misaligned(q0), qd0, q_ref, kp, kd, DT, qd_ref=qd_ref, f=misaligned(f),
                                              effort_limit=lim, use_damping=True, implicit_damping=True)
        same(got, pd_stepwise(m, q0, qd0, q_ref, kp, kd, DT, qd_ref, f, lim), "misaligned")


@pytest.mark.parametrize("name", sorted(SYNTHETIC))
def test_rollouts_on_synthetic_topologies_are_bit_identical_to_the_stepwise_loop(name, model_dir):
    path = SR.build(SYNTHETIC[name], model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    robot = O.load_robot(path, torch.float32)
    with torch.no_grad():
        for batch in (33, 4000):
            q0, qd0, _ = O.sample_inputs(robot, batch, seed=batch, vel_scale=0.02)
            q0, qd0 = q0.to(DEV), qd0.clamp(-1, 1).to(DEV)
            f = 0.05 * torch.randn(3, batch, robot.n_dofs, generator=torch.Generator().manual_seed(1)).to(DEV)
            for grav in (True, False):
                got = m.compute_forward_dynamics_rollout(q0, qd0, f, DT, grav, True, implicit_damping=True)
                same(got, stepwise(m, q0, qd0, f, DT, grav), (name, batch, grav))
        # the PD rollout, with per-row gains and every stream: F_chain64 takes the 16-row rung there
        pd_bit_identity(m, pd_case(m, robot, 40, 2, seed=2, unit_gains=True), name)


# ---------------------------------------------------------------------------------------------------------------------
# 2. accuracy: single step and rollouts against the fp64 restatement and the reference
# ---------------------------------------------------------------------------------------------------------------------
def nonsym_robot(stem, seed=17):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    gen = torch.Generator().manual_seed(seed)
    scale = robot.inertia.abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-6)
    robot.inertia = (robot.inertia + 0.05 * scale * torch.randn(robot.inertia.shape, generator=gen, dtype=torch.float64)).float().double()
    return robot


@pytest.mark.parametrize("nonsym", [False, True])
@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "trifinger_edu", "allegro_hand_description_left"])
def test_single_step_matches_fp64_restatement(stem, nonsym):
    robot = nonsym_robot(stem) if nonsym else O.load_robot(urdf_path(stem), torch.float64)
    gen = torch.Generator().manual_seed(5)
    robot.damping = robot.damping + 0.2 * torch.rand(robot.damping.shape, generator=gen, dtype=torch.float64).float().double()
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    table = O.link_table(robot.to(torch.float32)).float().to(DEV).contiguous()
    q, qd, f = O.sample_inputs(robot.to(torch.float32), 512, seed=9)
    for grav in (0, 1):
        for h in (1e-4, 1e-3, 1e-2):
            got = engine.forward_dynamics_raw(m._topology, table, q.to(DEV), qd.to(DEV), f.to(DEV),
                                              grav | engine.DAMPING, implicit_dt=h)
            want = I.forward_dynamics(robot, q.double(), qd.double(), f.double(), bool(grav), True, h)
            o32 = I.forward_dynamics(robot.to(torch.float32), q, qd, f, bool(grav), True, h)
            scale = want.abs().amax(1, keepdim=True).clamp_min(1e-6)
            err = float(((got.cpu().double() - want).abs() / scale).max())
            e32 = float(((o32.double() - want).abs() / scale).max())
            assert err <= max(8 * e32, 1e-5), (grav, h, err, e32)


@pytest.mark.parametrize("stem", SYMMETRIC)
def test_rollout_matches_reference_trajectories_and_gradients(stem):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".implicit_rollout.npz"), allow_pickle=False)
    dt = float(g["dt"])
    # family-relative: the goldens are the reference's fp32 autograd through a dense solve per step, whose own distance
    # from the fp64 restatement reaches 3.4e-3 of the q0 family on iiwa7_allegro and 3.3e-4 elsewhere
    tol = 5e-3 if stem == "iiwa7_allegro" else 5e-4
    const = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    for tag in ("g1d1", "g0d1"):
        grav = tag == "g1d1"
        with torch.no_grad():
            traj = const.compute_forward_dynamics_rollout(cuda(g["q0"]), cuda(g["qd0"]), cuda(g["f"]), dt, grav, True,
                                                          implicit_damping=True)
        for name, got in zip(("q", "qd", "qdd"), traj):
            want = g[f"{tag}.{name}"]
            scale = np.abs(want).max(axis=2, keepdims=True)
            rel = (np.abs(got.cpu().numpy() - want) / (scale + 1e-6)).max()
            assert rel < 2e-3, (tag, name, rel)
        m, params = learnable_model(stem)
        q0, qd0, f = cuda(g["q0"], True), cuda(g["qd0"], True), cuda(g["f"], True)
        traj = m.compute_forward_dynamics_rollout(q0, qd0, f, dt, grav, True, implicit_damping=True)
        sum((cuda(g[f"G_{k}"]) * v).sum() for k, v in zip(("q", "qd", "qdd"), traj)).backward()
        prefix = f"{tag}.grad."
        worst = 0.0
        for key, t in (("q0", q0), ("qd0", qd0), ("f", f)):
            worst = max(worst, family_close(t.grad.cpu().numpy(), g[prefix + key], tol, f"{tag}.{key}"))
        damping_checked = False
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in ("q0", "qd0", "f"):
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
            damping_checked |= pname == "joint_damping"
        assert damping_checked
        print(f"{stem} {tag}: worst family-relative gradient error vs reference {worst:.2e}")


def _grads(m, params, fn, ins, G):
    for p in params.values():
        p.grad = None
    ins = [t.detach().clone().requires_grad_(True) for t in ins]
    out = fn(m, *ins)
    out = out if isinstance(out, tuple) else (out,)
    sum((w * v).sum() for w, v in zip(G, out)).backward()
    return [t.grad for t in ins] + [torch.zeros_like(p) if p.grad is None else p.grad.clone() for p in params.values()]


def compare_by_kind(got, want, params, n_inputs, tol, what):
    """Each input and each link-parameter kind against the largest entry of its family in `want`."""
    kinds = [f"input{j}" for j in range(n_inputs)] + [pname for (_, pname) in params]
    for kind in dict.fromkeys(kinds):
        idx = [j for j, k in enumerate(kinds) if k == kind]
        fam = max(float(want[j].abs().max()) for j in idx)
        for j in idx:
            err = float((got[j] - want[j]).abs().max())
            assert err <= tol * max(fam, 1e-30), (what, kind, j, err, fam)


def compare_with_oracle(stem, got, loss_of_robot, ins, params, tol=1e-4, nonsym=False):
    robot = nonsym_robot(stem) if nonsym else O.load_robot(urdf_path(stem), torch.float64)
    names = ("trans", "rpy", "mass", "com", "inertia", "damping")
    for name in names:
        setattr(robot, name, getattr(robot, name).detach().clone().requires_grad_(True))
    dins = [t.detach().cpu().double().requires_grad_(True) for t in ins]
    want = torch.autograd.grad(loss_of_robot(robot, *dins), dins + [getattr(robot, nm) for nm in names], allow_unused=True)
    by = dict(zip(names, want[len(ins):]))
    worst = 0.0
    for a, b in zip(got[:len(ins)], want[:len(ins)]):
        worst = max(worst, family_close(a.cpu().numpy(), b.numpy(), tol, "input"))
    for ((i, pname), p), gp in zip(params.items(), got[len(ins):]):
        w = by[_ORACLE_PARAM[pname]]
        w = torch.zeros_like(getattr(robot, _ORACLE_PARAM[pname])) if w is None else w
        fam = float(w.abs().max())
        err = float((gp.cpu().double() - w[i]).abs().max())
        assert err <= tol * max(fam, 1e-30), (pname, i, err, fam)
        worst = max(worst, err / max(fam, 1e-30))
    return worst


@pytest.mark.parametrize("stem,nonsym", [("iiwa7", False), ("iiwa7", True), ("trifinger_edu", True),
                                         ("allegro_hand_description_left", False)])
def test_single_step_gradients_match_fp64_oracle_autograd(stem, nonsym):
    m, params = learnable_model(stem)
    if nonsym:
        robot = nonsym_robot(stem)
        with torch.no_grad():
            for (i, pname), p in params.items():
                if pname == "inertia_mat":
                    p.copy_(robot.inertia[i].float().to(DEV))
    robot32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f = (t.to(DEV) for t in O.sample_inputs(robot32, 300, seed=13))
    G = torch.randn(300, robot32.n_dofs, generator=torch.Generator().manual_seed(14))
    h = 1e-3
    got = _grads(m, params, lambda mm, a, b, c: mm.compute_forward_dynamics(a, b, c, True, True, implicit_damping_dt=h),
                 (q, qd, f), [G.to(DEV)])
    worst = compare_with_oracle(stem, got, lambda r, a, b, c: (G.double() * I.forward_dynamics(r, a, b, c, True, True, h)).sum(),
                                (q, qd, f), params, nonsym=nonsym)
    print(f"{stem} nonsym={nonsym}: worst family-relative single-step gradient error vs fp64 oracle {worst:.2e}")


@pytest.mark.parametrize("stem,batch,steps", [("iiwa7", 300, 12), ("trifinger_edu", 64, 8), ("allegro_hand_description_left", 40, 8)])
def test_rollout_gradients_match_stepwise_loop_and_fp64_oracle(stem, batch, steps):
    m, params = learnable_model(stem)
    q0, qd0, f = inputs(stem, batch, steps, seed=11)
    gen = torch.Generator().manual_seed(12)
    G = [torch.randn(steps, batch, m._n_dofs, generator=gen) for _ in range(3)]
    Gd = [x.to(DEV) for x in G]
    fused = _grads(m, params, lambda mm, a, b, c: mm.compute_forward_dynamics_rollout(a, b, c, DT, True, True, implicit_damping=True),
                   (q0, qd0, f), Gd)
    loop = _grads(m, params, lambda mm, a, b, c: stepwise(mm, a, b, c, DT, True), (q0, qd0, f), Gd)
    compare_by_kind(fused, loop, params, 3, 1e-4, "stepwise")
    worst = compare_with_oracle(stem, fused, lambda r, a, b, c: sum((w.double() * v).sum() for w, v in
                                                                   zip(G, I.forward_dynamics_rollout(r, a, b, c, DT, True))),
                                (q0, qd0, f), params)
    print(f"{stem}: worst family-relative rollout gradient error vs fp64 oracle {worst:.2e}")


@pytest.mark.parametrize("stem", ["iiwa7", "allegro_hand_description_left"])
def test_pd_rollout_gradients_match_stepwise_loop_and_fp64_oracle(stem):
    m, params = learnable_model(stem)
    with torch.no_grad():
        q0, qd0, q_ref, qd_ref, f, kp, kd, lim = pd_case(m, stem, 64, 6, seed=21)
    gen = torch.Generator().manual_seed(22)
    G = [torch.randn(6, 64, m._n_dofs, generator=gen) for _ in range(4)]
    Gd = [x.to(DEV) for x in G]
    ins = (q0, qd0, q_ref, qd_ref, f, kp, kd)

    def fused_fn(mm, *a):
        return tuple(mm.compute_pd_controlled_rollout(a[0], a[1], a[2], a[5], a[6], DT, qd_ref=a[3], f=a[4], effort_limit=lim,
                                                      use_damping=True, implicit_damping=True))

    fused = _grads(m, params, fused_fn, ins, Gd)
    loop = _grads(m, params, lambda mm, *a: pd_stepwise(mm, a[0], a[1], a[2], a[5], a[6], DT, a[3], a[4], lim), ins, Gd)
    compare_by_kind(fused, loop, params, len(ins), 1e-4, "stepwise")
    lim64 = lim.cpu().double()

    def oracle_loss(r, *a):
        out = I.pd_rollout(r, a[0], a[1], a[2], a[5], a[6], DT, a[3], a[4], lim64)
        return sum((w.double() * v).sum() for w, v in zip(G, out))

    worst = compare_with_oracle(stem, fused, oracle_loss, ins, params)
    print(f"{stem}: worst family-relative PD rollout gradient error vs fp64 oracle {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. the contact rollout
# ---------------------------------------------------------------------------------------------------------------------
CONTACT = [("iiwa7", ["iiwa_link_ee"], False), ("allegro_hand_description_left", OSDT.TIPS, True)]


@pytest.mark.parametrize("stem,names,pos", CONTACT)
def test_contact_rollout_matches_fp64_restatement(stem, names, pos):
    m = OSDT.model_of(stem)
    r64 = O.load_robot(urdf_path(stem), torch.float64)
    q0, qd0, _ = O.sample_inputs(O.load_robot(urdf_path(stem), torch.float32), 16, seed=31)
    qd0 = 0.2 * qd0
    T = 8
    f = 0.1 * torch.randn(T, 16, q0.shape[1], generator=torch.Generator().manual_seed(32))
    omega = 0.2 / DT
    with torch.no_grad():
        got = m.compute_contact_rollout(q0.to(DEV), qd0.to(DEV), f.to(DEV), names, DT, stabilization=omega, use_damping=True,
                                        position_only=pos, implicit_damping=True)
    want = I.contact_rollout(r64, q0.double(), qd0.double(), f.double(), names, DT, omega, position_only=pos)
    o32 = I.contact_rollout(r64.to(torch.float32), q0, qd0, f, names, DT, omega, position_only=pos)
    rows = got.solved.cpu() & want[4] & o32[4]
    assert int(rows.sum()) >= 12, int(rows.sum())
    for i, k in enumerate(("q", "qd", "qdd", "force")):
        g = getattr(got, k).cpu().double()[:, rows]
        w, w32 = want[i][:, rows], o32[i][:, rows].double()
        scale = w.abs().amax(-1, keepdim=True).clamp_min(1e-30)
        err = float(((g - w).abs() / scale).max())
        e32 = float(((w32 - w).abs() / scale).max())
        bound = max(8 * e32, 1e-5 if k in ("q", "qd") else 2e-4)
        print(f"{stem} {k}: {err:.2e} vs fp64 (fp32 restatement {e32:.2e})")
        assert err <= bound, (k, err, bound)


def test_held_allegro_fingertips_stay_finite_with_damping():
    m = OSDT.model_of("allegro_hand_description_left")
    robot = O.load_robot(urdf_path("allegro_hand_description_left"), torch.float32)
    q0, _, _ = O.sample_inputs(robot, 4096, seed=41)
    q0, qd0 = q0.to(DEV), torch.zeros_like(q0).to(DEV)
    T = 256
    f = torch.zeros(T, 4096, robot.n_dofs, device=DEV)
    with torch.no_grad():
        out = m.compute_contact_rollout(q0, qd0, f, OSDT.TIPS, DT, stabilization=0.2 / DT, use_damping=True,
                                        position_only=True, implicit_damping=True)
        p0 = torch.stack([m.compute_forward_kinematics(q0, nm)[0] for nm in OSDT.TIPS])
        p1 = torch.stack([m.compute_forward_kinematics(out.q[-1], nm)[0] for nm in OSDT.TIPS])
    solved = out.solved
    finite = torch.isfinite(out.q).all(2).all(0)
    share = float((solved & finite).float().mean())
    drift = (p1 - p0).norm(dim=2).amax(0)[solved & finite]
    print(f"Allegro tips held, implicit damping, dt = 1 ms, T = {T}: {share:.4f} of rows finite and solved, "
          f"tip drift median {float(drift.median()):.2e} m, max {float(drift.max()):.2e} m")
    assert bool((finite | ~solved).all())                      # an unsolved row is NaN by definition, a solved one finite
    assert share >= 0.9
    assert float(drift.max()) < 1e-2


# ---------------------------------------------------------------------------------------------------------------------
# 4. physics
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "trifinger_edu", "allegro_hand_description_left"])
def test_inverse_dynamics_closes_the_implicit_step(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    q0, qd0, f = inputs(stem, 512, 6, seed=51)
    d = I.damping_vector(O.load_robot(urdf_path(stem), torch.float32)).to(DEV)
    with torch.no_grad():
        for grav in (True, False):
            q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, f, DT, grav, True, implicit_damping=True)
            qs, qds = torch.cat([q0[None], q[:-1]]), torch.cat([qd0[None], qd[:-1]])
            for t in range(f.shape[0]):
                tau = m.compute_inverse_dynamics(qs[t], qds[t], qdd[t], grav, use_damping=False)
                closed = tau + d * qd[t]
                scale = (tau.abs() + (d * qd[t]).abs() + f[t].abs()).amax(1, keepdim=True).clamp_min(1e-3)
                err = float(((closed - f[t]).abs() / scale).max())
                assert err < 2e-3, (grav, t, err)


@pytest.mark.parametrize("stem", ["allegro_hand_description_left", "iiwa7_allegro"])
def test_damped_allegro_at_rest_stays_bounded_where_the_explicit_step_diverges(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q0, _, _ = O.sample_inputs(robot, 64, seed=61)
    q0 = q0.to(DEV)
    qd0 = torch.zeros_like(q0)
    with torch.no_grad():
        explicit = m.compute_forward_dynamics_rollout(q0, qd0, torch.zeros(10, 64, robot.n_dofs, device=DEV), DT, True, True)
        blown = (~torch.isfinite(explicit[1])).any(2).any(0)
        print(f"{stem}: explicit damped rollout non-finite within 10 steps on {int(blown.sum())} of 64 rows")
        assert bool(blown.all())                                 # today's documented behaviour: the premise
        T = 1000
        q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, torch.zeros(T, 64, robot.n_dofs, device=DEV), DT, True, True,
                                                        implicit_damping=True)
    assert bool(torch.isfinite(q).all() and torch.isfinite(qd).all())
    peak = float(qd.abs().max())
    print(f"{stem}: implicit damped rollout T = {T}: max |qd| {peak:.3g} rad/s, final max |qd| {float(qd[-1].abs().max()):.3g}")
    assert peak < 100.0                                          # the arm of iiwa7_allegro falls under gravity: 54 rad/s


def test_learning_link_damping_from_implicit_rollouts():
    from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar
    stem = "allegro_hand_description_left"
    gt = drm.DifferentiableRobotModel(urdf_path(stem), "gt", device=DEV)
    m = drm.DifferentiableRobotModel(urdf_path(stem), "learn", device=DEV)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    link = robot.controlled[2]
    true = float(robot.damping[link])
    m.make_link_param_learnable(robot.names[link], "joint_damping", UnconstrainedScalar(init_val=torch.tensor([0.5 * true])))
    q0, qd0, _ = O.sample_inputs(robot, 256, seed=71, vel_scale=0.2)
    q0, qd0 = q0.to(DEV), qd0.to(DEV)
    f = 0.05 * torch.randn(50, 256, robot.n_dofs, generator=torch.Generator().manual_seed(72)).to(DEV)
    with torch.no_grad():
        target = gt.compute_forward_dynamics_rollout(q0, qd0, f, DT, True, True, implicit_damping=True)[1]
    opt = torch.optim.Adam(m.parameters(), lr=0.3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.98)
    for _ in range(300):
        opt.zero_grad()
        qd = m.compute_forward_dynamics_rollout(q0, qd0, f, DT, True, True, implicit_damping=True)[1]
        loss = ((qd - target) ** 2).mean()
        loss.backward()
        opt.step()
        sched.step()
    learned = float(m._bodies[link].get_joint_damping_const())
    print(f"damping of {robot.names[link]}: true {true:.4g}, start {0.5 * true:.4g}, learned {learned:.4g}")
    assert abs(learned - true) < 0.02 * true


# ---------------------------------------------------------------------------------------------------------------------
# 5. the contract
# ---------------------------------------------------------------------------------------------------------------------
def test_launch_counts_graph_capture_and_double_backward():
    m, params = learnable_model("iiwa7")
    q0, qd0, f = inputs("iiwa7", 1000, 25, seed=2)
    const = drm.DifferentiableKUKAiiwa(device=DEV)
    const.compute_forward_dynamics_rollout(q0, qd0, f, DT, True, True, implicit_damping=True)
    x = pd_case(const, "iiwa7", 1000, 25, seed=3)
    before = engine.launch_count()
    with torch.no_grad():
        const.compute_forward_dynamics_rollout(q0, qd0, f, DT, True, True, implicit_damping=True)
        mid = engine.launch_count()
        const.compute_pd_controlled_rollout(x[0], x[1], x[2], x[5], x[6], DT, qd_ref=x[3], f=x[4], effort_limit=x[7],
                                            use_damping=True, implicit_damping=True)
    assert mid - before == 1 and engine.launch_count() - mid == 1
    qa = q0.clone().requires_grad_(True)
    q, qd, qdd = const.compute_forward_dynamics_rollout(qa, qd0, f, DT, True, True, implicit_damping=True)
    before = engine.launch_count()
    (q.sum() + qd.sum() + qdd.sum()).backward()
    assert engine.launch_count() - before == 2 * f.shape[0] + 1          # no table gradient: no reduction
    with torch.no_grad():
        m.compute_forward_dynamics_rollout(q0, qd0, f, DT, True, True, implicit_damping=True)
    q, qd, qdd = m.compute_forward_dynamics_rollout(qa, qd0, f, DT, True, True, implicit_damping=True)
    before = engine.launch_count()
    (q.sum() + qd.sum() + qdd.sum()).backward()
    assert engine.launch_count() - before <= 2 * f.shape[0] + 2 + 4     # 2T + 2, the rest the table build's backward
    # double backward raises, for the single step and the rollout
    for fn in (lambda a: const.compute_forward_dynamics(a, qd0[:8], f[0, :8], True, True, implicit_damping_dt=DT),
               lambda a: const.compute_forward_dynamics_rollout(a, qd0[:8], f[:3, :8], DT, True, True, implicit_damping=True)[0]):
        a = q0[:8].clone().requires_grad_(True)
        out = fn(a)
        (g,) = torch.autograd.grad(out.sum(), a, create_graph=True)
        with pytest.raises(RuntimeError, match="second-order"):
            g.sum().backward()
    # forward and backward captured in one CUDA graph
    m.fuse_learnable_parameters()
    flat = m.fused_link_params.flat
    q0, qd0, f = inputs("iiwa7", 777, 9, seed=9)
    G = torch.randn(9, 777, 7, generator=torch.Generator().manual_seed(3)).to(DEV)
    fa = f.clone().requires_grad_(True)

    def step():
        q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, fa, DT, True, True, implicit_damping=True)
        ((q + qd + qdd) * G).sum().backward()
        return q

    flat.grad, fa.grad = None, None
    eager = [step().detach().clone(), flat.grad.clone(), fa.grad.clone()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            flat.grad, fa.grad = None, None
            step()
    torch.cuda.current_stream().wait_stream(side)
    flat.grad = torch.zeros_like(flat)
    fa.grad = torch.zeros_like(fa)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        q = step()
    flat.grad.zero_()
    fa.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(q, eager[0]) and torch.equal(flat.grad, eager[1]) and torch.equal(fa.grad, eager[2])


def test_argument_refusals():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    q0, qd0, f = inputs("iiwa7", 4, 3, seed=1)
    kp = torch.ones(7, device=DEV)
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics(q0, qd0, f[0], True, False, implicit_damping_dt=DT)
    for bad in (0.0, -1e-3, float("inf"), float("nan")):
        with pytest.raises(AssertionError):
            m.compute_forward_dynamics(q0, qd0, f[0], True, True, implicit_damping_dt=bad)
        with pytest.raises(AssertionError):
            m.compute_forward_dynamics_rollout(q0, qd0, f, bad, True, True, implicit_damping=True)
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_rollout(q0, qd0, f, DT, True, False, implicit_damping=True)
    with pytest.raises(AssertionError):
        m.compute_pd_controlled_rollout(q0, qd0, f, kp, kp, DT, use_damping=False, implicit_damping=True)
    with pytest.raises(AssertionError):
        m.compute_contact_rollout(q0, qd0, f, ["iiwa_link_ee"], DT, use_damping=False, implicit_damping=True)
    # the C ABI: EINVAL without DRMB200_DAMPING or without a finite dt > 0, before any launch
    lib, topo, table = engine.lib(), ctypes.byref(m._topology), m._link_table().detach()
    out = torch.empty(3, 4, 7, device=DEV)
    P = engine._ptr
    s = engine._stream()
    ws = torch.empty(1 << 22, device=DEV)
    links = (ctypes.c_int32 * 1)(m._topology.n_links - 1)
    solved = torch.empty(4, dtype=torch.uint8, device=DEV)
    IMP = engine.IMPLICIT_DAMPING
    before = engine.launch_count()
    for flags, dt in ((engine.GRAVITY | IMP, DT), (engine.GRAVITY | engine.DAMPING | IMP, 0.0),
                      (engine.GRAVITY | engine.DAMPING | IMP, float("nan")), (engine.GRAVITY | engine.DAMPING | IMP, float("inf"))):
        c = ctypes.c_float(dt)
        rcs = [
            lib.drmb200_forward_dynamics_implicit_damping(topo, P(table), P(q0), P(qd0), P(f[0]), 4, flags, c, P(out[0]), s),
            lib.drmb200_forward_dynamics_implicit_damping_backward(topo, P(table), P(q0), P(qd0), P(f[0]), 4, flags, c, P(f[0]),
                                                                   P(out[0]), None, None, None, P(ws), s),
            lib.drmb200_forward_dynamics_rollout(topo, P(table), P(q0), P(qd0), P(f), 4, 3, c, flags, P(out), P(out), None, s),
            lib.drmb200_forward_dynamics_rollout_backward(topo, P(table), P(q0), P(qd0), P(f), 4, 3, c, flags, P(out), P(out),
                                                          P(f), None, None, P(out[0]), None, None, None, P(ws), s),
            lib.drmb200_pd_rollout(topo, P(table), P(q0), P(qd0), P(f), None, None, P(kp), P(kp), 0, None, 4, 3, c, flags,
                                   P(out), P(out), None, P(out), s),
            lib.drmb200_pd_rollout_backward(topo, P(table), P(q0), P(qd0), P(f), None, None, P(kp), P(kp), 0, None, 4, 3, c,
                                            flags, P(out), P(out), P(out), P(f), None, None, None, P(out[0]), None, None, None,
                                            None, None, None, None, P(ws), s),
            lib.drmb200_contact_rollout(topo, 1, links, P(table), P(q0), P(qd0), P(f), None, None, 4, 3, c, flags, 1, 0.0, 0.0,
                                        P(out), P(out), None, None, None, P(solved), s),
        ]
        assert rcs == [EINVAL] * len(rcs), (flags, dt, rcs)
    assert engine.launch_count() == before
    # the single-step entry implies DRMB200_IMPLICIT_DAMPING: DRMB200_DAMPING alone is enough
    rc = lib.drmb200_forward_dynamics_implicit_damping(topo, P(table), P(q0), P(qd0), P(f[0]), 4, engine.DAMPING,
                                                       ctypes.c_float(DT), P(out[0]), s)
    assert rc == 0
