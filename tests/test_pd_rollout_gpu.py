"""GPU: PD-controlled rollouts (csrc/rollout.cu) -- a diagonal joint-space PD law around T semi-implicit Euler steps of
the articulated-body kernel in one launch, and its adjoint stepped backwards in time:

  * zero gains without a limit reproduce the open-loop rollout bit for bit;
  * bit-identity with the Python loop `u = f + kp * (q_ref - q) + kd * (qd_ref - qd); u = clamp(u, -lim, lim)` followed by
    compute_forward_dynamics and the integrate, for every input combination, shared, per-row and mixed gains and both staging paths;
  * trajectories and gradients against the reference's own loop (tests/golden/*.pd_rollout.npz);
  * gradients against autograd through the same GPU loop and against the fp64 oracle;
  * reproducibility, launch counts, edge cases, CUDA graphs, learning and gain tuning.

Gradient tolerances are family-relative (each input and every link-parameter kind against the largest entry of its
family), 1e-4 as in test_rollout_gpu.py.
"""
import itertools
import os
import sys

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from conftest import GOLDEN_DIR, REPO, URDFS, urdf_path
from test_backward_gpu import _ORACLE_PARAM, cuda, learnable_model
from test_rollout_gpu import ARMS, FLAGS, bits, family_close, inputs, misaligned
from differentiable_robot_model_b200 import engine
from oracle import drm_oracle as O
from pd_rollout_oracle import pd_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = ("q", "qd", "qdd", "tau")
DIFF = ("q0", "qd0", "q_ref", "qd_ref", "f", "kp", "kd")


def stepwise(model, q0, qd0, q_ref, kp, kd, dt, qd_ref=None, f=None, lim=None, grav=True, damp=False):
    """The PD loop of compute_pd_controlled_rollout's docstring, one torch op per rounding."""
    q, qd = q0, qd0
    outs = ([], [], [], [])
    for t in range(q_ref.shape[0]):
        ff = torch.zeros_like(q) if f is None else f[t]
        vr = torch.zeros_like(q) if qd_ref is None else qd_ref[t]
        u = ff + kp * (q_ref[t] - q) + kd * (vr - qd)
        if lim is not None:
            u = torch.clamp(u, -lim, lim)
        qdd = model.compute_forward_dynamics(q, qd, u, grav, damp)
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, v in zip(outs, (q, qd, qdd, u)):
            lst.append(v)
    return tuple(torch.stack(lst) for lst in outs)


def pd_inputs(model, stem, batch, steps, seed, w=20.0):
    """q0, qd0, f as test_rollout_gpu.inputs; q_ref near q0, qd_ref small; per-row gains kp = w^2 H_kk(q0),
    kd = 2 w H_kk(q0) (stable explicit Euler on light links); a limit that binds for part of the entries, inf on joint 0."""
    q0, qd0, f = inputs(stem, batch, steps, seed)
    gen = torch.Generator().manual_seed(seed + 1000)
    n = q0.shape[1]
    q_ref = q0 + 0.1 * torch.randn(steps, batch, n, generator=gen).to(DEV)
    qd_ref = 0.2 * torch.randn(steps, batch, n, generator=gen).to(DEV)
    with torch.no_grad():
        H = torch.diagonal(model.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2).clamp_min(1e-6)
    kp, kd = (w * w) * H, (2 * w) * H
    lim = (0.02 * w * w * H.mean(0)).clone()
    lim[0] = float("inf")
    return dict(q0=q0, qd0=qd0, q_ref=q_ref, qd_ref=qd_ref, f=f, kp=kp, kd=kd, lim=lim)


def call(m, x, dt, grav=True, damp=False, **over):
    a = dict(x, **over)
    return m.compute_pd_controlled_rollout(a["q0"], a["qd0"], a["q_ref"], a["kp"], a["kd"], dt, qd_ref=a["qd_ref"], f=a["f"],
                                           effort_limit=a["lim"], include_gravity=grav, use_damping=damp)


def loop(m, x, dt, grav=True, damp=False, **over):
    a = dict(x, **over)
    return stepwise(m, a["q0"], a["qd0"], a["q_ref"], a["kp"], a["kd"], dt, a["qd_ref"], a["f"], a["lim"], grav, damp)


GAINS = ("shared", "row", "kp_row", "kd_row")     # both [n], both [B, n], kp [B, n] with kd [n], kp [n] with kd [B, n]


def gains(x, layout):
    """kp / kd of pd_inputs (per row) in one of the GAINS layouts; a shared gain is the mean over rows."""
    kp_row, kd_row = layout in ("row", "kp_row"), layout in ("row", "kd_row")
    return dict(kp=x["kp"] if kp_row else x["kp"].mean(0), kd=x["kd"] if kd_row else x["kd"].mean(0))


# ---------------------------------------------------------------------------------------------------------------------
# 1. zero gains: the open-loop rollout
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", ["iiwa7", "panda", "trifinger_edu", "allegro_hand_description_left"])
def test_zero_gains_reproduce_the_open_loop_rollout(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    with torch.no_grad():
        for batch, shared in ((65, True), (1000, False)):
            x = pd_inputs(m, stem, batch, 9, seed=batch)
            zero = torch.zeros_like(x["kp"][0] if shared else x["kp"])
            for grav, damp in FLAGS:
                got = call(m, x, 1e-3, grav, damp, kp=zero, kd=zero, qd_ref=None, lim=None)
                want = m.compute_forward_dynamics_rollout(x["q0"], x["qd0"], x["f"], 1e-3, grav, damp)
                for name, a, b in zip(KEYS, got, want):
                    assert torch.equal(bits(a), bits(b)), (batch, grav, damp, name)
                finite = torch.cat([x["q0"][None], got.q[:-1]]).isfinite() & torch.cat([x["qd0"][None], got.qd[:-1]]).isfinite()
                assert torch.equal(got.tau[finite], x["f"][finite])


# ---------------------------------------------------------------------------------------------------------------------
# 2. bit-identity with the stepwise loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_pd_rollout_is_bit_identical_to_the_stepwise_loop(stem):
    models = {"constant": drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV), "learnable": learnable_model(stem)[0]}
    dt, steps = 2.0 ** -10, 7
    combos = list(itertools.product(GAINS, (False, True), (False, True), (False, True)))   # gains, qd_ref, f, effort limit
    with torch.no_grad():
        for kind, m in models.items():
            for batch in (1, 63, 65, 1000):
                x = pd_inputs(m, stem, batch, steps, seed=batch + steps)
                for i, (layout, has_qdr, has_f, has_lim) in enumerate(combos):
                    grav, damp = FLAGS[(i + batch) % 4]
                    over = dict(gains(x, layout), qd_ref=x["qd_ref"] if has_qdr else None, f=x["f"] if has_f else None,
                                lim=x["lim"] if has_lim else None)
                    got = call(m, x, dt, grav, damp, **over)
                    want = loop(m, x, dt, grav, damp, **over)
                    for name, a, b in zip(KEYS, got, want):
                        assert torch.equal(bits(a), bits(b)), (kind, batch, layout, has_qdr, has_f, has_lim, grav, damp, name)
        # aligned bases (TMA bulk copies) and unaligned ones of every new input (cooperative copies), at a batch of 32-row
        # tiles and one that takes the 64-row tile on the Kuka (a batch that gives every SM a CTA; the model's shared
        # memory leaves room for two)
        m = models["constant"]
        for batch in (65, 20000):
            x = pd_inputs(m, stem, batch, 5, seed=3)
            want = loop(m, x, 1e-3, True, True)
            for name in (None, "q0", "q_ref", "qd_ref", "f", "kp", "kd"):
                got = call(m, x, 1e-3, True, True, **({} if name is None else {name: misaligned(x[name])}))
                for a, b in zip(got, want):
                    assert torch.equal(bits(a), bits(b)), (batch, name)


# ---------------------------------------------------------------------------------------------------------------------
# 3. reference goldens
# ---------------------------------------------------------------------------------------------------------------------
GOLDEN_STEMS = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro"]


@pytest.mark.parametrize("stem", GOLDEN_STEMS)
def test_pd_rollout_matches_reference_trajectories_and_gradients(stem):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".pd_rollout.npz"), allow_pickle=False)
    dt = float(g["dt"])
    tol = 1e-4
    tags = sorted({k.split(".")[0] for k in g.files if k.startswith("g1d")})
    const = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    lim = cuda(g["effort_limit"])
    for tag in tags:
        damp = tag == "g1d1"
        x = {k: cuda(g[k]) for k in DIFF}
        x["lim"] = lim
        with torch.no_grad():
            traj = call(const, x, dt, True, damp)
        for name, got in zip(KEYS, traj):
            want = g[f"{tag}.{name}"]
            scale = np.abs(want).max(axis=2, keepdims=True)
            rel = (np.abs(got.cpu().numpy() - want) / (scale + 1e-6)).max()
            assert rel < (2e-4 if stem in ARMS else 2e-3), (tag, name, rel)
        m, params = learnable_model(stem)
        x = {k: cuda(g[k], True) for k in DIFF}
        x["lim"] = lim
        traj = call(m, x, dt, True, damp)
        sum((cuda(g[f"G_{k}"]) * v).sum() for k, v in zip(KEYS, traj)).backward()
        prefix = f"{tag}.grad."
        worst = 0.0
        for key in DIFF:
            worst = max(worst, family_close(x[key].grad.cpu().numpy(), g[prefix + key], tol, f"{tag}.{key}"))
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in DIFF:
                continue
            pname, idx = key[len(prefix):].rsplit(".", 1)
            p = params[(int(idx), pname)]
            got = torch.zeros_like(p) if p.grad is None else p.grad
            fam = max(np.abs(g[k]).max() for k in g.files if k.startswith(prefix + pname + "."))
            err = np.abs(got.cpu().numpy().reshape(-1) - g[key].reshape(-1)).max()
            assert err <= tol * max(fam, 1e-30), (key, err, fam)
            worst = max(worst, err / max(fam, 1e-30))
        print(f"{stem} {tag}: worst family-relative gradient error vs reference {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. gradients against the stepwise GPU loop and the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _grads(m, params, fn, x, G, names):
    for p in params.values():
        p.grad = None
    leaves = {k: (v.detach().clone().requires_grad_(True) if k in names and v is not None else v) for k, v in x.items()}
    traj = fn(m, leaves)
    sum((w * v).sum() for w, v in zip(G, traj)).backward()
    return [leaves[k].grad for k in names] + [torch.zeros_like(p) if p.grad is None else p.grad.clone() for p in params.values()]


def _compare(got, want, kinds, names, tol=1e-4):
    worst = 0.0
    for kind in dict.fromkeys(kinds):
        idx = [j for j, k in enumerate(kinds) if k == kind]
        fam = max(float(want[j].abs().max()) for j in idx)
        for j in idx:
            err = float((got[j] - want[j]).abs().max())
            assert err <= tol * max(fam, 1e-30), (names[j], err, fam)
            worst = max(worst, err / max(fam, 1e-30))
    return worst


@pytest.mark.parametrize("stem,batch,steps,grav,damp,layout", [
    ("iiwa7", 500, 16, True, True, "row"), ("panda", 130, 9, True, False, "shared"),
    ("2link_robot", 65, 20, False, True, "kp_row"), ("fetch_arm_no_gripper", 64, 8, True, False, "kd_row"),
    ("trifinger_edu", 97, 8, True, False, "row"), ("allegro_hand_description_left", 40, 6, True, False, "shared"),
    ("iiwa7_allegro", 50, 6, True, False, "kp_row"), ("iiwa7", 300, 10, True, True, "kd_row")])
def test_pd_rollout_gradients_match_the_stepwise_loop(stem, batch, steps, grav, damp, layout):
    m, params = learnable_model(stem)
    x = pd_inputs(m, stem, batch, steps, seed=7)
    x.update(gains(x, layout))
    gen = torch.Generator().manual_seed(8)
    G = [torch.randn(steps, batch, m._n_dofs, generator=gen).to(DEV) for _ in KEYS]
    dt = 1e-3
    fused = _grads(m, params, lambda mm, a: call(mm, a, dt, grav, damp), x, G, DIFF)
    ref = _grads(m, params, lambda mm, a: loop(mm, a, dt, grav, damp), x, G, DIFF)
    with torch.no_grad():
        tau = call(m, x, dt, grav, damp).tau
    assert bool((tau.abs() == x["lim"]).any()), "the limit should bind somewhere"
    names = list(DIFF) + [f"{p}.{i}" for (i, p) in params]
    kinds = list(DIFF) + [p for (_, p) in params]
    worst = _compare(fused, ref, kinds, names)
    print(f"{stem}: worst family-relative gradient difference to the stepwise loop {worst:.2e}")


@pytest.mark.parametrize("stem,batch,steps,damp,nonsym,per_row", [("iiwa7", 300, 12, True, True, True),
                                                                  ("panda_no_gripper", 200, 10, False, False, False),
                                                                  ("trifinger_edu", 64, 8, True, True, False)])
def test_pd_rollout_gradients_match_fp64_oracle(stem, batch, steps, damp, nonsym, per_row):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    m, params = learnable_model(stem)
    if nonsym:
        gen = torch.Generator().manual_seed(17)
        scale = robot.inertia.abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-6)
        robot.inertia = (robot.inertia + 0.05 * scale * torch.randn(robot.inertia.shape, generator=gen, dtype=torch.float64)).float().double()
        with torch.no_grad():
            for (i, pname), p in params.items():
                if pname == "inertia_mat":
                    p.copy_(robot.inertia[i].float().to(DEV))
    x = pd_inputs(m, stem, batch, steps, seed=11)
    if not per_row:
        x["kp"], x["kd"] = x["kp"].mean(0), x["kd"].mean(0)
    gen = torch.Generator().manual_seed(12)
    G = [torch.randn(steps, batch, robot.n_dofs, generator=gen) for _ in KEYS]
    dt = 1e-3
    got = _grads(m, params, lambda mm, a: call(mm, a, dt, True, damp), x, [w.to(DEV) for w in G], DIFF)
    names = ("trans", "rpy", "mass", "com", "inertia", "damping")
    for name in names:
        setattr(robot, name, getattr(robot, name).detach().clone().requires_grad_(True))
    ins = {k: x[k].detach().cpu().double().requires_grad_(True) for k in DIFF}
    lim = x["lim"].cpu().double()
    traj = pd_rollout(robot, ins["q0"], ins["qd0"], ins["q_ref"], ins["kp"], ins["kd"], dt, ins["qd_ref"], ins["f"], lim,
                      True, damp)
    # rows where fp32 and fp64 put u on different sides of the limit would differ by a whole gradient term: there are none
    with torch.no_grad():
        tau32 = call(m, x, dt, True, damp).tau.cpu().double()
    assert torch.equal(tau32.abs() == lim.float().double(), traj[3].abs() == lim)
    want = torch.autograd.grad(sum((w.double() * v).sum() for w, v in zip(G, traj)),
                               [ins[k] for k in DIFF] + [getattr(robot, nm) for nm in names], allow_unused=True)
    by = dict(zip(names, want[len(DIFF):]))
    tol = 1e-4
    worst = 0.0
    for a, b, what in zip(got[:len(DIFF)], want[:len(DIFF)], DIFF):
        worst = max(worst, family_close(a.cpu().numpy(), b.numpy(), tol, what))
    for ((i, pname), p), gp in zip(params.items(), got[len(DIFF):]):
        w = by[_ORACLE_PARAM[pname]]
        w = torch.zeros_like(getattr(robot, _ORACLE_PARAM[pname])) if w is None else w
        fam = float(w.abs().max())
        err = float((gp.cpu().double() - w[i]).abs().max())
        assert err <= tol * max(fam, 1e-30), (pname, i, err, fam)
        worst = max(worst, err / max(fam, 1e-30))
    print(f"{stem}: worst family-relative gradient error vs fp64 oracle {worst:.2e}")


def test_pd_rollout_tau_gradient_and_the_clamp_rule():
    """Only g_tau upstream: f_grad is g_tau where the clamp passes and 0 where it binds (no state gradient reaches the
    torques of the same step); q_ref_grad = kp f_grad, qd_ref_grad = kd f_grad there."""
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    x = pd_inputs(m, "iiwa7", 300, 1, seed=21)
    for k in ("f", "q_ref", "qd_ref"):
        x[k] = x[k].clone().requires_grad_(True)
    out = call(m, x, 1e-3)
    Gt = torch.randn_like(out.tau)
    (Gt * out.tau).sum().backward()
    u = x["f"] + x["kp"] * (x["q_ref"] - x["q0"]) + x["kd"] * (x["qd_ref"] - x["qd0"])
    passes = (u >= -x["lim"]) & (u <= x["lim"])
    assert 0 < int((~passes).sum()) < passes.numel()
    assert torch.equal(x["f"].grad, torch.where(passes, Gt, torch.zeros_like(Gt)))
    assert torch.equal(x["q_ref"].grad, x["kp"] * x["f"].grad)
    assert torch.equal(x["qd_ref"].grad, x["kd"] * x["f"].grad)


# ---------------------------------------------------------------------------------------------------------------------
# 5. reproducibility, fused parameters
# ---------------------------------------------------------------------------------------------------------------------
def test_pd_rollout_gradients_are_reproducible_and_fused_parameters_agree():
    base = drm.DifferentiableKUKAiiwa(device=DEV)
    x = pd_inputs(base, "iiwa7", 3001, 10, seed=5)
    x["kp"], x["kd"] = x["kp"].mean(0), x["kd"].mean(0)
    G = [torch.randn(10, 3001, 7, generator=torch.Generator().manual_seed(6 + i)).to(DEV) for i in range(4)]

    def run(fuse):
        m, params = learnable_model("iiwa7")
        flat = m.fuse_learnable_parameters() if fuse else None
        leaves = {k: x[k].clone().requires_grad_(True) for k in ("kp", "kd", "q_ref")}
        out = call(m, dict(x, **leaves), 1e-3, True, True)
        sum((w * v).sum() for w, v in zip(G, out)).backward()
        if fuse:       # the modules' Parameters are views of the flat vector: read each one's slice of its gradient
            grads = {k: flat.grad[(p.data_ptr() - flat.data_ptr()) // 4:][:p.numel()].view(p.shape) for k, p in params.items()}
        else:
            grads = {k: p.grad.clone() for k, p in params.items()}
        grads.update({k: v.grad for k, v in leaves.items()})
        return grads

    a, b, fused = run(False), run(False), run(True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
        assert torch.allclose(fused[k], a[k], rtol=1e-5, atol=1e-6 * float(a[k].abs().max())), k


# ---------------------------------------------------------------------------------------------------------------------
# 6. launch counts
# ---------------------------------------------------------------------------------------------------------------------
def test_pd_rollout_launch_counts():
    const = drm.DifferentiableKUKAiiwa(device=DEV)
    x = pd_inputs(const, "iiwa7", 1000, 25, seed=2)
    call(const, x, 1e-3)                                          # warm the cached table
    before = engine.launch_count()
    with torch.no_grad():
        call(const, x, 1e-3)
    assert engine.launch_count() - before == 1
    m, params = learnable_model("iiwa7")
    before = engine.launch_count()
    with torch.no_grad():
        call(m, x, 1e-3)
    table_build = engine.launch_count() - before - 1
    assert table_build >= 1
    kp = x["kp"].clone().requires_grad_(True)
    before = engine.launch_count()
    out = call(m, x, 1e-3, kp=kp)
    assert engine.launch_count() - before == 1 + table_build
    loss = sum(v.sum() for v in out)
    before = engine.launch_count()
    loss.backward()
    T = x["q_ref"].shape[0]
    # 2T + 2 library launches; the rest is the table build's backward
    assert engine.launch_count() - before <= 2 * T + 2 + 4


# ---------------------------------------------------------------------------------------------------------------------
# 7. edge cases, double backward, CUDA graphs
# ---------------------------------------------------------------------------------------------------------------------
def test_pd_rollout_edge_cases():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    x = pd_inputs(m, "iiwa7", 4, 3, seed=1)
    # T = 0 and B = 0
    out = call(m, x, 1e-3, q_ref=x["q_ref"][:0], qd_ref=None, f=None)
    assert all(t.shape == (0, 4, 7) for t in out)
    qa, kpa = x["q0"].clone().requires_grad_(True), x["kp"].mean(0).clone().requires_grad_(True)
    out = call(m, x, 1e-3, q0=qa, kp=kpa, q_ref=x["q_ref"][:0].clone(), qd_ref=None, f=None)
    sum(v.sum() for v in out).backward()
    assert torch.equal(qa.grad, torch.zeros_like(qa)) and torch.equal(kpa.grad, torch.zeros_like(kpa))
    out = call(m, x, 1e-3, q0=x["q0"][:0], qd0=x["qd0"][:0], q_ref=x["q_ref"][:, :0], qd_ref=x["qd_ref"][:, :0],
               f=x["f"][:, :0], kp=x["kp"][0], kd=x["kd"][0])
    assert out.q.shape == (3, 0, 7)
    # 1-D inputs give [T, n]; gains [n] only
    x1 = dict(q0=x["q0"][2], qd0=x["qd0"][2], q_ref=x["q_ref"][:, 2], qd_ref=x["qd_ref"][:, 2], f=x["f"][:, 2],
              kp=x["kp"][2], kd=x["kd"][2], lim=x["lim"])
    one = call(m, x1, 1e-3)
    full = call(m, x, 1e-3)
    assert one.q.shape == (3, 7)
    for a, b in zip(one, full):
        assert torch.equal(a, b[:, 2])
    # documented errors
    bad = [dict(q0=x["q0"].cpu(), qd0=x["qd0"].cpu()),                 # device
           dict(q_ref=x["q_ref"].double()),                            # dtype
           dict(kp=x["kp"].double()),
           dict(q_ref=x["q_ref"][0]),                                  # shapes
           dict(qd0=x["qd0"][:3]),
           dict(qd_ref=x["qd_ref"][:2]),
           dict(f=x["f"][..., :6]),
           dict(kp=x["kp"][:3]),                                       # a gain that is neither [n] nor [B, n]
           dict(kd=x["kd"][:, :6]),
           dict(lim=x["lim"][:6]),
           dict(lim=torch.where(torch.arange(7, device=DEV) == 3, 0.0, x["lim"])),          # limit <= 0
           dict(lim=torch.where(torch.arange(7, device=DEV) == 3, float("nan"), x["lim"]))]  # NaN limit
    for over in bad:
        with pytest.raises(AssertionError):
            call(m, x, 1e-3, **over)
    # a limit is checked once per tensor and version: an in-place change of a checked limit is caught
    lim = x["lim"].clone()
    call(m, x, 1e-3, lim=lim)
    lim[3] = 0.0
    with pytest.raises(AssertionError):
        call(m, x, 1e-3, lim=lim)
    with pytest.raises(AssertionError):
        call(m, x1, 1e-3, kp=x["kp"][2:3])                             # [1, n] gains with 1-D q0
    # the raw binding passes one layout flag for both gains: it refuses gains of different shapes (the model expands them)
    with pytest.raises(RuntimeError, match="same shape"):
        engine.pd_rollout_raw(m._topology, m._link_table(), x["q0"], x["qd0"], x["q_ref"], x["kp"], x["kd"][0], 1e-3, 1)


def test_pd_rollout_double_backward_raises():
    m, _ = learnable_model("iiwa7")
    x = pd_inputs(m, "iiwa7", 8, 3, seed=4)
    kp = x["kp"].clone().requires_grad_(True)
    out = call(m, x, 1e-3, kp=kp)
    (g,) = torch.autograd.grad(sum(v.sum() for v in out), kp, create_graph=True)
    with pytest.raises(RuntimeError, match="second-order"):
        g.sum().backward()


def test_pd_rollout_forward_and_backward_capture_in_one_cuda_graph():
    m, params = learnable_model("iiwa7")
    m.fuse_learnable_parameters()
    flat = m.fused_link_params.flat
    x = pd_inputs(m, "iiwa7", 777, 9, seed=9)
    x["kp"], x["kd"] = x["kp"].mean(0), x["kd"].mean(0)
    G = torch.randn(9, 777, 7, generator=torch.Generator().manual_seed(3)).to(DEV)
    kp = x["kp"].clone().requires_grad_(True)
    qr = x["q_ref"].clone().requires_grad_(True)

    def step():
        flat.grad = kp.grad = qr.grad = None
        out = call(m, x, 1e-3, True, True, kp=kp, q_ref=qr)
        (sum(out) * G).sum().backward()
        return out.q, out.tau, flat.grad, kp.grad, qr.grad

    eager = [t.detach().clone() for t in step()]      # detached: no eager autograd graph (default-stream nodes) stays alive
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    flat.grad, kp.grad, qr.grad = torch.zeros_like(flat), torch.zeros_like(kp), torch.zeros_like(qr)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = call(m, x, 1e-3, True, True, kp=kp, q_ref=qr)
        (sum(out) * G).sum().backward()
    for t in (flat.grad, kp.grad, qr.grad):
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip((out.q, out.tau, flat.grad, kp.grad, qr.grad), eager):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# 8. learning and gain tuning
# ---------------------------------------------------------------------------------------------------------------------
def test_learning_link_parameters_from_pd_tracked_trajectories():
    """A link's mass, CoM and inertia, perturbed, are recovered from the trajectories the true model follows under the
    same PD controller: identification from logs of a position-controlled robot.  The link is the elbow's (its mass and
    CoM load the shoulder joints through gravity, which the controller does not compensate); dt = 2^-10 s keeps explicit
    Euler stable under the diagonal gains, whose coupled closed-loop rates exceed w on the wrist.  Measured on an H100,
    the largest errors left were 0.7 % of the initial one for the mass, 1.1 % for the CoM and 8 % for the rotational
    inertia, which 48 ms of motion excites less than gravity does the first moment; the bounds leave a wide margin."""
    from differentiable_robot_model_b200.rigid_body_params import PositiveScalar, UnconstrainedTensor
    torch.manual_seed(0)
    gt = drm.DifferentiableKUKAiiwa(device=DEV)
    m = drm.DifferentiableRobotModel(gt.urdf_path, "learn", device=DEV)
    link = "iiwa_link_4"
    body = gt._bodies[[b.name for b in gt._bodies].index(link)]
    mass, com, inertia = (t().detach().clone().cpu() for t in (body.inertia.mass, body.inertia.com, body.inertia.inertia_mat))
    m.make_link_param_learnable(link, "mass", PositiveScalar(init_param=1.5 * mass.reshape(1, 1)))
    m.make_link_param_learnable(link, "com", UnconstrainedTensor(dim1=1, dim2=3, init_tensor=(com + 0.05).reshape(1, 3)))
    m.make_link_param_learnable(link, "inertia_mat", UnconstrainedTensor(dim1=3, dim2=3, init_tensor=1.5 * inertia.reshape(3, 3)))
    x = pd_inputs(gt, "iiwa7", 512, 48, seed=4)
    x["f"] = 0.5 * torch.randn(48, 512, 7, device=DEV)
    dt = 2.0 ** -10
    with torch.no_grad():
        target = call(gt, x, dt, True, True)
    var_q = target.q.var(dim=1, keepdim=True) + 1e-8
    var_qd = target.qd.var(dim=1, keepdim=True) + 1e-6
    opt = torch.optim.Adam(m.parameters(), lr=1e-2)
    losses = []
    for _ in range(100):
        opt.zero_grad()
        pred = call(m, x, dt, True, True)
        loss = (((pred.q - target.q) ** 2) / var_q).mean() + (((pred.qd - target.qd) ** 2) / var_qd).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    learned = m._bodies[[b.name for b in m._bodies].index(link)].inertia
    errors = {"mass": (float((learned.mass().detach().cpu() - mass).abs()), 0.5 * float(mass)),
              "com": (float((learned.com().detach().cpu().reshape(3) - com.reshape(3)).abs().max()), 0.05),
              "inertia": (float((learned.inertia_mat().detach().cpu().reshape(3, 3) - inertia.reshape(3, 3)).abs().max()),
                          0.5 * float(inertia.abs().max()))}
    print(f"loss {losses[0]:.3e} -> {losses[-1]:.3e}; |error| learned / initial: "
          + ", ".join(f"{k} {a:.3g} / {b:.3g}" for k, (a, b) in errors.items()))
    assert np.isfinite(losses).all()
    assert losses[-1] < 0.1 * losses[0], (losses[0], losses[-1])
    assert errors["mass"][0] < 0.05 * errors["mass"][1], errors
    assert errors["com"][0] < 0.1 * errors["com"][1], errors
    assert errors["inertia"][0] < 0.5 * errors["inertia"][1], errors


def test_gain_tuning_lowers_tracking_and_torque_cost():
    sys.path.insert(0, os.path.join(REPO, "examples"))
    import tune_pd_gains_iiwa as ex
    hist, kp, kd = ex.run(batch=128, steps=100, iters=40, log=lambda *_: None)
    assert np.isfinite(hist).all() and hist[-1] < 0.7 * hist[0], (hist[0], hist[-1])
    assert bool((kp > 0).all() and (kd > 0).all())


def test_tune_pd_gains_example_smoke():
    sys.path.insert(0, os.path.join(REPO, "examples"))
    import tune_pd_gains_iiwa as ex
    hist, _, _ = ex.run(batch=16, steps=20, iters=3, log=lambda *_: None)
    assert len(hist) == 3 and np.isfinite(hist).all()
