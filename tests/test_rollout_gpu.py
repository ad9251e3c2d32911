"""GPU: forward-dynamics rollouts (csrc/rollout.cu) -- T semi-implicit Euler steps over the articulated-body kernel in one
launch, and the ABA adjoint stepped backwards in time:

  * bit-identity with the Python loop of compute_forward_dynamics + `qd = qd + dt * qdd; q = q + dt * qd`;
  * trajectories and gradients against the reference's own loop (tests/golden/*.rollout.npz);
  * gradients against autograd through the same GPU loop and against the fp64 oracle;
  * reproducibility, launch counts, edge cases, CUDA graphs and a small system-identification loop.

Gradient tolerances are family-relative (each of q0, qd0, f and every link-parameter kind against the largest entry of
its family), as in test_forward_dynamics_backward_gpu.py, but 1e-4 throughout: measured on an H100 the worst family-relative
errors were 1.1e-5 against the reference's goldens, 1.1e-6 against autograd through the stepwise GPU loop (arms and hands
alike) and 1.4e-6 against the fp64 oracle.
"""
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from conftest import GOLDEN_DIR, URDFS, urdf_path
from test_backward_gpu import _ORACLE_PARAM, cuda, learnable_model
from differentiable_robot_model_b200 import engine
from oracle import drm_oracle as O
from rollout_oracle import forward_dynamics_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ARMS = {"iiwa7", "panda_no_gripper", "panda", "fetch_arm_no_gripper", "fetch_arm_no_gripper_small_damping", "2link_robot"}
FLAGS = [(g, d) for g in (True, False) for d in (True, False)]


def stepwise(model, q0, qd0, f, dt, grav, damp):
    q, qd = q0, qd0
    qs, qds, qdds = [], [], []
    for t in range(f.shape[0]):
        qdd = model.compute_forward_dynamics(q, qd, f[t], grav, damp)
        qd = qd + dt * qdd
        q = q + dt * qd
        qs.append(q)
        qds.append(qd)
        qdds.append(qdd)
    return torch.stack(qs), torch.stack(qds), torch.stack(qdds)


def inputs(stem, batch, steps, seed, fscale=0.05):
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, _ = O.sample_inputs(robot, batch, seed=seed, vel_scale=0.02)
    gen = torch.Generator().manual_seed(seed)
    f = fscale * torch.randn(steps, batch, robot.n_dofs, generator=gen)
    return q.to(DEV), qd.clamp(-1, 1).to(DEV), f.to(DEV)


def misaligned(t):
    """A contiguous copy of t whose base address is 4 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, device=t.device, dtype=t.dtype)
    out = buf[1:].view(t.shape)
    out.copy_(t)
    return out


def bits(t):
    """Bit pattern of an fp32 tensor: identical trajectories compare equal even where a stiff damped model diverged to NaN."""
    return t.contiguous().view(torch.int32)


def family_close(got, want, tol, what):
    got, want = np.asarray(got, dtype=np.float64).reshape(-1), np.asarray(want, dtype=np.float64).reshape(-1)
    scale = np.abs(want).max() if want.size else 0.0
    err = np.abs(got - want).max() if got.size else 0.0
    assert err <= tol * max(scale, 1e-30), f"{what}: |err| {err:.3e} vs family scale {scale:.3e} (tol {tol})"
    return err / max(scale, 1e-30)


# ---------------------------------------------------------------------------------------------------------------------
# 1. bit-identity with the stepwise loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_rollout_is_bit_identical_to_the_stepwise_loop(stem):
    models = {"constant": drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV), "learnable": learnable_model(stem)[0]}
    with torch.no_grad():
        for kind, m in models.items():
            for batch in (1, 63, 65, 1000):
                for steps in (1, 17):
                    q0, qd0, f = inputs(stem, batch, steps, seed=batch + steps)
                    for dt in (2.0 ** -9, 1e-3):
                        for grav, damp in FLAGS:
                            got = m.compute_forward_dynamics_rollout(q0, qd0, f, dt, grav, damp)
                            want = stepwise(m, q0, qd0, f, dt, grav, damp)
                            for name, a, b in zip(("q", "qd", "qdd"), got, want):
                                assert torch.equal(bits(a), bits(b)), (kind, batch, steps, dt, grav, damp, name)
        # unaligned bases (cooperative copies) and the 64-configuration tile (a batch that fills every SM)
        m = models["constant"]
        for batch in (65, 20000):
            q0, qd0, f = inputs(stem, batch, 5, seed=3)
            want = stepwise(m, q0, qd0, f, 1e-3, True, True)
            for args in ((misaligned(q0), qd0, f), (q0, qd0, misaligned(f))):
                got = m.compute_forward_dynamics_rollout(*args, 1e-3, True, True)
                for a, b in zip(got, want):
                    assert torch.equal(bits(a), bits(b)), batch


# ---------------------------------------------------------------------------------------------------------------------
# 2. reference goldens
# ---------------------------------------------------------------------------------------------------------------------
GOLDEN_STEMS = ["2link_robot", "iiwa7", "panda_no_gripper", "trifinger_edu", "iiwa7_allegro"]


@pytest.mark.parametrize("stem", GOLDEN_STEMS)
def test_rollout_matches_reference_trajectories_and_gradients(stem):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".rollout.npz"), allow_pickle=False)
    dt = float(g["dt"])
    tol = 1e-4
    tags = sorted({k.split(".")[0] for k in g.files if k.startswith("g1d")})
    const = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    for tag in tags:
        damp = tag == "g1d1"
        with torch.no_grad():
            traj = const.compute_forward_dynamics_rollout(cuda(g["q0"]), cuda(g["qd0"]), cuda(g["f"]), dt, True, damp)
        for name, got in zip(("q", "qd", "qdd"), traj):
            want = g[f"{tag}.{name}"]
            scale = np.abs(want).max(axis=2, keepdims=True)
            rel = (np.abs(got.cpu().numpy() - want) / (scale + 1e-6)).max()
            assert rel < (2e-4 if stem in ARMS else 2e-3), (tag, name, rel)
        m, params = learnable_model(stem)
        q0, qd0, f = cuda(g["q0"], True), cuda(g["qd0"], True), cuda(g["f"], True)
        traj = m.compute_forward_dynamics_rollout(q0, qd0, f, dt, True, damp)
        sum((cuda(g[f"G_{k}"]) * v).sum() for k, v in zip(("q", "qd", "qdd"), traj)).backward()
        prefix = f"{tag}.grad."
        worst = 0.0
        for key, t in (("q0", q0), ("qd0", qd0), ("f", f)):
            worst = max(worst, family_close(t.grad.cpu().numpy(), g[prefix + key], tol, f"{tag}.{key}"))
        for key in g.files:
            if not key.startswith(prefix) or key[len(prefix):] in ("q0", "qd0", "f"):
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
# 3. gradients against the stepwise GPU loop and the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _grads(m, params, fn, q0, qd0, f, G):
    for p in params.values():
        p.grad = None
    ins = [t.detach().clone().requires_grad_(True) for t in (q0, qd0, f)]
    traj = fn(m, *ins)
    sum((w * v).sum() for w, v in zip(G, traj)).backward()
    return [t.grad for t in ins] + [torch.zeros_like(p) if p.grad is None else p.grad.clone() for p in params.values()]


@pytest.mark.parametrize("stem,batch,steps,grav,damp", [("iiwa7", 500, 16, True, True), ("panda", 130, 9, True, False),
                                                        ("2link_robot", 65, 20, False, True), ("fetch_arm_no_gripper", 64, 8, True, False),
                                                        ("trifinger_edu", 97, 8, True, False),
                                                        ("allegro_hand_description_left", 40, 6, True, False),
                                                        ("iiwa7_allegro", 50, 6, True, False)])
def test_rollout_gradients_match_the_stepwise_loop(stem, batch, steps, grav, damp):
    m, params = learnable_model(stem)
    q0, qd0, f = inputs(stem, batch, steps, seed=7)
    gen = torch.Generator().manual_seed(8)
    G = [torch.randn(steps, batch, m._n_dofs, generator=gen).to(DEV) for _ in range(3)]
    dt = 1e-3
    fused = _grads(m, params, lambda mm, a, b, c: mm.compute_forward_dynamics_rollout(a, b, c, dt, grav, damp), q0, qd0, f, G)
    loop = _grads(m, params, lambda mm, a, b, c: stepwise(mm, a, b, c, dt, grav, damp), q0, qd0, f, G)
    names = ["q0", "qd0", "f"] + [f"{p}.{i}" for (i, p) in params]
    kinds = ["q0", "qd0", "f"] + [p for (_, p) in params]
    tol = 1e-4
    worst = 0.0
    for kind in dict.fromkeys(kinds):
        idx = [j for j, k in enumerate(kinds) if k == kind]
        fam = max(float(loop[j].abs().max()) for j in idx)
        for j in idx:
            err = float((fused[j] - loop[j]).abs().max())
            assert err <= tol * max(fam, 1e-30), (names[j], err, fam)
            worst = max(worst, err / max(fam, 1e-30))
    print(f"{stem}: worst family-relative gradient difference to the stepwise loop {worst:.2e}")


@pytest.mark.parametrize("stem,batch,steps,damp,nonsym", [("iiwa7", 300, 12, True, True), ("panda_no_gripper", 200, 10, False, False),
                                                          ("trifinger_edu", 64, 8, True, True)])
def test_rollout_gradients_match_fp64_oracle(stem, batch, steps, damp, nonsym):
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
    q0, qd0, f = inputs(stem, batch, steps, seed=11)
    gen = torch.Generator().manual_seed(12)
    G = [torch.randn(steps, batch, robot.n_dofs, generator=gen) for _ in range(3)]
    dt = 1e-3
    got = _grads(m, params, lambda mm, a, b, c: mm.compute_forward_dynamics_rollout(a, b, c, dt, True, damp), q0, qd0, f,
                 [x.to(DEV) for x in G])
    names = ("trans", "rpy", "mass", "com", "inertia", "damping")
    for name in names:
        setattr(robot, name, getattr(robot, name).detach().clone().requires_grad_(True))
    ins = [t.detach().cpu().double().requires_grad_(True) for t in (q0, qd0, f)]
    traj = forward_dynamics_rollout(robot, *ins, dt, True, damp)
    want = torch.autograd.grad(sum((w.double() * v).sum() for w, v in zip(G, traj)),
                               ins + [getattr(robot, nm) for nm in names], allow_unused=True)
    by = dict(zip(names, want[3:]))
    tol = 1e-4
    worst = 0.0
    for a, b, what in zip(got[:3], want[:3], ("q0", "qd0", "f")):
        worst = max(worst, family_close(a.cpu().numpy(), b.numpy(), tol, what))
    for ((i, pname), p), gp in zip(params.items(), got[3:]):
        w = by[_ORACLE_PARAM[pname]]
        w = torch.zeros_like(getattr(robot, _ORACLE_PARAM[pname])) if w is None else w
        fam = float(w.abs().max())
        err = float((gp.cpu().double() - w[i]).abs().max())
        assert err <= tol * max(fam, 1e-30), (pname, i, err, fam)
        worst = max(worst, err / max(fam, 1e-30))
    print(f"{stem}: worst family-relative gradient error vs fp64 oracle {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. reproducibility, fused parameters
# ---------------------------------------------------------------------------------------------------------------------
def test_rollout_table_gradient_is_reproducible_and_fused_parameters_agree():
    q0, qd0, f = inputs("iiwa7", 3001, 10, seed=5)
    G = torch.randn(10, 3001, 7, generator=torch.Generator().manual_seed(6)).to(DEV)

    def run(fuse):
        m, params = learnable_model("iiwa7")
        flat = m.fuse_learnable_parameters() if fuse else None
        q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, f, 1e-3, True, True)
        ((q + qd + qdd) * G).sum().backward()
        if fuse:       # the modules' Parameters are views of the flat vector: read each one's slice of its gradient
            return {k: flat.grad[(p.data_ptr() - flat.data_ptr()) // 4:][:p.numel()].view(p.shape) for k, p in params.items()}
        return {k: p.grad.clone() for k, p in params.items()}

    a, b, fused = run(False), run(False), run(True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
        assert torch.allclose(fused[k], a[k], rtol=1e-5, atol=1e-6 * float(a[k].abs().max())), k


# ---------------------------------------------------------------------------------------------------------------------
# 5. launch counts
# ---------------------------------------------------------------------------------------------------------------------
def test_rollout_launch_counts():
    const = drm.DifferentiableKUKAiiwa(device=DEV)
    q0, qd0, f = inputs("iiwa7", 1000, 25, seed=2)
    const.compute_forward_dynamics_rollout(q0, qd0, f, 1e-3)         # warm the cached table
    before = engine.launch_count()
    with torch.no_grad():
        const.compute_forward_dynamics_rollout(q0, qd0, f, 1e-3)
    assert engine.launch_count() - before == 1
    m, params = learnable_model("iiwa7")
    before = engine.launch_count()
    with torch.no_grad():
        m.compute_forward_dynamics_rollout(q0, qd0, f, 1e-3)
    table_build = engine.launch_count() - before - 1
    assert table_build >= 1
    qa = q0.clone().requires_grad_(True)
    before = engine.launch_count()
    q, qd, qdd = m.compute_forward_dynamics_rollout(qa, qd0, f, 1e-3)
    assert engine.launch_count() - before == 1 + table_build
    loss = q.sum() + qd.sum() + qdd.sum()
    before = engine.launch_count()
    loss.backward()
    T = f.shape[0]
    # 2T + 2 library launches; the rest is the table build's backward
    assert engine.launch_count() - before <= 2 * T + 2 + 4


# ---------------------------------------------------------------------------------------------------------------------
# 6. edge cases
# ---------------------------------------------------------------------------------------------------------------------
def test_rollout_edge_cases():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    q0, qd0, f = inputs("iiwa7", 4, 3, seed=1)
    # T = 0 and B = 0
    q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, f[:0], 1e-3)
    assert q.shape == qd.shape == qdd.shape == (0, 4, 7)
    qa = q0.clone().requires_grad_(True)
    q, qd, qdd = m.compute_forward_dynamics_rollout(qa, qd0, f[:0].clone(), 1e-3)
    (q.sum() + qd.sum() + qdd.sum()).backward()
    assert torch.equal(qa.grad, torch.zeros_like(q0))
    q, qd, qdd = m.compute_forward_dynamics_rollout(q0[:0], qd0[:0], f[:, :0], 1e-3)
    assert q.shape == (3, 0, 7)
    # 1-D inputs give [T, n]
    q1, qd1, qdd1 = m.compute_forward_dynamics_rollout(q0[2], qd0[2], f[:, 2], 1e-3)
    q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, f, 1e-3)
    assert q1.shape == (3, 7)
    assert torch.equal(q1, q[:, 2]) and torch.equal(qd1, qd[:, 2]) and torch.equal(qdd1, qdd[:, 2])
    # documented errors
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_rollout(q0.cpu(), qd0.cpu(), f.cpu(), 1e-3)
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_rollout(q0, qd0, f[0], 1e-3)                    # 2-D f with 2-D q0
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_rollout(q0, qd0[:3], f, 1e-3)
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_rollout(q0[:, :6], qd0[:, :6], f[..., :6], 1e-3)
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_rollout(q0.double(), qd0.double(), f.double(), 1e-3)
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_rollout(q0, qd0, f[:, :3], 1e-3)


# ---------------------------------------------------------------------------------------------------------------------
# 7. CUDA graphs
# ---------------------------------------------------------------------------------------------------------------------
def test_rollout_forward_and_backward_capture_in_one_cuda_graph():
    m, params = learnable_model("iiwa7")
    m.fuse_learnable_parameters()
    flat = m.fused_link_params.flat
    q0, qd0, f = inputs("iiwa7", 777, 9, seed=9)
    G = torch.randn(9, 777, 7, generator=torch.Generator().manual_seed(3)).to(DEV)
    fa = f.clone().requires_grad_(True)

    def step():
        flat.grad = None
        fa.grad = None
        q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, fa, 1e-3, True, True)
        loss = ((q + qd + qdd) * G).sum()
        loss.backward()
        return q, flat.grad, fa.grad

    eager = [t.detach().clone() for t in step()]      # detached: no eager autograd graph (default-stream nodes) stays alive
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    flat.grad = torch.zeros_like(flat)
    fa.grad = torch.zeros_like(fa)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        q, qd, qdd = m.compute_forward_dynamics_rollout(q0, qd0, fa, 1e-3, True, True)
        ((q + qd + qdd) * G).sum().backward()
    flat.grad.zero_()
    fa.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(q, eager[0])
    assert torch.equal(flat.grad, eager[1])
    assert torch.equal(fa.grad, eager[2])


# ---------------------------------------------------------------------------------------------------------------------
# 8. learning from a simulated trajectory
# ---------------------------------------------------------------------------------------------------------------------
def test_learning_link_inertia_from_a_rollout():
    from differentiable_robot_model_b200.rigid_body_params import PositiveScalar, UnconstrainedTensor
    torch.manual_seed(0)
    gt = drm.DifferentiableKUKAiiwa(device=DEV)
    m = drm.DifferentiableRobotModel(gt.urdf_path, "learn", device=DEV)
    m.make_link_param_learnable("iiwa_link_1", "mass", PositiveScalar())
    m.make_link_param_learnable("iiwa_link_1", "com", UnconstrainedTensor(dim1=1, dim2=3))
    m.make_link_param_learnable("iiwa_link_1", "inertia_mat", UnconstrainedTensor(dim1=3, dim2=3))
    q0, qd0, _ = inputs("iiwa7", 512, 1, seed=4)
    tau = 2.0 * torch.randn(16, 512, 7, device=DEV)
    dt = 2.0 ** -8
    with torch.no_grad():
        target = gt.compute_forward_dynamics_rollout(q0, qd0, tau, dt, use_damping=True)[1]
    var = target.var(dim=1, keepdim=True) + 1e-6
    opt = torch.optim.Adam(m.parameters(), lr=1e-2)
    losses = []
    for _ in range(100):
        opt.zero_grad()
        pred = m.compute_forward_dynamics_rollout(q0, qd0, tau, dt, use_damping=True)[1]
        loss = (((pred - target) ** 2) / var).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert np.isfinite(losses).all()
    assert losses[-1] < 0.2 * losses[0], (losses[0], losses[-1])
