"""GPU: the analytic backward kernels (csrc/backward.cu) through torch.autograd, against

  * the gradients of the reference's own autograd graph (tests/golden/*.npz, every shipped URDF);
  * torch.autograd of the fp64 oracle on larger seeded batches (including the quaternion output);
and that the table-gradient reduction is bitwise reproducible.

Tolerance: the golden gradients are fp32 autograd results of the reference (noise ~1e-6 relative to
the largest entry); the kernels are compared with rtol 2e-4 and an absolute floor of 2e-5 x the
largest gradient entry of the same loss.
"""
import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden, urdf_path
import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar, UnconstrainedTensor
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def learnable_model(stem):
    """Every link parameter replaced by an unconstrained module initialised at the URDF value
    (mirrors make_all_learnable in tests/golden/make_golden.py)."""
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    params = {}
    for i, body in enumerate(m._bodies):
        if i == 0:
            continue
        inits = {
            "mass": UnconstrainedScalar(init_val=body.inertia.mass().detach().clone()),
            "com": UnconstrainedTensor(1, 3, init_tensor=body.inertia.com().detach().clone().reshape(1, 3)),
            "inertia_mat": UnconstrainedTensor(3, 3, init_tensor=body.inertia.inertia_mat().detach().clone().reshape(3, 3)),
        }
        if body.joint_idx is not None:
            inits["trans"] = UnconstrainedTensor(1, 3, init_tensor=body.trans().detach().clone().reshape(1, 3))
            inits["rot_angles"] = UnconstrainedTensor(1, 3, init_tensor=body.rot_angles().detach().clone().reshape(1, 3))
            inits["joint_damping"] = UnconstrainedScalar(init_val=body.joint_damping().detach().clone())
        for pname, module in inits.items():
            m.make_link_param_learnable(body.name, pname, module)
            params[(i, pname)] = module.param
    return m, params


def cuda(a, grad=False):
    t = torch.tensor(np.asarray(a), dtype=torch.float32, device=DEV)
    return t.requires_grad_(True) if grad else t


def shifted(x):
    """The same values in a fresh contiguous tensor whose base address is 4 bytes past a 16-byte boundary: kernels must take
    their cooperative-copy staging instead of TMA bulk copies / float4 accesses for it."""
    buf = x.new_empty(x.numel() + 1)
    buf[1:].copy_(x.reshape(-1))
    out = buf[1:].view_as(x)
    assert out.data_ptr() % 16 != 0 and out.is_contiguous()
    return out


def check_against_golden(g, prefix, params, input_grads):
    scale = max(float(np.abs(g[k]).max()) for k in g.files if k.startswith(prefix + "."))
    tol = dict(rtol=2e-4, atol=2e-5 * max(scale, 1.0))
    for key, got in input_grads.items():
        assert_close(got.cpu().numpy(), g[f"{prefix}.{key}"], what=f"{prefix}.{key}", **tol)
    checked = 0
    for key in g.files:
        if not key.startswith(prefix + "."):
            continue
        rest = key[len(prefix) + 1:]
        if "." not in rest:
            continue
        pname, idx = rest.rsplit(".", 1)
        p = params[(int(idx), pname)]
        got = torch.zeros_like(p) if p.grad is None else p.grad
        assert_close(got.cpu().numpy().reshape(g[key].shape), g[key], what=key, **tol)
        checked += 1
    assert checked > 0


def test_fk_jacobian_gradients_match_reference_autograd(robot_stem):
    g = load_golden(robot_stem)
    for link in g["fk_links"].tolist()[:2]:
        m, params = learnable_model(robot_stem)
        q = cuda(g["q"], grad=True)
        pos, _ = m.compute_forward_kinematics(q, link)
        jl, ja = m.compute_endeffector_jacobian(q, link)
        loss = (cuda(g["G_pos"]) * pos).sum() + (cuda(g["G_jl"]) * jl).sum() + (cuda(g["G_ja"]) * ja).sum()
        loss.backward()
        check_against_golden(g, f"fkgrad.{link}", params, {"q": q.grad})


def test_inverse_dynamics_gradients_match_reference_autograd(robot_stem):
    g = load_golden(robot_stem)
    m, params = learnable_model(robot_stem)
    q, qd, qdd = cuda(g["q"], True), cuda(g["qd"], True), cuda(g["qdd"], True)
    tau = m.compute_inverse_dynamics(q, qd, qdd, include_gravity=True, use_damping=True)
    (cuda(g["G_tau"]) * tau).sum().backward()
    check_against_golden(g, "idgrad", params, {"q": q.grad, "qd": qd.grad, "qdd": qdd.grad})


_ORACLE_PARAM = {"trans": "trans", "rot_angles": "rpy", "mass": "mass", "com": "com", "inertia_mat": "inertia",
                 "joint_damping": "damping"}


def _oracle_grads(stem, loss_fn, inputs):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    for name in set(_ORACLE_PARAM.values()):
        getattr(robot, name).requires_grad_(True)
    ins = [t.detach().cpu().double().requires_grad_(True) for t in inputs]
    loss = loss_fn(robot, *ins)
    wrt = ins + [getattr(robot, n) for n in ("trans", "rpy", "mass", "com", "inertia", "damping")]
    grads = torch.autograd.grad(loss, wrt, allow_unused=True)
    by = dict(zip(("trans", "rpy", "mass", "com", "inertia", "damping"), grads[len(ins):]))
    return grads[:len(ins)], by, robot


def _compare_params(params, by, robot, scale, skip_fixed_kinematic):
    tol = dict(rtol=2e-4, atol=2e-5 * max(scale, 1.0))
    for (i, pname), p in params.items():
        want = by[_ORACLE_PARAM[pname]]
        want = torch.zeros_like(getattr(robot, _ORACLE_PARAM[pname])) if want is None else want
        got = torch.zeros_like(p) if p.grad is None else p.grad
        assert_close(got.cpu().numpy().reshape(-1), want[i].numpy().reshape(-1), what=f"{pname}.{i}", **tol)


@pytest.mark.parametrize("stem,link,batch", [("iiwa7", "iiwa_link_ee", 1000), ("iiwa7", "iiwa_link_5", 130),
                                             ("allegro_hand_description_left", "link_7.0_tip", 517),
                                             ("iiwa7_allegro", "link_15.0_tip", 259), ("panda", "panda_leftfinger", 64)])
def test_fk_jacobian_gradients_match_fp64_oracle(stem, link, batch):
    """All four outputs (including the quaternion, whose gradient the reference gets wrong) at once."""
    robot = O.load_robot(urdf_path(stem), torch.float64)
    q64, _, _ = O.sample_inputs(robot, batch, seed=batch, dtype=torch.float64)
    q32 = q64.float()
    gen = torch.Generator().manual_seed(batch)
    n = robot.n_dofs
    Gp, Gq = torch.randn(batch, 3, generator=gen), torch.randn(batch, 4, generator=gen)
    Gl, Ga = torch.randn(batch, 3, n, generator=gen), torch.randn(batch, 3, n, generator=gen)

    m, params = learnable_model(stem)
    q = q32.to(DEV).requires_grad_(True)
    pos, quat, jl, ja = m.compute_fk_and_jacobian(q, link)
    # the oracle decides the quaternion sign per row; align signs so both losses are the same function
    o_pos, o_quat = O.forward_kinematics(robot, q32.double(), link)
    sign = torch.sign((quat.detach().cpu().double() * o_quat).sum(1, keepdim=True))
    Gq_dev = (Gq * sign.float()).to(DEV)
    loss = (Gp.to(DEV) * pos).sum() + (Gq_dev * quat).sum() + (Gl.to(DEV) * jl).sum() + (Ga.to(DEV) * ja).sum()
    loss.backward()

    def oracle_loss(rb, qq):
        p, qu = O.forward_kinematics(rb, qq, link)
        l, a = O.jacobian(rb, qq, link)
        return (Gp.double() * p).sum() + (Gq.double() * qu).sum() + (Gl.double() * l).sum() + (Ga.double() * a).sum()

    (dq,), by, rb = _oracle_grads(stem, oracle_loss, [q32])
    scale = max(float(dq.abs().max()), max(float(v.abs().max()) for v in by.values() if v is not None))
    assert_close(q.grad.cpu().numpy(), dq.numpy(), rtol=2e-4, atol=2e-5 * max(scale, 1.0), what="dq")
    _compare_params({k: v for k, v in params.items() if k[1] in ("trans", "rot_angles")}, by, rb, scale, True)


@pytest.mark.parametrize("stem,batch,grav,damp", [("iiwa7", 1000, True, True), ("panda_no_gripper", 300, False, True),
                                                  ("allegro_hand_description_left", 200, True, False),
                                                  ("trifinger_edu", 129, True, True), ("jaco_clean", 77, False, False),
                                                  ("iiwa7_allegro", 130, True, True)])
def test_inverse_dynamics_gradients_match_fp64_oracle(stem, batch, grav, damp):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    q, qd, qdd = (t.float() for t in O.sample_inputs(robot, batch, seed=batch + 1, dtype=torch.float64))
    gen = torch.Generator().manual_seed(batch)
    G = torch.randn(batch, robot.n_dofs, generator=gen)
    m, params = learnable_model(stem)
    qg, qdg, qddg = (t.to(DEV).requires_grad_(True) for t in (q, qd, qdd))
    tau = m.compute_inverse_dynamics(qg, qdg, qddg, include_gravity=grav, use_damping=damp)
    (G.to(DEV) * tau).sum().backward()

    (dq, dqd, dqdd), by, rb = _oracle_grads(
        stem, lambda r, a, b, c: (G.double() * O.inverse_dynamics(r, a, b, c, grav, damp)).sum(), [q, qd, qdd])
    scale = max(float(x.abs().max()) for x in (dq, dqd, dqdd))
    scale = max(scale, max(float(v.abs().max()) for v in by.values() if v is not None))
    tol = dict(rtol=2e-4, atol=2e-5 * max(scale, 1.0))
    assert_close(qg.grad.cpu().numpy(), dq.numpy(), what="dq", **tol)
    assert_close(qdg.grad.cpu().numpy(), dqd.numpy(), what="dqd", **tol)
    assert_close(qddg.grad.cpu().numpy(), dqdd.numpy(), what="dqdd", **tol)
    _compare_params(params, by, rb, scale, False)


def test_table_gradient_is_bitwise_reproducible_and_input_only_path_works():
    m, params = learnable_model("iiwa7")
    robot = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, 70001, seed=3))
    G = torch.randn(70001, 7, device=DEV)

    def run():
        for p in params.values():
            p.grad = None
        tau = m.compute_inverse_dynamics(q, qd, qdd)
        (G * tau).sum().backward()
        return torch.cat([p.grad.reshape(-1) for p in params.values()]).clone()

    a, b = run(), run()
    assert torch.equal(a, b)
    # grads w.r.t. q only (trajectory optimisation use case): constant model, no table gradient
    const = drm.DifferentiableKUKAiiwa(device=DEV)
    qg = q[:5000].clone().requires_grad_(True)
    pos, _ = const.compute_forward_kinematics(qg, "iiwa_link_ee")
    pos.square().sum().backward()
    jl, _ = const.compute_endeffector_jacobian(qg.detach(), "iiwa_link_ee")
    want = torch.einsum("bi,bij->bj", 2 * pos.detach(), jl)              # d|p|^2/dq = 2 p^T J_lin
    assert float((qg.grad - want).abs().max()) < 1e-4


def test_learning_loop_reduces_loss():
    """examples/learn_dynamics_iiwa.py in miniature: recover link-1 mass / inertia / trans from torques."""
    torch.manual_seed(0)
    gt = drm.DifferentiableKUKAiiwa(device=DEV)
    robot = O.load_robot(gt.urdf_path, torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, 4096, seed=9))
    target = gt.compute_inverse_dynamics(q, qd, qdd)
    from differentiable_robot_model_b200.rigid_body_params import PositiveScalar
    m = drm.DifferentiableRobotModel(gt.urdf_path, "learn", device=DEV)
    m.make_link_param_learnable("iiwa_link_1", "mass", PositiveScalar())
    m.make_link_param_learnable("iiwa_link_1", "inertia_mat", UnconstrainedTensor(dim1=3, dim2=3))
    m.make_link_param_learnable("iiwa_link_2", "trans", UnconstrainedTensor(dim1=1, dim2=3))
    opt = torch.optim.Adam(m.parameters(), lr=3e-2)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        loss = (m.compute_inverse_dynamics(q, qd, qdd) - target).square().mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.2 * losses[0], losses[::10]


@pytest.mark.parametrize("stem,batch,grav,damp", [("iiwa7", 70001, True, True), ("allegro_hand_description_left", 999, True, True),
                                                  ("trifinger_edu", 130, False, False), ("iiwa7_allegro", 257, True, False)])
def test_inertial_only_backward_matches_the_full_adjoint(stem, batch, grav, damp):
    """With only mass / com / inertia_mat / damping learnable and no input gradients the RNEA backward takes the
    single-sweep kernel (DRMB200_INERTIAL_GRADS_ONLY); its gradients must equal the full adjoint kernel's."""
    from differentiable_robot_model_b200 import engine

    def model(with_kinematic):
        m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
        params = {}
        for i, body in enumerate(m._bodies):
            if i == 0:
                continue
            mods = {"mass": UnconstrainedScalar(init_val=body.inertia.mass().detach().clone()),
                    "com": UnconstrainedTensor(1, 3, init_tensor=body.inertia.com().detach().clone().reshape(1, 3)),
                    "inertia_mat": UnconstrainedTensor(3, 3, init_tensor=body.inertia.inertia_mat().detach().clone().reshape(3, 3))}
            if body.joint_idx is not None:
                mods["joint_damping"] = UnconstrainedScalar(init_val=body.joint_damping().detach().clone())
                if with_kinematic:       # a learnable joint origin forces the full adjoint kernel
                    mods["trans"] = UnconstrainedTensor(1, 3, init_tensor=body.trans().detach().clone().reshape(1, 3))
            for pname, mod in mods.items():
                m.make_link_param_learnable(body.name, pname, mod)
                params[(i, pname)] = mod.param
        return m, params

    robot = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=11))
    G = torch.randn(batch, robot.n_dofs, device=DEV)
    grads = []
    for with_kin in (False, True):
        m, params = model(with_kin)
        assert m._kinematic_params_learnable() == with_kin
        tau = m.compute_inverse_dynamics(q, qd, qdd, include_gravity=grav, use_damping=damp)
        (G * tau).sum().backward()
        grads.append({k: p.grad.clone() for k, p in params.items() if k[1] != "trans"})
    scale = max(float(g.abs().max()) for g in grads[1].values())
    for k in grads[0]:
        assert_close(grads[0][k].cpu().numpy(), grads[1][k].cpu().numpy(), rtol=1e-4, atol=1e-5 * max(scale, 1.0), what=str(k))


def test_training_step_replays_from_a_cuda_graph():
    """Forward (FK + RNEA + ABA), backward (three analytic adjoint kernels + reductions) and the Adam update captured
    once in a CUDA graph: replays must reproduce the eager optimisation trajectory (no hidden syncs / allocations in
    the library, launches on the capturing stream)."""
    robot = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, 4096, seed=9))
    f = torch.randn(4096, 7, generator=torch.Generator().manual_seed(2)).to(DEV)
    target = torch.randn(4096, 7, generator=torch.Generator().manual_seed(3)).to(DEV)

    def make():
        m, params = learnable_model("iiwa7")
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)

        def step():
            opt.zero_grad(set_to_none=False)
            with m.shared_link_table():
                pos, _, jl, _ = m.compute_fk_and_jacobian(q, "iiwa_link_ee")
                tau = m.compute_inverse_dynamics(q, qd, qdd)
                acc = m.compute_forward_dynamics(q, qd, f, use_damping=True)
            loss = (tau - target).square().mean() + pos.square().mean() + jl.square().mean() + 1e-4 * acc.square().mean()
            loss.backward()
            opt.step()
            return loss
        return step

    eager = make()
    want = [float(eager().detach()) for _ in range(6)]

    step = make()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = [float(step().detach()) for _ in range(3)]          # warm-up iterations are real optimisation steps
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step()
    got.append(float(loss))                                        # capture does not execute: value comes from replay
    got = got[:3]
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        got.append(float(loss))
    np.testing.assert_allclose(got, want, rtol=2e-4)
    assert got[-1] < got[0]


@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "fetch_arm_no_gripper", "2link_robot"])
@pytest.mark.parametrize("batch", [1, 63, 64, 130, 4099])
def test_chain_adjoint_kernel_matches_the_tree_kernel(stem, batch):
    """Serial chains take the two-sweep RNEA adjoint kernel (option rnea_bwd_chain, default on); every gradient must agree
    with the general tree kernel: all gradients (learnable model), input gradients only (constant model), bulk-copy and
    cooperative staging (inputs off 16-byte alignment), full and partial tiles."""
    from differentiable_robot_model_b200 import engine

    if engine.get_option("rnea_bwd_chain") == 0:
        pytest.skip("the two-sweep kernel is switched off (DRMB200_RNEA_BWD_CHAIN=0)")
    robot = O.load_robot(urdf_path(stem), torch.float32)
    n = robot.n_dofs
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=batch + 5))
    G = torch.randn(batch, n, device=DEV)
    learn, params = learnable_model(stem)
    const = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)

    def run(model, unaligned, grav, damp):
        for p in params.values():
            p.grad = None
        ins = [(shifted(t) if unaligned else t.clone()).requires_grad_(True) for t in (q, qd, qdd)]
        tau = model.compute_inverse_dynamics(*ins, include_gravity=grav, use_damping=damp)
        (G * tau).sum().backward()
        out = [t.grad.clone() for t in ins]
        if model is learn:
            out += [p.grad.clone() if p.grad is not None else torch.zeros_like(p) for p in params.values()]
        return out

    try:
        for model in (learn, const):
            for unaligned, grav, damp in ((False, True, True), (True, False, True), (False, True, False)):
                engine.set_option("rnea_bwd_chain", 0)
                want = run(model, unaligned, grav, damp)
                engine.set_option("rnea_bwd_chain", 1)
                before = engine.launch_count()
                got = run(model, unaligned, grav, damp)
                assert engine.launch_count() > before
                scale = max(float(w.abs().max()) for w in want)
                for i, (a, b) in enumerate(zip(got, want)):
                    assert_close(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-4, atol=1e-5 * max(scale, 1.0),
                                 what=f"{stem} B={batch} learnable={model is learn} unaligned={unaligned} grad {i}")
    finally:
        engine.set_option("rnea_bwd_chain", 1)
