"""GPU: the autograd contract of every differentiable entry point, beyond one plain backward with every input asking for
a gradient.

  1. Second order.  The backward kernels are first-order only; differentiating their gradients (a Hessian, a gradient
     penalty, a MAML-style inner step on the link parameters) must raise instead of silently treating the gradients as
     constants, and first-order gradients taken under ``create_graph=True`` must equal the plain ones bit for bit.
  2. Subsets of requested gradients.  The launchers pass NULL for every input gradient nobody asked for and for every
     skipped output; each subset is compared with fp64 oracle autograd, tensors not asked for keep ``grad is None``, a
     subset that runs the same kernel as the all-inputs run must reproduce its gradient bit for bit, and one that changes
     kernel must agree within tolerance.
  3. Layouts and reuse of upstream gradients: stride-0, transposed, one column, off 16-byte alignment, ``retain_graph``
     twice, a side stream, an empty batch.

Tolerances: inverse dynamics, kinematics and the mass matrix use test_backward_gpu.py's (rtol 2e-4, atol 2e-5 x the
largest oracle gradient of the same loss).  Forward dynamics and rollouts use the family-relative tolerances of
test_forward_dynamics_backward_gpu.py and test_rollout_gpu.py (the fp32 articulated-body algorithm amplifies rounding by
the conditioning of the articulated inertias).  Bit-identity is the sharp check: a wrong pointer or a skipped accumulation
changes bits, not just the last digit.
"""
import ctypes

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from conftest import assert_close, urdf_path
from differentiable_robot_model_b200 import engine
from oracle import drm_oracle as O
from rollout_oracle import forward_dynamics_rollout
from test_backward_gpu import _ORACLE_PARAM, _compare_params, _oracle_grads, learnable_model, shifted
from test_rollout_gpu import inputs as rollout_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STEMS = ["iiwa7", "panda", "iiwa7_allegro"]          # serial chain kernel, folded fixed links, tree kernel
BATCHES = [257, 1024]                                 # ragged tiles, bulk-staged tiles
EE = {"iiwa7": "iiwa_link_ee", "panda": "panda_leftfinger", "iiwa7_allegro": "link_15.0_tip"}
SECOND_EE = {"iiwa7": "iiwa_link_5", "panda": "panda_link4", "iiwa7_allegro": "link_3.0_tip"}
ARMS = {"iiwa7", "panda"}
ORACLE_NAMES = ("trans", "rpy", "mass", "com", "inertia", "damping")


def _tol(scale):
    return dict(rtol=2e-4, atol=2e-5 * max(scale, 1.0))


def _freeze(params, kinds=None):
    for (_, pname), p in params.items():
        if kinds is None or pname in kinds:
            p.requires_grad_(False)


def _family_close(got, want, tol, what):
    got, want = np.asarray(got, dtype=np.float64).reshape(-1), np.asarray(want, dtype=np.float64).reshape(-1)
    scale = np.abs(want).max() if want.size else 0.0
    err = np.abs(got - want).max() if got.size else 0.0
    assert err <= tol * max(scale, 1e-30), f"{what}: |err| {err:.3e} vs family scale {scale:.3e} (tol {tol})"


def _compare_param_families(params, by, robot, tol):
    """Per parameter kind, each link's gradient against the largest oracle entry of that kind (family-relative)."""
    for (i, pname), p in params.items():
        want = by[_ORACLE_PARAM[pname]]
        want = torch.zeros_like(getattr(robot, _ORACLE_PARAM[pname])) if want is None else want
        got = torch.zeros_like(p) if p.grad is None else p.grad
        fam = float(want.abs().max())
        err = float((got.cpu().double().reshape(-1) - want[i].reshape(-1)).abs().max())
        assert err <= tol * max(fam, 1e-30), (pname, i, err, fam)


def _assert_param_grads_equal(params, reference, what):
    for key, p in params.items():
        assert p.grad is not None, (what, key)
        assert torch.equal(p.grad, reference[key].grad), (what, key)


def _assert_no_param_grads(params, what):
    for key, p in params.items():
        assert p.grad is None, (what, key)


# ---------------------------------------------------------------------------------------------------------------------
# 1. second order raises; first order under create_graph is unchanged
# ---------------------------------------------------------------------------------------------------------------------
ENTRY_POINTS = ["forward_kinematics", "endeffector_jacobian", "fk_and_jacobian", "fk_and_jacobian_multi",
                "forward_kinematics_all_links", "inverse_dynamics", "non_linear_effects", "lagrangian_inertia_matrix",
                "lagrangian_inertia_matrix_stacked", "forward_dynamics", "forward_dynamics_crba", "forward_dynamics_rollout"]


def _scalar_entry(m, name, stem, qd, qdd, f):
    """q -> a scalar through one differentiable entry point (the plain sum of its outputs)."""
    link, link2 = EE[stem], SECOND_EE[stem]

    def total(outs):
        return sum(o.sum() for o in outs)

    return {
        "forward_kinematics": lambda q: total(m.compute_forward_kinematics(q, link)),
        "endeffector_jacobian": lambda q: total(m.compute_endeffector_jacobian(q, link)),
        "fk_and_jacobian": lambda q: total(m.compute_fk_and_jacobian(q, link)),
        "fk_and_jacobian_multi": lambda q: sum(total(v) for v in m.compute_fk_and_jacobian_multi(q, [link, link2]).values()),
        "forward_kinematics_all_links": lambda q: sum(total(v) for v in m.compute_forward_kinematics_all_links(q).values()),
        "inverse_dynamics": lambda q: m.compute_inverse_dynamics(q, qd, qdd).sum(),
        "non_linear_effects": lambda q: m.compute_non_linear_effects(q, qd).sum(),
        "lagrangian_inertia_matrix": lambda q: m.compute_lagrangian_inertia_matrix(q).sum(),
        "lagrangian_inertia_matrix_stacked": lambda q: m.compute_lagrangian_inertia_matrix_stacked(q).sum(),
        "forward_dynamics": lambda q: m.compute_forward_dynamics(q, qd, f[0]).sum(),
        "forward_dynamics_crba": lambda q: m.compute_forward_dynamics_crba(q, qd, f[0]).sum(),
        "forward_dynamics_rollout": lambda q: total(m.compute_forward_dynamics_rollout(q, qd, f, 1e-3)),
    }[name]


@pytest.fixture(params=["per_module", "fused"])
def second_order_case(request):
    stem = "iiwa7"
    m, params = learnable_model(stem)
    leaves = [m.fuse_learnable_parameters()] if request.param == "fused" else list(params.values())
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, 3, seed=21))
    f = 0.5 * torch.randn(2, 3, robot.n_dofs, generator=torch.Generator().manual_seed(22)).to(DEV)
    return stem, m, leaves, q, qd, qdd, f


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_second_order_raises_and_first_order_is_unchanged(second_order_case, entry):
    stem, m, leaves, q0, qd, qdd, f = second_order_case
    fn = _scalar_entry(m, entry, stem, qd, qdd, f)

    # Hessian w.r.t. q: torch's default (strict=False) would fill an all-zero Hessian if the kernels' gradients were
    # treated as constants
    with pytest.raises(RuntimeError, match="second-order derivatives"):
        torch.autograd.functional.hessian(fn, q0.clone())

    # gradient penalty on q
    q = q0.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(fn(q), q, create_graph=True)
    with pytest.raises(RuntimeError, match="second-order derivatives"):
        (fn(q) + g.square().sum()).backward()

    # MAML-style inner step on the link parameters: the outer loss depends on p - lr * dL/dp
    inner = torch.autograd.grad(fn(q0), leaves, create_graph=True, allow_unused=True)
    adapted = [p - 1e-3 * gp for p, gp in zip(leaves, inner) if gp is not None]
    assert adapted, "no link parameter received a gradient"
    with pytest.raises(RuntimeError, match="compute_inverse_dynamics_derivatives"):
        (fn(q0) + sum(a.square().sum() for a in adapted)).backward()
    for p in leaves:
        p.grad = None

    # first order, with and without create_graph: bit-identical.  Except on the CRBA route: torch's own backward of
    # torch.linalg.solve is not bit-identical with and without create_graph, so the gradient the kernels receive there
    # differs in rounding
    q = q0.clone().requires_grad_(True)
    plain = torch.autograd.grad(fn(q), [q] + leaves, allow_unused=True)
    graphed = torch.autograd.grad(fn(q), [q] + leaves, allow_unused=True, create_graph=True)
    assert plain[0] is not None
    scale = max(float(a.abs().max()) for a in plain if a is not None)
    for i, (a, b) in enumerate(zip(plain, graphed)):
        assert (a is None) == (b is None), i
        if a is None:
            continue
        if entry == "forward_dynamics_crba":
            torch.testing.assert_close(b.detach(), a, rtol=1e-3, atol=1e-4 * scale)
        else:
            assert torch.equal(a, b.detach()), (entry, i)


# ---------------------------------------------------------------------------------------------------------------------
# 2. subsets of requested gradients
# ---------------------------------------------------------------------------------------------------------------------
def _samples(stem, batch, seed):
    robot = O.load_robot(urdf_path(stem), torch.float64)
    q, qd, qdd = (t.float() for t in O.sample_inputs(robot, batch, seed=seed, dtype=torch.float64))
    return robot, q, qd, qdd


def _run(m, fn, values, asked):
    """fn(m, *inputs) -> scalar loss on the GPU with only the inputs named in `asked` requiring grad; {name: grad}."""
    ins = {k: v.to(DEV).clone().requires_grad_(k in asked) for k, v in values.items()}
    fn(m, *ins.values()).backward()
    return {k: t.grad for k, t in ins.items()}


def _check_subsets(stem, fn, values, want, tol_of, table_want=None):
    """The shared skeleton for inverse and forward dynamics (three inputs plus the link table).

    full:  every input and every link parameter -> the adjoint kernel with table columns;
    const: every input, frozen parameters -> the input-only kernel;
    each single input with frozen parameters -> that kernel again with two input-gradient pointers NULL: bit-identical
    to `const`; the table alone -> the `full` kernel with every input-gradient pointer NULL: bit-identical to `full`."""
    names = list(values)
    m_full, p_full = learnable_model(stem)
    full = _run(m_full, fn, values, set(names))
    for k in names:
        tol_of(full[k], want[k], f"full {k}")
    if table_want is not None:
        table_want(p_full)

    m_c, p_c = learnable_model(stem)
    _freeze(p_c)
    const = _run(m_c, fn, values, set(names))
    for k in names:
        tol_of(const[k], want[k], f"const {k}")
    for name in names:
        got = _run(m_c, fn, values, {name})
        for k in names:
            if k == name:
                assert torch.equal(got[k], const[k]), f"{name} alone differs from the all-inputs run"
            else:
                assert got[k] is None, (name, k)
        _assert_no_param_grads(p_c, f"{name} alone")

    m_t, p_t = learnable_model(stem)
    got = _run(m_t, fn, values, set())
    assert all(g is None for g in got.values())
    _assert_param_grads_equal(p_t, p_full, "table alone")
    return m_full, p_full


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("stem", STEMS)
def test_inverse_dynamics_gradient_subsets(stem, batch):
    robot, q, qd, qdd = _samples(stem, batch, seed=batch + 3)
    G = torch.randn(batch, robot.n_dofs, generator=torch.Generator().manual_seed(batch))
    (dq, dqd, dqdd), by, rb = _oracle_grads(
        stem, lambda r, a, b, c: (G.double() * O.inverse_dynamics(r, a, b, c, True, True)).sum(), [q, qd, qdd])
    scale = max(float(x.abs().max()) for x in (dq, dqd, dqdd))
    scale = max(scale, max(float(v.abs().max()) for v in by.values() if v is not None))
    tol = _tol(scale)
    Gd = G.to(DEV)

    def fn(m, a, b, c):
        return (Gd * m.compute_inverse_dynamics(a, b, c, include_gravity=True, use_damping=True)).sum()

    def close(got, want, what):
        assert_close(got.cpu().numpy(), want.numpy(), what=f"{stem} B={batch} {what}", **tol)

    _, p_full = _check_subsets(stem, fn, {"q": q, "qd": qd, "qdd": qdd}, {"q": dq, "qd": dqd, "qdd": dqdd}, close,
                               lambda params: _compare_params(params, by, rb, scale, False))

    # the table alone with only inertial parameters learning: the single-sweep kernel (DRMB200_INERTIAL_GRADS_ONLY)
    m_i, p_i = learnable_model(stem)
    _freeze(p_i, ("trans", "rot_angles"))
    assert not m_i._kinematic_params_learnable()
    got = _run(m_i, fn, {"q": q, "qd": qd, "qdd": qdd}, set())
    assert all(g is None for g in got.values())
    inertial = {k: p for k, p in p_i.items() if k[1] not in ("trans", "rot_angles")}
    _assert_no_param_grads({k: p for k, p in p_i.items() if k not in inertial}, "frozen joint origins")
    _compare_params(inertial, by, rb, scale, False)
    for key, p in inertial.items():
        assert_close(p.grad.cpu().numpy(), p_full[key].grad.cpu().numpy(), what=f"inertial-only {key}", **tol)


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("stem", STEMS)
def test_forward_dynamics_gradient_subsets(stem, batch):
    robot, q, qd, _ = _samples(stem, batch, seed=batch + 4)
    gen = torch.Generator().manual_seed(batch + 1)
    f = torch.randn(batch, robot.n_dofs, generator=gen)
    G = torch.randn(batch, robot.n_dofs, generator=gen)
    (dq, dqd, df), by, rb = _oracle_grads(
        stem, lambda r, a, b, c: (G.double() * O.forward_dynamics(r, a, b, c, True, True)).sum(), [q, qd, f])
    ftol = 2e-3 if stem in ARMS else 2e-2
    Gd = G.to(DEV)

    def fn(m, a, b, c):
        return (Gd * m.compute_forward_dynamics(a, b, c, include_gravity=True, use_damping=True)).sum()

    def close(got, want, what):
        _family_close(got.cpu().numpy(), want.numpy(), ftol, f"{stem} B={batch} {what}")

    m_full, _ = _check_subsets(stem, fn, {"q": q, "qd": qd, "f": f}, {"q": dq, "qd": dqd, "f": df}, close,
                               lambda params: _compare_param_families(params, by, rb, ftol))

    # f alone against an independent kernel: G^T dqdd/df from the forward-mode derivatives kernel
    got = _run(m_full, fn, {"q": q, "qd": qd, "f": f}, {"f"})
    with torch.no_grad():
        dqdd_df = m_full.compute_forward_dynamics_derivatives(q.to(DEV), qd.to(DEV), f.to(DEV), True, True)[2]
    want = torch.einsum("bi,bij->bj", Gd, dqdd_df)
    _family_close(got["f"].cpu().numpy(), want.cpu().numpy(), 1e-4, f"{stem} B={batch} f vs derivatives kernel")


ROLLOUT_UPSTREAMS = ["q", "qd", "qdd", "last_step", "all"]


def _rollout_upstream(kind, steps, batch, n, seed):
    gen = torch.Generator().manual_seed(seed)
    G = [torch.randn(steps, batch, n, generator=gen) for _ in range(3)]
    if kind in ("q", "qd", "qdd"):
        keep = ("q", "qd", "qdd").index(kind)
        G = [g if i == keep else torch.zeros_like(g) for i, g in enumerate(G)]
    elif kind == "last_step":
        for g in G:
            g[:-1] = 0
    return G


@pytest.mark.parametrize("steps", [1, 5])
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("stem", STEMS)
def test_rollout_gradient_subsets(stem, batch, steps):
    dt = 1e-3
    q0, qd0, f = (t.cpu() for t in rollout_inputs(stem, batch, steps, seed=batch + steps))
    values = {"q0": q0, "qd0": qd0, "f": f}
    n = q0.shape[1]
    tol = 1e-4

    robot = O.load_robot(urdf_path(stem), torch.float64)
    for name in ORACLE_NAMES:
        getattr(robot, name).requires_grad_(True)
    o_ins = [t.double().requires_grad_(True) for t in values.values()]
    o_traj = forward_dynamics_rollout(robot, *o_ins, dt, True, False)
    wrt = o_ins + [getattr(robot, nm) for nm in ORACLE_NAMES]

    for kind in ROLLOUT_UPSTREAMS:
        G = _rollout_upstream(kind, steps, batch, n, seed=batch + 7)
        o_loss = sum((g.double() * v).sum() for g, v in zip(G, o_traj))
        o_grads = torch.autograd.grad(o_loss, wrt, retain_graph=True, allow_unused=True)
        want = dict(zip(values, o_grads[:3]))
        by = dict(zip(ORACLE_NAMES, o_grads[3:]))
        Gd = [g.to(DEV) for g in G]

        def fn(m, a, b, c):
            return sum((g * v).sum() for g, v in zip(Gd, m.compute_forward_dynamics_rollout(a, b, c, dt, True, False)))

        def close(got, w, what):
            _family_close(got.cpu().numpy(), w.numpy(), tol, f"{stem} B={batch} T={steps} upstream={kind} {what}")

        _check_subsets(stem, fn, values, want, close, lambda params: _compare_param_families(params, by, robot, tol))


def _rollout_adjoint(m, q0, qd0, f, dt, flags, g):
    """drmb200_forward_dynamics_rollout_backward called directly, so that upstream gradients can be NULL (autograd hands
    the Function materialised zeros instead)."""
    T, B, n = f.shape
    table = m._link_table().detach().contiguous()
    q, qd, _ = engine.forward_dynamics_rollout_raw(m._topology, table, q0, qd0, f, dt, flags)
    outs = [torch.full_like(q0, float("nan")), torch.full_like(q0, float("nan")), torch.full_like(f, float("nan")),
            torch.zeros_like(table)]
    nbytes = int(engine.lib().drmb200_forward_dynamics_rollout_backward_workspace_bytes(ctypes.byref(m._topology), B))
    ws = torch.empty((max(nbytes, 4) + 3) // 4, device=q0.device, dtype=torch.float32)
    rc = engine.lib().drmb200_forward_dynamics_rollout_backward(
        ctypes.byref(m._topology), engine._ptr(table), engine._ptr(q0), engine._ptr(qd0), engine._ptr(f), B, T,
        ctypes.c_float(dt), flags, engine._ptr(q), engine._ptr(qd), *[engine._ptr(x) for x in g], *[engine._ptr(o) for o in outs],
        engine._ptr(ws), engine._stream())
    engine._check(rc, "drmb200_forward_dynamics_rollout_backward")
    return outs


@pytest.mark.parametrize("stem", STEMS)
def test_rollout_adjoint_null_upstream_equals_zero_upstream(stem):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    q0, qd0, f = rollout_inputs(stem, 257, 5, seed=30)
    G = [torch.randn(f.shape, generator=torch.Generator().manual_seed(31 + i)).to(DEV) for i in range(3)]
    for keep in range(3):
        nulls = [G[i] if i == keep else None for i in range(3)]
        zeros = [G[i] if i == keep else torch.zeros_like(G[i]) for i in range(3)]
        a = _rollout_adjoint(m, q0, qd0, f, 1e-3, engine.GRAVITY, nulls)
        b = _rollout_adjoint(m, q0, qd0, f, 1e-3, engine.GRAVITY, zeros)
        for i, (x, y) in enumerate(zip(a, b)):
            assert torch.isfinite(x).all(), (keep, i)
            assert torch.equal(x, y), (keep, i)


FK_OUTPUTS = ("pos", "quat", "jac_lin", "jac_ang")


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("stem", STEMS)
def test_fk_output_and_input_subsets(stem, batch):
    """Each output alone, skipped (NULL upstream pointers: compute_forward_kinematics skips the Jacobians,
    compute_endeffector_jacobian the pose) and returned but unused (compute_fk_and_jacobian, zero upstream); q alone and
    the table alone."""
    link = EE[stem]
    robot, q, _, _ = _samples(stem, batch, seed=batch + 5)
    n = robot.n_dofs
    gen = torch.Generator().manual_seed(batch + 2)
    G = {"pos": torch.randn(batch, 3, generator=gen), "quat": torch.randn(batch, 4, generator=gen),
         "jac_lin": torch.randn(batch, 3, n, generator=gen), "jac_ang": torch.randn(batch, 3, n, generator=gen)}
    const = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    with torch.no_grad():
        quat = const.compute_forward_kinematics(q.to(DEV), link)[1].cpu().double()
    sign = torch.sign((quat * O.forward_kinematics(robot, q.double(), link)[1]).sum(1, keepdim=True)).float()
    G_dev = {k: (v * sign if k == "quat" else v).to(DEV) for k, v in G.items()}

    for out in FK_OUTPUTS:
        def oracle_loss(rb, qq):
            p, qu = O.forward_kinematics(rb, qq, link)
            jl, ja = O.jacobian(rb, qq, link)
            return (G[out].double() * dict(pos=p, quat=qu, jac_lin=jl, jac_ang=ja)[out]).sum()

        (dq,), by, rb = _oracle_grads(stem, oracle_loss, [q])
        scale = max(float(dq.abs().max()), max(float(v.abs().max()) for v in by.values() if v is not None))
        tol = _tol(scale)
        pose_out = out in ("pos", "quat")

        def skipped(m, qq):
            if pose_out:
                o = m.compute_forward_kinematics(qq, link)[FK_OUTPUTS.index(out)]
            else:
                o = m.compute_endeffector_jacobian(qq, link)[FK_OUTPUTS.index(out) - 2]
            return (G_dev[out] * o).sum()

        def unused(m, qq):
            return (G_dev[out] * m.compute_fk_and_jacobian(qq, link)[FK_OUTPUTS.index(out)]).sum()

        # q alone (constant table: the kernel without table columns)
        m_c, p_c = learnable_model(stem)
        _freeze(p_c)
        got = {route: _run(m_c, fn, {"q": q}, {"q"})["q"] for route, fn in (("skipped", skipped), ("unused", unused))}
        assert torch.equal(got["skipped"], got["unused"]), f"{stem} {out}: skipped and unused outputs differ"
        assert_close(got["skipped"].cpu().numpy(), dq.numpy(), what=f"{stem} B={batch} {out} q", **tol)
        _assert_no_param_grads(p_c, out)

        # the table alone
        per_route = {}
        for route, fn in (("skipped", skipped), ("unused", unused)):
            m_t, p_t = learnable_model(stem)
            assert _run(m_t, fn, {"q": q}, set())["q"] is None
            _compare_params(p_t, by, rb, scale, True)
            per_route[route] = p_t
        _assert_param_grads_equal(per_route["skipped"], per_route["unused"], f"{stem} {out} table")


@pytest.mark.parametrize("path", ["multi", "all_links"])
@pytest.mark.parametrize("batch", BATCHES)
def test_multi_link_and_all_links_gradient_on_one_link(batch, path):
    """A gradient on one link of the multi-link / all-links outputs equals the single-link gradient bit for bit (the same
    kernel runs for that link; the others get zero upstream or are skipped); a gradient on the root alone is exactly zero."""
    stem = "iiwa7_allegro"
    link, other = SECOND_EE[stem], EE[stem]
    robot, q, _, _ = _samples(stem, batch, seed=batch + 6)
    n = robot.n_dofs
    gen = torch.Generator().manual_seed(batch + 3)
    G = [torch.randn(batch, 3, generator=gen).to(DEV), torch.randn(batch, 4, generator=gen).to(DEV),
         torch.randn(batch, 3, n, generator=gen).to(DEV), torch.randn(batch, 3, n, generator=gen).to(DEV)]
    root = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV).get_link_names()[0]
    if path == "all_links":
        G = G[:2]

    def outputs(m, qq, name):
        if path == "multi":
            return m.compute_fk_and_jacobian_multi(qq, [root, other, link] if name == root else [other, link])[name]
        return m.compute_forward_kinematics_all_links(qq)[name]

    def single(m, qq):
        outs = m.compute_fk_and_jacobian(qq, link) if path == "multi" else m.compute_forward_kinematics(qq, link)
        return sum((g * o).sum() for g, o in zip(G, outs))

    for asked in ({"q"}, {"q", "table"}):
        results = []
        for fn in (single, lambda m, qq: sum((g * o).sum() for g, o in zip(G, outputs(m, qq, link)))):
            m, params = learnable_model(stem)
            if "table" not in asked:
                _freeze(params)
            results.append((_run(m, fn, {"q": q}, {"q"})["q"], params))
        (g_single, p_single), (g_multi, p_multi) = results
        assert torch.equal(g_multi, g_single), (path, asked)
        if "table" in asked:
            _assert_param_grads_equal(p_multi, p_single, f"{path} one link")

        m, params = learnable_model(stem)
        if "table" not in asked:
            _freeze(params)
        got = _run(m, lambda mm, qq: sum((g * o).sum() for g, o in zip(G, outputs(mm, qq, root))), {"q": q}, {"q"})["q"]
        assert torch.count_nonzero(got) == 0, (path, "root")
        for key, p in params.items():
            assert p.grad is None or torch.count_nonzero(p.grad) == 0, (path, "root", key)


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("stem", STEMS)
def test_mass_matrix_gradient_subsets(stem, batch):
    robot, q, _, _ = _samples(stem, batch, seed=batch + 8)
    n = robot.n_dofs
    G = torch.randn(batch, n, n, generator=torch.Generator().manual_seed(batch + 4))

    def oracle_H(r, qq):
        zero = torch.zeros_like(qq)
        eye = torch.eye(n, dtype=qq.dtype)
        return torch.stack([O.inverse_dynamics(r, qq, zero, eye[j].expand_as(qq), False, False) for j in range(n)], dim=2)

    (dq,), by, rb = _oracle_grads(stem, lambda r, qq: (G.double() * oracle_H(r, qq)).sum(), [q])
    scale = max(float(dq.abs().max()), max(float(v.abs().max()) for v in by.values() if v is not None))
    tol = _tol(scale)
    Gd = G.to(DEV)

    def fn(m, qq):
        return (Gd * m.compute_lagrangian_inertia_matrix(qq)).sum()

    m_full, p_full = learnable_model(stem)
    full = _run(m_full, fn, {"q": q}, {"q"})["q"]
    assert_close(full.cpu().numpy(), dq.numpy(), what=f"{stem} B={batch} full q", **tol)
    _compare_params(p_full, by, rb, scale, False)

    m_c, p_c = learnable_model(stem)
    _freeze(p_c)
    got = _run(m_c, fn, {"q": q}, {"q"})["q"]
    assert_close(got.cpu().numpy(), dq.numpy(), what=f"{stem} B={batch} q alone", **tol)
    assert_close(got.cpu().numpy(), full.cpu().numpy(), what=f"{stem} B={batch} q alone vs full", **tol)
    _assert_no_param_grads(p_c, "q alone")

    m_t, p_t = learnable_model(stem)
    assert _run(m_t, fn, {"q": q}, set())["q"] is None
    _assert_param_grads_equal(p_t, p_full, "table alone")


# ---------------------------------------------------------------------------------------------------------------------
# 3. layouts and reuse of upstream gradients
# ---------------------------------------------------------------------------------------------------------------------
def _layout_case(stem="iiwa7", batch=257):
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=41))
    G = torch.randn(batch, robot.n_dofs, generator=torch.Generator().manual_seed(42)).to(DEV)
    return q, qd, qdd, G


def _id_grads(backward, stem="iiwa7"):
    """Run inverse dynamics on a learnable model with every input requiring grad, call backward(tau), return every grad."""
    q, qd, qdd, _ = _layout_case(stem)
    m, params = learnable_model(stem)
    ins = [t.clone().requires_grad_(True) for t in (q, qd, qdd)]
    tau = m.compute_inverse_dynamics(*ins)
    backward(tau)
    return [t.grad.clone() for t in ins] + [p.grad.clone() for p in params.values()]


def _assert_all_equal(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, i)


def test_upstream_gradient_layouts():
    _, _, _, G = _layout_case()
    ones = _id_grads(lambda tau: tau.backward(torch.ones_like(tau)))
    _assert_all_equal(_id_grads(lambda tau: tau.sum().backward()), ones, "stride-0 from sum()")
    _assert_all_equal(_id_grads(lambda tau: tau.backward(torch.ones(1, tau.shape[1], device=DEV).expand_as(tau))), ones,
                      "expanded row")

    dense = _id_grads(lambda tau: tau.backward(G))
    _assert_all_equal(_id_grads(lambda tau: (tau.t() * G.t()).sum().backward()), dense, "loss on tau.t()")
    _assert_all_equal(_id_grads(lambda tau: tau.backward(G.t().contiguous().t())), dense, "column-major upstream")
    _assert_all_equal(_id_grads(lambda tau: tau.backward(shifted(G))), dense, "upstream off 16-byte alignment")

    col = torch.zeros_like(G)
    col[:, 3] = G[:, 3]
    _assert_all_equal(_id_grads(lambda tau: (tau[:, 3] * G[:, 3]).sum().backward()), _id_grads(lambda tau: tau.backward(col)),
                      "loss on one column")

    # the same on the kinematics: a loss on the transposed Jacobian, and an unaligned upstream
    q = _layout_case()[0]
    gen = torch.Generator().manual_seed(43)
    Gj = torch.randn(q.shape[0], 3, q.shape[1], generator=gen).to(DEV)

    def fk_grads(backward):
        m, params = learnable_model("iiwa7")
        qq = q.clone().requires_grad_(True)
        backward(m.compute_endeffector_jacobian(qq, "iiwa_link_ee")[0])
        return [qq.grad.clone()] + [p.grad.clone() for p in params.values()]

    want = fk_grads(lambda jl: jl.backward(Gj))
    _assert_all_equal(fk_grads(lambda jl: (jl.transpose(1, 2) * Gj.transpose(1, 2)).sum().backward()), want, "fk transposed")
    _assert_all_equal(fk_grads(lambda jl: jl.backward(shifted(Gj))), want, "fk unaligned upstream")


def test_retain_graph_twice_and_a_side_stream():
    q, qd, qdd, G = _layout_case()
    m, params = learnable_model("iiwa7")
    ins = [t.clone().requires_grad_(True) for t in (q, qd, qdd)]
    loss = (G * m.compute_inverse_dynamics(*ins)).sum() + m.compute_forward_kinematics(ins[0], "iiwa_link_ee")[0].sum() \
        + m.compute_forward_dynamics(ins[0], ins[1], ins[2]).sum()
    grads = []
    for _ in range(2):
        for t in ins + list(params.values()):
            t.grad = None
        loss.backward(retain_graph=True)
        grads.append([t.grad.clone() for t in ins + list(params.values())])
    _assert_all_equal(grads[0], grads[1], "retain_graph")

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        m2, params2 = learnable_model("iiwa7")
        ins2 = [t.clone().requires_grad_(True) for t in (q, qd, qdd)]
        loss2 = (G * m2.compute_inverse_dynamics(*ins2)).sum() + m2.compute_forward_kinematics(ins2[0], "iiwa_link_ee")[0].sum() \
            + m2.compute_forward_dynamics(ins2[0], ins2[1], ins2[2]).sum()
        loss2.backward()
        got = [t.grad.clone() for t in ins2 + list(params2.values())]
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    _assert_all_equal(got, grads[0], "side stream")


@pytest.mark.parametrize("stem", ["iiwa7", "iiwa7_allegro"])
def test_empty_batch_backward(stem):
    m, params = learnable_model(stem)
    n = m._n_dofs
    q, qd, x = (torch.zeros(0, n, device=DEV, requires_grad=True) for _ in range(3))
    f = torch.zeros(3, 0, n, device=DEV, requires_grad=True)
    link, link2 = EE[stem], SECOND_EE[stem]
    losses = {
        "fk": lambda: sum(o.sum() for o in m.compute_fk_and_jacobian(q, link)),
        "multi": lambda: sum(o.sum() for v in m.compute_fk_and_jacobian_multi(q, [link, link2]).values() for o in v),
        "all_links": lambda: sum(o.sum() for v in m.compute_forward_kinematics_all_links(q).values() for o in v),
        "inverse_dynamics": lambda: m.compute_inverse_dynamics(q, qd, x).sum(),
        "forward_dynamics": lambda: m.compute_forward_dynamics(q, qd, x).sum(),
        "mass_matrix": lambda: m.compute_lagrangian_inertia_matrix(q).sum(),
        "rollout": lambda: sum(o.sum() for o in m.compute_forward_dynamics_rollout(q, qd, f, 1e-3)),
    }
    for name, loss in losses.items():
        for t in (q, qd, x, f, *params.values()):
            t.grad = None
        loss().backward()
        assert q.grad is not None and q.grad.shape == (0, n), name
        for key, p in params.items():
            assert p.grad is None or torch.count_nonzero(p.grad) == 0, (name, key)
