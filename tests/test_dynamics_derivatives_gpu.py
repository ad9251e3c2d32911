"""GPU: the dynamics Jacobians (compute_inverse_dynamics_derivatives / compute_forward_dynamics_derivatives,
csrc/dynamics_derivatives.cu) against autograd of the fp64 oracle, the reference's goldens, the adjoint kernels, the
mass-matrix kernel and the rollout kernel; on every shipped robot and the synthetic topology families.

Errors are per configuration, relative to that configuration's largest entry of the same matrix; the bound is
max(8 x the fp32 oracle's error on the same rows, 2e-5), per (robot, matrix)."""
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor
from conftest import GOLDEN_DIR, URDFS, urdf_path
import derivatives_oracle as D
import synthetic_robots as S
import tile_mirrors as TM
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL, LARGE = 131, 4099
# rows of the LARGE batch compared with the oracle: a spread over every tile plus the ragged tail
LARGE_ROWS = torch.cat([torch.arange(SMALL, LARGE - 3, 97), torch.arange(LARGE - 3, LARGE)])
ID_FLAGS = [(True, True), (True, False), (False, True), (False, False)]
FD_FLAGS = [(True, False), (True, True)]


def per_config_error(got, want):
    """max over configurations of max|got_b - want_b| / max|want_b| (configurations whose matrix is all zero: absolute)."""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, f"shape {tuple(got.shape)} vs {tuple(want.shape)}"
    if want.numel() == 0:
        return 0.0
    B = want.shape[0]
    scale = want.reshape(B, -1).abs().amax(1)
    err = (got - want).reshape(B, -1).abs().amax(1)
    return float(torch.where(scale > 0, err / scale.clamp_min(1e-300), err).max())


def check(what, got, want64, want32, floor=2e-5):
    e32 = per_config_error(want32, want64)
    err = per_config_error(got, want64)
    bound = max(8 * e32, floor)
    print(f"ERR {what}: {err:.2e} (bound {bound:.2e})")
    assert np.isfinite(err) and err <= bound, f"{what}: per-configuration error {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"


def robots(stem, nonsym):
    """fp32 / fp64 oracle robots (the fp64 one holds exactly the fp32 values) and the device table built from them."""
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if nonsym:
        r32 = D.perturbed(r32)
    r64 = r32.to(torch.float64)
    return r32, r64, O.link_table(r32).float().to(DEV).contiguous()


def inputs(robot, B, seed=3):
    q, qd, qdd = O.sample_inputs(robot.to(torch.float64), B, seed=seed, dtype=torch.float32)
    f = torch.randn(B, robot.n_dofs, generator=torch.Generator().manual_seed(seed))
    return q, qd, qdd, f


def oracle_rows(B):
    return torch.arange(B) if B == SMALL else LARGE_ROWS


def model_of(stem):
    return drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)


# ------------------------------------------------------------------------------------------------
# shipped robots against autograd of the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_shipped_robots_match_oracle_autograd(stem, nonsym):
    r32, r64, table = robots(stem, nonsym)
    m = model_of(stem)
    topo = m._topology
    folded = engine.fold_link_table(topo, table)
    for B in (SMALL, LARGE):
        q, qd, qdd, f = inputs(r32, B)
        rows = oracle_rows(B)
        dev = [t.to(DEV) for t in (q, qd, qdd, f)]
        sub = [t[rows] for t in (q, qd, qdd, f)]
        for grav, damp in ID_FLAGS:
            flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
            got = engine.inverse_dynamics_derivatives_raw(topo, table, dev[0], dev[1], dev[2], flags)
            w64 = D.inverse_dynamics_derivatives(r64, *(t.double() for t in sub[:3]), grav, damp)
            w32 = D.inverse_dynamics_derivatives(r32, *sub[:3], grav, damp)
            for k, name in enumerate(("dtau_dq", "dtau_dqd")):
                check(f"{stem} B={B} g{grav:d}d{damp:d} {name}", got[k].cpu()[rows], w64[k], w32[k])
            if folded is not None:
                pre = engine.inverse_dynamics_derivatives_raw(topo, folded, dev[0], dev[1], dev[2], flags, folded=folded)
                for a, b in zip(pre, got):
                    assert torch.equal(a, b), "prefolded rows must give the per-CTA fold's result bit for bit"
        for grav, damp in FD_FLAGS:
            flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
            got = engine.forward_dynamics_derivatives_raw(topo, table, dev[0], dev[1], dev[3], flags)
            w64 = D.forward_dynamics_derivatives(r64, sub[0].double(), sub[1].double(), sub[3].double(), grav, damp)
            w32 = D.forward_dynamics_derivatives(r32, sub[0], sub[1], sub[3], grav, damp)
            for k, name in enumerate(("dqdd_dq", "dqdd_dqd", "dqdd_df")):
                check(f"{stem} B={B} g{grav:d}d{damp:d} {name}", got[k].cpu()[rows], w64[k], w32[k])
            if folded is not None:
                pre = engine.forward_dynamics_derivatives_raw(topo, folded, dev[0], dev[1], dev[3], flags, folded=folded)
                for a, b in zip(pre, got):
                    assert torch.equal(a, b), "prefolded rows must give the per-CTA fold's result bit for bit"


# ------------------------------------------------------------------------------------------------
# the reference's own autograd Jacobians
# ------------------------------------------------------------------------------------------------
GOLDEN = ["iiwa7", "panda_no_gripper", "fetch_arm_no_gripper", "2link_robot", "allegro_hand_description_left_small_damping"]


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".deriv.npz"), allow_pickle=False)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=torch.float32)
        inertia[0] = r32.inertia[0]
        r32.inertia = inertia
    table = O.link_table(r32).float().to(DEV).contiguous()
    topo = model_of(stem)._topology
    q, qd, qdd, f = (torch.tensor(g[k]).to(DEV) for k in ("q", "qd", "qdd", "f"))
    pre = "" if tag == "sym" else "nonsym."
    # the goldens are the reference's fp32 evaluation: the bound is the fp64 oracle's distance from them
    r64 = r32.to(torch.float64)
    qc, qdc, qddc, fc = (t.double().cpu() for t in (q, qd, qdd, f))
    for grav, damp in ID_FLAGS:
        flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
        got = engine.inverse_dynamics_derivatives_raw(topo, table, q, qd, qdd, flags)
        w64 = D.inverse_dynamics_derivatives(r64, qc, qdc, qddc, grav, damp)
        for k, name in enumerate(("dq", "dqd")):
            key = f"{pre}id.g{grav:d}d{damp:d}.{name}"
            want = torch.tensor(g[key])
            check(f"{stem} {key}", got[k].cpu(), want, w64[k].float(), floor=2e-4)
    for grav, damp in FD_FLAGS:
        flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
        got = engine.forward_dynamics_derivatives_raw(topo, table, q, qd, f, flags)
        w64 = D.forward_dynamics_derivatives(r64, qc, qdc, fc, grav, damp)
        for k, name in enumerate(("dq", "dqd", "df")):
            key = f"{pre}fd.g1d{damp:d}.{name}"
            check(f"{stem} {key}", got[k].cpu(), torch.tensor(g[key]), w64[k].float(), floor=2e-4)


# ------------------------------------------------------------------------------------------------
# consistency with the other kernels
# ------------------------------------------------------------------------------------------------
CONSISTENCY = ["iiwa7", "panda", "trifinger_edu", "allegro_hand_description_left"]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", CONSISTENCY)
def test_vector_jacobian_products_match_the_adjoint_kernels(stem, nonsym):
    r32, _, table = robots(stem, nonsym)
    topo = model_of(stem)._topology
    q, qd, qdd, f = (t.to(DEV) for t in inputs(r32, 257, seed=8))
    G = torch.randn(q.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    for flags in (engine.GRAVITY | engine.DAMPING, 0):
        dq, dqd = engine.inverse_dynamics_derivatives_raw(topo, table, q, qd, qdd, flags)
        qa, qda = q.clone().requires_grad_(True), qd.clone().requires_grad_(True)
        tau = engine.InverseDynamicsFunction.apply(table, qa, qda, qdd, topo, flags)
        gq, gqd = torch.autograd.grad((G * tau).sum(), [qa, qda])
        assert rel(torch.einsum("bi,bij->bj", G, dq), gq) < 5e-5
        assert rel(torch.einsum("bi,bij->bj", G, dqd), gqd) < 5e-5
        dq, dqd, df = engine.forward_dynamics_derivatives_raw(topo, table, q, qd, f, flags)
        qa, qda, fa = q.clone().requires_grad_(True), qd.clone().requires_grad_(True), f.clone().requires_grad_(True)
        qdd_ = engine.ForwardDynamicsFunction.apply(table, qa, qda, fa, topo, flags)
        gq, gqd, gf = torch.autograd.grad((G * qdd_).sum(), [qa, qda, fa])
        assert rel(torch.einsum("bi,bij->bj", G, dq), gq) < 5e-5
        assert rel(torch.einsum("bi,bij->bj", G, dqd), gqd) < 5e-5
        assert rel(torch.einsum("bi,bij->bj", G, df), gf) < 5e-5


@pytest.mark.parametrize("stem", CONSISTENCY)
def test_force_columns_and_symmetric_models_against_the_mass_matrix(stem):
    m = model_of(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, _, f = (t.to(DEV) for t in inputs(r32, 300, seed=10))
    n = m._n_dofs
    dq, dqd, df = m.compute_forward_dynamics_derivatives(q, qd, f, True, True)
    for j in range(n):
        e = torch.zeros_like(q)
        e[:, j] = 1
        col = m.compute_forward_dynamics(q, torch.zeros_like(qd), e, False, False)
        assert rel(df[:, :, j], col) < 1e-5
    # symmetric inertias: the articulated-body algorithm inverts the RNEA, so dqdd/dx = -H^-1 dtau/dx at qdd = FD
    qdd = m.compute_forward_dynamics(q, qd, f, True, True)
    tq, tqd = m.compute_inverse_dynamics_derivatives(q, qd, qdd, True, True)
    Hinv = torch.linalg.inv(m.compute_lagrangian_inertia_matrix(q).double())
    assert rel(-Hinv @ tq.double(), dq) < 2e-3
    assert rel(-Hinv @ tqd.double(), dqd) < 2e-3
    assert rel(Hinv, df) < 2e-3


@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "trifinger_edu"])
def test_euler_step_linearisation_matches_rollout_autograd(stem):
    """A = d(q1, qd1)/d(q0, qd0), B = d(q1, qd1)/df of one semi-implicit Euler step, from the FD derivatives, against
    autograd through compute_forward_dynamics_rollout with T = 1."""
    m = model_of(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, _, f = (t.to(DEV) for t in inputs(r32, 16, seed=12))
    n, dt = m._n_dofs, 0.01
    Dq, Dqd, Df = (t.double() for t in m.compute_forward_dynamics_derivatives(q, qd, f, True, True))
    I = torch.eye(n, dtype=torch.float64, device=DEV).expand(q.shape[0], n, n)
    dqd1 = (dt * Dq, I + dt * Dqd, dt * Df)
    dq1 = tuple(dt * t for t in dqd1)
    dq1 = (I + dq1[0], dq1[1], dq1[2])
    q0, qd0, fa = q.clone().requires_grad_(True), qd.clone().requires_grad_(True), f.unsqueeze(0).clone().requires_grad_(True)
    q1, qd1, _ = m.compute_forward_dynamics_rollout(q0, qd0, fa, dt, True, True)
    for out, lin in ((q1[0], dq1), (qd1[0], dqd1)):
        for i in range(n):
            grads = torch.autograd.grad(out[:, i].sum(), [q0, qd0, fa], retain_graph=True)
            for g, L in zip(grads, lin):
                assert rel(g.reshape(-1, n), L[:, i, :]) < 1e-4, (stem, i)


# ------------------------------------------------------------------------------------------------
# learnable and fused link parameters
# ------------------------------------------------------------------------------------------------
def test_learnable_and_fused_models_equal_a_constant_model():
    stem = "iiwa7"
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd, f = (t.to(DEV) for t in inputs(r32, 333, seed=13))
    learn = model_of(stem)
    init = torch.tensor([[0.3, 0.01, -0.02], [0.015, 0.25, 0.005], [-0.01, 0.02, 0.2]])
    learn.make_link_param_learnable("iiwa_link_3", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.clone()))
    learn.make_link_param_learnable("iiwa_link_5", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.t().clone()))
    fused = model_of(stem)
    fused.make_link_param_learnable("iiwa_link_3", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.clone()))
    fused.make_link_param_learnable("iiwa_link_5", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.t().clone()))
    fused.fuse_learnable_parameters()
    # a constant model with the same values: the learnable model's table, folded once, through the prefolded entries
    table = learn._link_table().detach()
    topo = learn._topology
    folded = engine.fold_link_table(topo, table)
    want_id = engine.inverse_dynamics_derivatives_raw(topo, table, q, qd, qdd, engine.GRAVITY | engine.DAMPING, folded=folded)
    want_fd = engine.forward_dynamics_derivatives_raw(topo, table, q, qd, f, engine.GRAVITY, folded=folded)
    for m in (learn, fused):
        got_id = m.compute_inverse_dynamics_derivatives(q, qd, qdd)
        got_fd = m.compute_forward_dynamics_derivatives(q, qd, f)
        for a, b in zip(got_id + got_fd, want_id + want_fd):
            assert not a.requires_grad
            assert rel(a, b) < 1e-6


# ------------------------------------------------------------------------------------------------
# launch geometry, capture and edge cases
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", ["iiwa7", "allegro_hand_description_left", "2link_robot"])
def test_rows_are_independent_of_batch_and_alignment(stem):
    m = model_of(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd, f = (t.to(DEV) for t in inputs(r32, 20011, seed=14))
    big_id = m.compute_inverse_dynamics_derivatives(q, qd, qdd)
    big_fd = m.compute_forward_dynamics_derivatives(q, qd, f)
    rows = torch.tensor([0, 1, 17, 5003, 20010], device=DEV)
    small_id = m.compute_inverse_dynamics_derivatives(q[rows], qd[rows], qdd[rows])
    small_fd = m.compute_forward_dynamics_derivatives(q[rows], qd[rows], f[rows])
    for a, b in zip(big_id + big_fd, small_id + small_fd):
        assert torch.equal(a[rows], b)

    def shifted(t):                                     # the same values 4 bytes off 16-byte alignment
        buf = torch.empty(t.numel() + 1, device=DEV)
        v = buf[1:].view(t.shape)
        v.copy_(t)
        assert v.data_ptr() % 16 != 0
        return v
    for B in (1003, 1024):
        ids = m.compute_inverse_dynamics_derivatives(shifted(q[:B]), shifted(qd[:B]), shifted(qdd[:B]))
        fds = m.compute_forward_dynamics_derivatives(shifted(q[:B]), shifted(qd[:B]), shifted(f[:B]))
        for a, b in zip(ids + fds, big_id + big_fd):
            assert torch.equal(a, b[:B])


def test_one_launch_per_call_and_cuda_graph_capture():
    m = model_of("panda")
    r32 = O.load_robot(urdf_path("panda"), torch.float32)
    q, qd, qdd, f = (t.to(DEV) for t in inputs(r32, 4099, seed=15))
    want_id = m.compute_inverse_dynamics_derivatives(q, qd, qdd)
    want_fd = m.compute_forward_dynamics_derivatives(q, qd, f)
    torch.cuda.synchronize()
    before = engine.launch_count()
    m.compute_inverse_dynamics_derivatives(q, qd, qdd)
    assert engine.launch_count() == before + 1
    m.compute_forward_dynamics_derivatives(q, qd, f)
    assert engine.launch_count() == before + 2
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_inverse_dynamics_derivatives(q, qd, qdd)
        m.compute_forward_dynamics_derivatives(q, qd, f)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got_id = m.compute_inverse_dynamics_derivatives(q, qd, qdd)
        got_fd = m.compute_forward_dynamics_derivatives(q, qd, f)
    for t in got_id + got_fd:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(got_id + got_fd, want_id + want_fd):
        assert torch.equal(a, b)


def test_edge_cases():
    m = model_of("iiwa7")
    n = m._n_dofs
    r32 = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd, qdd, f = (t.to(DEV) for t in inputs(r32, 3, seed=16))
    empty = torch.zeros(0, n, device=DEV)
    for out in m.compute_inverse_dynamics_derivatives(empty, empty, empty) + m.compute_forward_dynamics_derivatives(empty, empty, empty):
        assert out.shape == (0, n, n)
    one_id = m.compute_inverse_dynamics_derivatives(q[1], qd[1], qdd[1], False, False)
    one_fd = m.compute_forward_dynamics_derivatives(q[1], qd[1], f[1], False, True)
    all_id = m.compute_inverse_dynamics_derivatives(q, qd, qdd, False, False)
    all_fd = m.compute_forward_dynamics_derivatives(q, qd, f, False, True)
    for a, b in zip(one_id + one_fd, all_id + all_fd):
        assert a.shape == (n, n)
        assert torch.equal(a, b[1])
    with pytest.raises(AssertionError):
        m.compute_inverse_dynamics_derivatives(q[:, :5], qd[:, :5], qdd[:, :5])
    with pytest.raises(AssertionError):
        m.compute_forward_dynamics_derivatives(q, qd[:2], f)
    with pytest.raises(AssertionError):
        m.compute_inverse_dynamics_derivatives(q.cpu(), qd.cpu(), qdd.cpu())
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        engine.forward_dynamics_derivatives_raw(m._topology, m._link_table(), q.cpu(), qd.cpu(), f.cpu(), 0)
    with pytest.raises(RuntimeError, match="fp32-only"):
        engine.inverse_dynamics_derivatives_raw(m._topology, m._link_table(), q.double(), qd.double(), qdd.double(), 0)


# ------------------------------------------------------------------------------------------------
# synthetic topologies
# ------------------------------------------------------------------------------------------------
FAM = S.families()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_deriv"))


@pytest.mark.parametrize("name", sorted(FAM))
def test_synthetic_families_match_oracle_or_are_refused(name, model_dir):
    spec = FAM[name]
    path = S.build(spec, model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    r32 = O.load_robot(path, torch.float32)
    for i, nm in enumerate(r32.names):                 # every third abstract link non-symmetric, in any document order
        k = int(nm[1:])
        if k % 3 == 1:
            gen = torch.Generator().manual_seed(k)
            r32.inertia[i] += 0.05 * r32.inertia[i].abs().max() * torch.randn(3, 3, generator=gen)
    r64 = r32.to(torch.float64)
    n = r32.n_dofs
    table = O.link_table(r32).float().to(DEV).contiguous()
    topo = m._topology
    par, mov = spec.doc()
    if n == 0:
        z = torch.zeros(5, 0, device=DEV)
        assert engine.inverse_dynamics_derivatives_raw(topo, table, z, z, z, 3)[0].shape == (5, 0, 0)
        assert engine.forward_dynamics_derivatives_raw(topo, table, z, z, z, 1)[2].shape == (5, 0, 0)
        return
    for fd in (False, True):
        # the outcome the host code gives (tests/tile_mirrors.py, pinned to it by tests/test_tile_choice.py)
        tile, need = TM.deriv_choice(*TM.deriv_program(par, mov), fd)
        call = (lambda: engine.forward_dynamics_derivatives_raw(topo, table, *inp, flags)) if fd else \
            (lambda: engine.inverse_dynamics_derivatives_raw(topo, table, *inp, flags))
        q, qd, qdd, f = inputs(r32, LARGE, seed=17)
        for B in (SMALL, LARGE):
            inp = [t[:B].to(DEV) for t in ((q, qd, f) if fd else (q, qd, qdd))]
            if tile is None:
                flags = 3
                before = engine.launch_count()
                with pytest.raises(RuntimeError, match=rf"needs {need} B of shared memory per CTA"):
                    call()
                assert engine.launch_count() == before
                break
            rows = oracle_rows(B)
            sub = [t[rows] for t in (q, qd, f if fd else qdd)]
            fn = D.forward_dynamics_derivatives if fd else D.inverse_dynamics_derivatives
            for grav, damp in ((True, not fd), (True, True)) if fd else ((True, True),):
                flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
                got = call()
                w64 = fn(r64, *(t.double() for t in sub), grav, damp)
                w32 = fn(r32, *sub, grav, damp)
                for k in range(len(got)):
                    check(f"{name} {'FD' if fd else 'ID'} TC={tile} B={B} g{grav:d}d{damp:d} out{k}", got[k].cpu()[rows], w64[k],
                          w32[k])


def test_nine_slot_model_is_refused_like_rnea_and_aba(model_dir):
    spec = S.refusal_families()["H_nine_slots"]
    m = drm.DifferentiableRobotModel(S.build(spec, model_dir), "H", device=DEV)
    z = torch.zeros(5, m._n_dofs, device=DEV)
    for call in (m.compute_inverse_dynamics, m.compute_forward_dynamics, m.compute_inverse_dynamics_derivatives,
                 m.compute_forward_dynamics_derivatives):
        with pytest.raises(RuntimeError, match="more than 8 live branch points"):
            call(z, z, z)
