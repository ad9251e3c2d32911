"""GPU: batched Levenberg-Marquardt inverse kinematics (compute_inverse_kinematics, csrc/inverse_kinematics.cu) against
tests/ik_oracle.py in fp64: one step on every shipped robot, chaining, honest error reports, success rate, joint limits,
joints off the path, batch / alignment independence, hard inputs, synthetic topologies, learnable models, launches, graphs
and argument errors.

One-step comparisons exclude rows whose fp64 accept margin |E' - E| / E is under 1e-3 (there fp32 rounding may decide the
other way) and count them; elsewhere the accept decision and the damping must agree and q is within max(8 x the fp32
oracle's error, 2e-5) of the fp64 oracle, absolute in radians."""
import ctypes

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor
from conftest import URDFS, urdf_path
import ik_oracle as IK
import synthetic_robots as S
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL, LARGE = 131, 4099
EE = {
    "2link_robot": "endEffector", "iiwa7": "iiwa_link_ee", "panda_no_gripper": "panda_virtual_ee_link",
    "panda": "panda_virtual_ee_link", "allegro_hand_description_left": "link_15.0_tip",
    "allegro_hand_description_left_small_damping": "link_3.0_tip", "trifinger_edu": "finger_tip_link_240",
    "jaco_clean": "j2n6s300_link_finger_tip_3", "jaco": "j2n6s300_link_6", "fetch_arm_no_gripper": "virtual_ee_link",
    "fetch_arm_no_gripper_small_damping": "virtual_ee_link", "iiwa7_allegro": "link_15.0_tip",
}
_MODELS = {}


def model_of(stem):
    if stem not in _MODELS:
        _MODELS[stem] = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    return _MODELS[stem]


def oracles(path):
    r32 = O.load_robot(path, torch.float32)
    return r32, r32.to(torch.float64)


def cuda(*ts):
    return [None if t is None else t.to(DEV) for t in ts]


def path_dofs(robot, link):
    dofs, i = set(), robot.index(link)
    while i > 0:
        if robot.dof[i] >= 0:
            dofs.add(robot.dof[i])
        i = robot.parent[i]
    return dofs


def compare_one_step(what, m, r32, r64, link, q0, tpos, tquat, limits=True):
    """max_iters = 1 against the fp64 oracle from the same fp32 inputs; returns the number of excluded margin rows."""
    lo, hi = m._joint_limit_tensors() if limits else (None, None)
    res = m.compute_inverse_kinematics(*cuda(q0), link, *cuda(tpos, tquat), max_iters=1, respect_joint_limits=limits)
    lo_c, hi_c = (None, None) if lo is None else (lo.cpu(), hi.cpu())
    w64 = IK.solve(r64, q0.double(), link, tpos, tquat, None if lo_c is None else lo_c.double(),
                   None if hi_c is None else hi_c.double(), max_iters=1)
    w32 = IK.solve(r32, q0, link, tpos, tquat, lo_c, hi_c, max_iters=1)
    keep = w64["margin"] >= 1e-3
    excluded = int((~keep).sum())
    lam = res.damping.cpu()
    acc = lam < IK.DAMPING_INIT
    assert bool((acc[keep] == w64["accepted"][keep]).all()), f"{what}: accept decisions differ"
    assert torch.allclose(lam[keep].double(), w64["damping"][keep], rtol=1e-6, atol=0), f"{what}: damping differs"
    q = res.q.cpu().double()[keep]
    e32 = float((w32["q"].double()[keep] - w64["q"][keep]).abs().max()) if bool(keep.any()) else 0.0
    err = float((q - w64["q"][keep]).abs().max()) if bool(keep.any()) else 0.0
    bound = max(8 * e32, 2e-5)
    print(f"ERR {what}: q {err:.2e} (bound {bound:.2e}), {excluded} margin rows of {q0.shape[0]}")
    assert np.isfinite(err) and err <= bound, f"{what}: q error {err:.3e} > {bound:.3e}"
    assert excluded <= max(3, q0.shape[0] // 100), f"{what}: {excluded} rows within the accept margin"
    return excluded


# ------------------------------------------------------------------------------------------------
# 1. one step against the fp64 oracle, every shipped robot
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "position"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_one_step_matches_the_fp64_oracle(stem, pose):
    m = model_of(stem)
    r32, r64 = oracles(urdf_path(stem))
    link = EE[stem]
    for B in (SMALL, LARGE):
        q0, tpos, tquat = IK.problem(r64, link, B, seed=1)
        compare_one_step(f"{stem} {'pose' if pose else 'pos'} B={B}", m, r32, r64, link, q0, tpos, tquat if pose else None)


@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper"])
def test_without_limits_matches_the_unclamped_oracle(stem):
    m = model_of(stem)
    r32, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = IK.problem(r64, EE[stem], SMALL, seed=2)
    q0 = q0 + 3.0 * torch.randn(q0.shape, generator=torch.Generator().manual_seed(2))    # far outside the limits
    compare_one_step(f"{stem} no limits", m, r32, r64, EE[stem], q0, tpos, tquat, limits=False)
    res = m.compute_inverse_kinematics(*cuda(q0), EE[stem], *cuda(tpos, tquat), max_iters=0, respect_joint_limits=False)
    assert torch.equal(res.q.cpu(), q0)


# ------------------------------------------------------------------------------------------------
# 2. chaining is exact
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem,pose", [("iiwa7", True), ("panda_no_gripper", True), ("allegro_hand_description_left", False),
                                       ("iiwa7_allegro", True)])
def test_k_iterations_equal_k_chained_single_iterations(stem, pose):
    m = model_of(stem)
    r32, r64 = oracles(urdf_path(stem))
    link = EE[stem]
    q0, tpos, tquat = cuda(*IK.problem(r64, link, LARGE, seed=3))
    tquat = tquat if pose else None
    one = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=32)
    q, damp = q0, None
    for _ in range(32):
        step = m.compute_inverse_kinematics(q, link, tpos, tquat, max_iters=1, damping=damp)
        q, damp = step.q, step.damping
    for a, b in zip(one, step):
        assert torch.equal(a, b)
    # K = 0: the clamped start and its errors
    zero = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=0)
    lo, hi = m._joint_limit_tensors()
    assert torch.equal(zero.q, torch.minimum(torch.maximum(q0, lo), hi))
    assert bool((zero.damping == IK.DAMPING_INIT).all())
    w = IK.evaluate(r64, zero.q.cpu().double(), link, tpos.cpu(), None if tquat is None else tquat.cpu())
    assert float((zero.pos_error.cpu().double() - w[3]).abs().max()) < 2e-5
    assert float((zero.rot_error.cpu().double() - w[4]).abs().max()) < 2e-5


# ------------------------------------------------------------------------------------------------
# 3 and 4. honest reports and success rate
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem,pose", [("iiwa7", True), ("panda_no_gripper", True), ("iiwa7", False)])
def test_reports_are_honest_and_the_success_rate_matches_the_oracle(stem, pose):
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    link = EE[stem]
    q0, tpos, tquat = IK.problem(r64, link, LARGE, seed=0)
    tquat = tquat if pose else None
    res = m.compute_inverse_kinematics(*cuda(q0), link, *cuda(tpos, tquat), max_iters=100)
    # the errors reported at the returned q, by the fp64 oracle's FK
    _, _, _, perr, rerr = IK.evaluate(r64, res.q.cpu().double(), link, tpos, tquat)
    dp = float((res.pos_error.cpu().double() - perr).abs().max())
    dr = float((res.rot_error.cpu().double() - rerr).abs().max())
    print(f"{stem}: reported vs fp64 errors at the returned q: pos {dp:.2e} m, rot {dr:.2e} rad")
    assert dp < 2e-6 and dr < 2e-5
    conv = res.converged.cpu()
    # converged rows are within tolerance by the oracle's measure (up to fp32 evaluation error)
    assert bool((perr[conv] <= 1e-4 + 2e-6).all()) and bool((rerr[conv] <= 1e-3 + 2e-5).all())
    lo, hi = IK.joint_limits(r64, torch.float32)
    w64 = IK.solve(r64, q0.double(), link, tpos, tquat, lo.double(), hi.double(), max_iters=100)
    got, want = float(conv.double().mean()), float(w64["converged"].double().mean())
    print(f"{stem} {'pose' if pose else 'position'}: converged kernel {got:.4f}, fp64 oracle {want:.4f}")
    assert abs(got - want) <= 0.01


# ------------------------------------------------------------------------------------------------
# 5. joint limits and joints off the path
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", ["jaco", "panda_no_gripper", "iiwa7"])
def test_returned_joints_respect_the_fp32_limits(stem):
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = IK.problem(r64, EE[stem], LARGE, seed=4, noise=2.0)
    q0 = q0 + 4.0 * torch.randn(q0.shape, generator=torch.Generator().manual_seed(4))
    lo, hi = m._joint_limit_tensors()
    for K in (0, 1, 20):
        res = m.compute_inverse_kinematics(*cuda(q0), EE[stem], *cuda(tpos, tquat), max_iters=K)
        assert bool(((res.q >= lo) & (res.q <= hi)).all())


@pytest.mark.parametrize("stem,link", [("allegro_hand_description_left", "link_3.0_tip"), ("iiwa7_allegro", "link_7.0_tip"),
                                       ("jaco", "j2n6s300_link_6")])
def test_joints_off_the_path_never_move(stem, link):
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = IK.problem(r64, link, LARGE, seed=5)
    lo, hi = m._joint_limit_tensors()
    q0 = torch.minimum(torch.maximum(q0.to(DEV), lo), hi)       # in limits: the clamp is the identity
    on = sorted(path_dofs(r64, link))
    off = [c for c in range(r64.n_dofs) if c not in on]
    assert off
    res = m.compute_inverse_kinematics(q0, link, *cuda(tpos, tquat), max_iters=20)
    assert torch.equal(res.q[:, off], q0[:, off])
    assert not torch.equal(res.q[:, on], q0[:, on])


# ------------------------------------------------------------------------------------------------
# 6. rows do not depend on the batch or on alignment
# ------------------------------------------------------------------------------------------------
def shifted(t):
    """The same values 4 bytes off 16-byte alignment."""
    buf = torch.empty(t.numel() + 1, device=DEV, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


@pytest.mark.parametrize("stem,pose", [("iiwa7", True), ("allegro_hand_description_left", False), ("panda", True)])
def test_rows_are_independent_of_batch_and_alignment(stem, pose):
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    link = EE[stem]
    q0, tpos, tquat = cuda(*IK.problem(r64, link, LARGE, seed=6))
    tquat = tquat if pose else None
    damp = 10.0 ** (-3 * torch.rand(LARGE, device=DEV) - 1)
    big = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=20, damping=damp)
    rows = torch.tensor([0, 1, 63, 64, 2048, LARGE - 1], device=DEV)
    small = m.compute_inverse_kinematics(q0[:SMALL], link, tpos[:SMALL], None if tquat is None else tquat[:SMALL],
                                         max_iters=20, damping=damp[:SMALL])
    for a, b in zip(big, small):
        assert torch.equal(a[:SMALL], b)
    for r in rows.tolist():
        one = m.compute_inverse_kinematics(q0[r], link, tpos[r], None if tquat is None else tquat[r], max_iters=20,
                                           damping=damp[r])
        for a, b in zip(big, one):
            assert torch.equal(a[r], b)
    # every input and output 4 bytes off 16-byte alignment, through the C ABI
    lo, hi = m._joint_limit_tensors()
    n = m._n_dofs
    outs = [shifted(torch.zeros(LARGE, n, device=DEV)), shifted(torch.zeros(LARGE, device=DEV)),
            shifted(torch.zeros(LARGE, device=DEV)), shifted(torch.zeros(LARGE, device=DEV, dtype=torch.uint8)),
            shifted(torch.zeros(LARGE, device=DEV))]
    ins = [shifted(t) if t is not None else None for t in (q0, tpos, tquat, lo, hi, damp)]
    ptr = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = engine.lib().drmb200_inverse_kinematics(
        ctypes.byref(m._topology), m._name_to_idx_map[link], ptr(m._link_table()), *[ptr(t) for t in ins], LARGE, 20,
        ctypes.c_float(1e-2), ctypes.c_float(1e-4), ctypes.c_float(1e-3), *[ptr(t) for t in outs],
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    outs[3] = outs[3].view(torch.bool)
    for a, b in zip(outs, big):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# 7. hard inputs, synthetic topologies, learnable models
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper"])
def test_singular_start_and_unreachable_target_stay_finite(stem):
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    link = EE[stem]
    _, tpos, tquat = cuda(*IK.problem(r64, link, SMALL, seed=7))
    zero = torch.zeros(SMALL, m._n_dofs, device=DEV)
    for quat in (tquat, None):
        res = m.compute_inverse_kinematics(zero, link, tpos, quat, max_iters=100)
        assert all(bool(torch.isfinite(t).all()) for t in (res.q, res.pos_error, res.rot_error, res.damping))
        far = tpos + torch.tensor([10.0, 0.0, 0.0], device=DEV)
        res = m.compute_inverse_kinematics(zero, link, far, quat, max_iters=100)
        assert not bool(res.converged.any())
        assert all(bool(torch.isfinite(t).all()) for t in (res.q, res.pos_error, res.rot_error, res.damping))
        assert bool((res.damping <= engine.IK_DAMPING_MAX).all()) and bool((res.pos_error > 7.0).all())


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_ik"))


@pytest.mark.parametrize("name", ["F_chain64", "F_tree64", "D_fixed", "G_one_joint"])
def test_synthetic_topologies_match_the_oracle(name, model_dir):
    path = S.build(S.families()[name], model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    r32, r64 = oracles(path)
    # the link with the most movable joints on its root path
    link = max(r64.names, key=lambda nm: (len(path_dofs(r64, nm)), nm))
    for B in (SMALL, LARGE):
        q0, tpos, tquat = IK.problem(r64, link, B, seed=8)
        for quat in (tquat, None):
            compare_one_step(f"{name} {link} B={B} {'pose' if quat is not None else 'pos'}", m, r32, r64, link, q0, tpos, quat)
    res = m.compute_inverse_kinematics(*cuda(q0), link, *cuda(tpos, tquat), max_iters=50)
    assert bool(torch.isfinite(res.q).all())


def test_learnable_and_fused_models_use_current_values():
    stem, link = "iiwa7", "iiwa_link_ee"
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = cuda(*IK.problem(r64, link, SMALL, seed=9))
    const = model_of(stem).compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=10)
    for fuse in (False, True):
        m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
        init = m._bodies[m._name_to_idx_map["iiwa_link_4"]].trans().detach().cpu().reshape(1, 3) + 0.01
        m.make_link_param_learnable("iiwa_link_4", "trans", UnconstrainedTensor(1, 3, init_tensor=init.clone()))
        if fuse:
            m.fuse_learnable_parameters()
        for _ in range(2):
            res = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=10)
            want = engine.inverse_kinematics_raw(m._topology, m._name_to_idx_map[link], m._link_table().detach(), q0, tpos,
                                                 tquat, *m._joint_limit_tensors(), max_iters=10)
            for a, b in zip(res, want):
                assert not a.requires_grad
                assert torch.equal(a, b)
            assert not torch.equal(res.q, const.q)
            with torch.no_grad():                                  # the next call must see the edited value
                p = m.fused_link_params.flat if fuse else next(iter(m._learnable_module("iiwa_link_4", "trans").parameters()))
                p.add_(0.02)


# ------------------------------------------------------------------------------------------------
# 8. launches, graphs, arguments
# ------------------------------------------------------------------------------------------------
def test_one_launch_per_call_and_cuda_graph_capture():
    m = model_of("panda_no_gripper")
    _, r64 = oracles(urdf_path("panda_no_gripper"))
    link = EE["panda_no_gripper"]
    q0, tpos, tquat = cuda(*IK.problem(r64, link, LARGE, seed=10))
    m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=1)
    torch.cuda.synchronize()
    for K in (0, 1, 100):
        before = engine.launch_count()
        m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=K)
        assert engine.launch_count() == before + 1
    want = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=30)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=30)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=30)
    for t in got:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_argument_errors_and_shapes(model_dir):
    m = model_of("iiwa7")
    n, link = m._n_dofs, EE["iiwa7"]
    _, r64 = oracles(urdf_path("iiwa7"))
    q0, tpos, tquat = cuda(*IK.problem(r64, link, 3, seed=11))
    one = m.compute_inverse_kinematics(q0[1], link, tpos[1], tquat[1], max_iters=5)
    allr = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=5)
    assert isinstance(one, drm.robot_model.InverseKinematicsResult)
    assert one.q.shape == (n,) and one.pos_error.shape == () and one.converged.dtype == torch.bool
    for a, b in zip(one, allr):
        assert torch.equal(a, b[1])
    empty = m.compute_inverse_kinematics(q0[:0], link, tpos[:0], tquat[:0])
    assert empty.q.shape == (0, n) and empty.damping.shape == (0,)
    with pytest.raises(KeyError):
        m.compute_inverse_kinematics(q0, "no_such_link", tpos)
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics(q0, link, tpos[:2])
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics(q0, link, tpos, damping=torch.ones(2, device=DEV))
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics(q0.cpu(), link, tpos.cpu())
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics(q0[:, :5], link, tpos)
    topo, table, ee = m._topology, m._link_table(), m._name_to_idx_map[link]
    lo, hi = m._joint_limit_tensors()
    bad = [dict(max_iters=-1), dict(pos_tol=-1e-4), dict(rot_tol=-1.0), dict(damping_init=0.0), dict(damping_init=-1.0)]
    for kw in bad:
        with pytest.raises(RuntimeError, match="drmb200_inverse_kinematics failed"):
            engine.inverse_kinematics_raw(topo, ee, table, q0, tpos, tquat, lo, hi, **kw)
    with pytest.raises(RuntimeError, match="both be given"):
        engine.inverse_kinematics_raw(topo, ee, table, q0, tpos, tquat, lo, None)
    with pytest.raises(RuntimeError, match="no movable joint"):
        engine.inverse_kinematics_raw(topo, 0, table, q0, tpos, tquat)
    with pytest.raises(RuntimeError, match="fp32-only"):
        engine.inverse_kinematics_raw(topo, ee, table, q0.double(), tpos, tquat)
    fixed = drm.DifferentiableRobotModel(S.build(S.families()["G_all_fixed"], model_dir), "G", device=DEV)
    z = torch.zeros(4, 0, device=DEV)
    with pytest.raises(RuntimeError, match="without movable joints"):
        engine.inverse_kinematics_raw(fixed._topology, fixed._topology.n_links - 1, fixed._link_table(), z,
                                      torch.zeros(4, 3, device=DEV))
