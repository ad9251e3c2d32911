"""GPU: multi-link Levenberg-Marquardt inverse kinematics (compute_inverse_kinematics_multi, csrc/inverse_kinematics_multi.cu)
against tests/ik_multi_oracle.py in fp64: one step on hands and arm + hand trees in both the task-space and the joint-space
system, bit-identity with the single-link kernel for one link, chaining, honest error reports, success rate, joint limits,
joints outside the union of the paths, batch / alignment independence, synthetic topologies, learnable models, launches,
graphs and argument errors.

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
import ik_multi_oracle as IKM
import ik_oracle as IK
import synthetic_robots as S
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL, LARGE = 131, 4099
TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
JACO_TIPS = ["j2n6s300_link_finger_tip_1", "j2n6s300_link_finger_tip_2", "j2n6s300_link_finger_tip_3"]
CASES = {
    "allegro_4tips": ("allegro_hand_description_left", TIPS),
    "trifinger_3tips": ("trifinger_edu", ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"]),
    "iiwa7_allegro_4tips": ("iiwa7_allegro", TIPS),
    "jaco_3tips": ("jaco", JACO_TIPS),
    "jaco_3tips_ee": ("jaco", JACO_TIPS + ["j2n6s300_end_effector"]),
}
# the single-link kernel's test links (tests/test_inverse_kinematics_gpu.py)
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


def space(robot, links, pose):
    M = (6 if pose else 3) * len(links)
    return "task" if M <= len(IKM.union_dofs(robot, links)) else "joint"


def compare_one_step(what, m, r32, r64, links, q0, tpos, tquat, limits=True):
    """max_iters = 1 against the fp64 oracle from the same fp32 inputs; returns the number of excluded margin rows."""
    lo, hi = m._joint_limit_tensors() if limits else (None, None)
    res = m.compute_inverse_kinematics_multi(*cuda(q0), links, *cuda(tpos, tquat), max_iters=1, respect_joint_limits=limits)
    lo_c, hi_c = (None, None) if lo is None else (lo.cpu(), hi.cpu())
    w64 = IKM.solve(r64, q0.double(), links, tpos, tquat, None if lo_c is None else lo_c.double(),
                    None if hi_c is None else hi_c.double(), max_iters=1)
    w32 = IKM.solve(r32, q0, links, tpos, tquat, lo_c, hi_c, max_iters=1)
    keep = w64["margin"] >= 1e-3
    excluded = int((~keep).sum())
    lam = res.damping.cpu()
    acc = lam < IKM.DAMPING_INIT
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
# 1. one step against the fp64 oracle, both systems
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "position"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_one_step_matches_the_fp64_oracle(case, pose):
    stem, links = CASES[case]
    m = model_of(stem)
    r32, r64 = oracles(urdf_path(stem))
    sp = space(r64, links, pose)
    for B in (SMALL, LARGE):
        q0, tpos, tquat = IKM.problem(r64, links, B, seed=1)
        compare_one_step(f"{case} {'pose' if pose else 'pos'} {sp} B={B}", m, r32, r64, links, q0, tpos, tquat if pose else None)


def test_the_cases_exercise_both_systems():
    want = {("allegro_4tips", False): "task", ("allegro_4tips", True): "joint", ("trifinger_3tips", False): "task",
            ("iiwa7_allegro_4tips", True): "joint", ("iiwa7_allegro_4tips", False): "task", ("jaco_3tips_ee", False): "task"}
    for (case, pose), sp in want.items():
        stem, links = CASES[case]
        assert space(O.load_robot(urdf_path(stem), torch.float64), links, pose) == sp, (case, pose)


# ------------------------------------------------------------------------------------------------
# 2. one link: the single-link kernel, bit for bit where the system is the same
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "position"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_one_link_equals_the_single_link_kernel(stem, pose):
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    link = EE[stem]
    q0, tpos, tquat = cuda(*IK.problem(r64, link, LARGE, seed=2))
    tquat = tquat if pose else None
    damp = 10.0 ** (-3 * torch.rand(LARGE, device=DEV) - 1)
    for K in (1, 20):
        one = m.compute_inverse_kinematics(q0, link, tpos, tquat, max_iters=K, damping=damp)
        multi = m.compute_inverse_kinematics_multi(q0, [link], tpos[None], None if tquat is None else tquat[None],
                                                   max_iters=K, damping=damp)
        assert multi.pos_error.shape == (1, LARGE) and multi.rot_error.shape == (1, LARGE)
        if space(r64, [link], pose) == "task":
            for a, b in zip((multi.q, multi.pos_error[0], multi.rot_error[0], multi.converged, multi.damping), one):
                assert torch.equal(a, b)
        elif K == 1:
            # M > n_u: the joint-space system, the same step up to fp32 rounding, which J^T J (the square of J's
            # condition number) amplifies near singular starts: within 1e-3 rad.  Rows whose accept decision differs (a
            # trial error within rounding of the start's) are at most 1 %.
            same = multi.damping == one.damping
            assert int((~same).sum()) <= LARGE // 100
            dq = float((multi.q - one.q)[same].abs().max())
            print(f"{stem} {'pose' if pose else 'pos'} joint space vs task space: q {dq:.2e}, {int((~same).sum())} decisions differ")
            assert dq <= 1e-3


# ------------------------------------------------------------------------------------------------
# 3. chaining is exact
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,pose", [("iiwa7_allegro_4tips", True), ("allegro_4tips", False), ("jaco_3tips_ee", True)])
def test_k_iterations_equal_k_chained_single_iterations(case, pose):
    stem, links = CASES[case]
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = cuda(*IKM.problem(r64, links, LARGE, seed=3))
    tquat = tquat if pose else None
    one = m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=24)
    q, damp = q0, None
    for _ in range(24):
        step = m.compute_inverse_kinematics_multi(q, links, tpos, tquat, max_iters=1, damping=damp)
        q, damp = step.q, step.damping
    for a, b in zip(one, step):
        assert torch.equal(a, b)
    zero = m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=0)
    lo, hi = m._joint_limit_tensors()
    assert torch.equal(zero.q, torch.minimum(torch.maximum(q0, lo), hi))
    assert bool((zero.damping == IKM.DAMPING_INIT).all())


# ------------------------------------------------------------------------------------------------
# 4. honest reports and success rate
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,pose", [("iiwa7_allegro_4tips", True), ("allegro_4tips", True), ("allegro_4tips", False)])
def test_reports_are_honest_and_the_success_rate_matches_the_oracle(case, pose):
    stem, links = CASES[case]
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = IKM.problem(r64, links, LARGE, seed=0)
    tquat = tquat if pose else None
    res = m.compute_inverse_kinematics_multi(*cuda(q0), links, *cuda(tpos, tquat), max_iters=100)
    _, _, _, perr, rerr = IKM.evaluate(r64, res.q.cpu().double(), links, tpos.double(),
                                       None if tquat is None else tquat.double())
    dp = float((res.pos_error.cpu().double() - perr).abs().max())
    dr = float((res.rot_error.cpu().double() - rerr).abs().max())
    print(f"{case}: reported vs fp64 errors at the returned q: pos {dp:.2e} m, rot {dr:.2e} rad")
    assert dp < 4e-6 and dr < 4e-5
    conv = res.converged.cpu()
    within = ((res.pos_error <= 1e-4) & (res.rot_error <= 1e-3)).all(0).cpu()
    assert torch.equal(conv, within)                     # converged is exactly the tolerance test on the reported errors
    assert bool((perr[:, conv] <= 1e-4 + 4e-6).all()) and bool((rerr[:, conv] <= 1e-3 + 4e-5).all())
    lo, hi = IK.joint_limits(r64, torch.float32)
    w64 = IKM.solve(r64, q0.double(), links, tpos, tquat, lo.double(), hi.double(), max_iters=100)
    got, want = float(conv.double().mean()), float(w64["converged"].double().mean())
    print(f"{case} {'pose' if pose else 'position'}: converged kernel {got:.4f}, fp64 oracle {want:.4f}")
    assert abs(got - want) <= 0.01


# ------------------------------------------------------------------------------------------------
# 5. joint limits and joints outside the union of the paths
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["jaco_3tips_ee", "iiwa7_allegro_4tips"])
def test_returned_joints_respect_the_fp32_limits(case):
    stem, links = CASES[case]
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = IKM.problem(r64, links, LARGE, seed=4, noise=2.0)
    q0 = q0 + 4.0 * torch.randn(q0.shape, generator=torch.Generator().manual_seed(4))
    lo, hi = m._joint_limit_tensors()
    for K in (0, 1, 20):
        for quat in (tquat, None):
            res = m.compute_inverse_kinematics_multi(*cuda(q0), links, *cuda(tpos, quat), max_iters=K)
            assert bool(((res.q >= lo) & (res.q <= hi)).all())


@pytest.mark.parametrize("stem,links", [("allegro_hand_description_left", ["link_3.0_tip", "link_7.0_tip"]),
                                        ("iiwa7_allegro", ["link_3.0_tip", "link_11.0_tip"])])
def test_joints_outside_the_union_never_move(stem, links):
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = IKM.problem(r64, links, LARGE, seed=5)
    lo, hi = m._joint_limit_tensors()
    q0 = torch.minimum(torch.maximum(q0.to(DEV), lo), hi)       # in limits: the clamp is the identity
    on = IKM.union_dofs(r64, links)
    off = [c for c in range(r64.n_dofs) if c not in on]
    assert off
    for quat in (tquat, None):
        res = m.compute_inverse_kinematics_multi(q0, links, *cuda(tpos, quat), max_iters=20)
        assert torch.equal(res.q[:, off], q0[:, off])
        assert not torch.equal(res.q[:, on], q0[:, on])


# ------------------------------------------------------------------------------------------------
# 6. rows do not depend on the batch or on alignment
# ------------------------------------------------------------------------------------------------
def rows(res, r):
    """Rows r of a result: q, converged and damping are [B, ...], the per-link errors [n_ee, B]."""
    q, pos_err, rot_err, converged, damping = res
    return q[r], pos_err[:, r], rot_err[:, r], converged[r], damping[r]


def shifted(t):
    """The same values 4 bytes off 16-byte alignment."""
    buf = torch.empty(t.numel() + 1, device=DEV, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


@pytest.mark.parametrize("case,pose", [("iiwa7_allegro_4tips", True), ("allegro_4tips", False), ("trifinger_3tips", True)])
def test_rows_are_independent_of_batch_and_alignment(case, pose):
    stem, links = CASES[case]
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = cuda(*IKM.problem(r64, links, LARGE, seed=6))
    tquat = tquat if pose else None
    damp = 10.0 ** (-3 * torch.rand(LARGE, device=DEV) - 1)
    big = m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=20, damping=damp)
    small = m.compute_inverse_kinematics_multi(q0[:SMALL], links, tpos[:, :SMALL].contiguous(),
                                               None if tquat is None else tquat[:, :SMALL].contiguous(),
                                               max_iters=20, damping=damp[:SMALL])
    for a, b in zip(rows(big, slice(0, SMALL)), small):
        assert torch.equal(a, b)
    for r in (0, 1, 63, 64, 2048, LARGE - 1):
        one = m.compute_inverse_kinematics_multi(q0[r], links, tpos[:, r], None if tquat is None else tquat[:, r],
                                                 max_iters=20, damping=damp[r])
        assert one.q.shape == (m._n_dofs,) and one.pos_error.shape == (len(links),) and one.converged.shape == ()
        for a, b in zip(rows(big, r), one):
            assert torch.equal(a, b)
    # every input and output 4 bytes off 16-byte alignment, through the C ABI
    lo, hi = m._joint_limit_tensors()
    n, E = m._n_dofs, len(links)
    outs = [shifted(torch.zeros(LARGE, n, device=DEV)), shifted(torch.zeros(E, LARGE, device=DEV)),
            shifted(torch.zeros(E, LARGE, device=DEV)), shifted(torch.zeros(LARGE, device=DEV, dtype=torch.uint8)),
            shifted(torch.zeros(LARGE, device=DEV))]
    ins = [shifted(t) if t is not None else None for t in (q0, tpos, tquat, lo, hi, damp)]
    ptr = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    idx = (ctypes.c_int32 * E)(*[m._name_to_idx_map[l] for l in links])
    rc = engine.lib().drmb200_inverse_kinematics_multi(
        ctypes.byref(m._topology), E, idx, ptr(m._link_table()), *[ptr(t) for t in ins], LARGE, 20,
        ctypes.c_float(1e-2), ctypes.c_float(1e-4), ctypes.c_float(1e-3), *[ptr(t) for t in outs],
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    outs[3] = outs[3].view(torch.bool)
    for a, b in zip(outs, big):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# 7. synthetic topologies, learnable models
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_ik_multi"))


def path_dofs(robot, link):
    return IKM.union_dofs(robot, [link])


@pytest.mark.parametrize("name", ["F_chain64", "F_tree64", "A_bfs_movable_palm", "C_random", "D_fixed"])
def test_synthetic_topologies_match_the_oracle(name, model_dir):
    """Eight links (or all with a movable joint on their path) with the deepest paths.  The largest models fit: one row
    needs at most 2n + 2 M n_u + 2 M + 7 n_ee + m (m + 1) / 2 + m + 6 n_u + 96 floats (M <= 48, n, n_u <= 63,
    m = min(M, n_u), 8 branch slots of 12) plus 12 per walked link and 2n per CTA: under 36 KB, far below 227 KB."""
    path = S.build(S.families()[name], model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    r32, r64 = oracles(path)
    links = sorted((nm for nm in r64.names if path_dofs(r64, nm)), key=lambda nm: (-len(path_dofs(r64, nm)), nm))[:8]
    n, n_u, M = r64.n_dofs, len(IKM.union_dofs(r64, links)), 6 * len(links)
    mm = min(M, n_u)
    floats = 2 * n + 2 * M * n_u + 2 * M + 7 * len(links) + mm * (mm + 1) // 2 + mm + 6 * n_u + 96 + 12 * 63 + 2 * n
    assert floats * 4 < 227 * 1024
    for B in (SMALL, LARGE):
        q0, tpos, tquat = IKM.problem(r64, links, B, seed=8)
        for quat in (tquat, None):
            compare_one_step(f"{name} {len(links)} links B={B} {'pose' if quat is not None else 'pos'} "
                             f"{space(r64, links, quat is not None)}", m, r32, r64, links, q0, tpos, quat)
    res = m.compute_inverse_kinematics_multi(*cuda(q0), links, *cuda(tpos, tquat), max_iters=50)
    assert bool(torch.isfinite(res.q).all())


def test_learnable_and_fused_models_use_current_values():
    stem, links = "iiwa7", ["iiwa_link_ee", "iiwa_link_5"]
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = cuda(*IKM.problem(r64, links, SMALL, seed=9))
    const = model_of(stem).compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=10)
    for fuse in (False, True):
        m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
        init = m._bodies[m._name_to_idx_map["iiwa_link_4"]].trans().detach().cpu().reshape(1, 3) + 0.01
        m.make_link_param_learnable("iiwa_link_4", "trans", UnconstrainedTensor(1, 3, init_tensor=init.clone()))
        if fuse:
            m.fuse_learnable_parameters()
        for _ in range(2):
            res = m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=10)
            want = engine.inverse_kinematics_multi_raw(m._topology, [m._name_to_idx_map[l] for l in links],
                                                       m._link_table().detach(), q0, tpos, tquat, *m._joint_limit_tensors(),
                                                       max_iters=10)
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
    stem, links = CASES["iiwa7_allegro_4tips"]
    m = model_of(stem)
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = cuda(*IKM.problem(r64, links, LARGE, seed=10))
    m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=1)
    torch.cuda.synchronize()
    for K in (0, 1, 100):
        before = engine.launch_count()
        m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=K)
        assert engine.launch_count() == before + 1
    want = m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=30)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=30)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=30)
    for t in got:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_argument_errors_and_shapes(model_dir):
    stem, links = CASES["allegro_4tips"]
    m = model_of(stem)
    n = m._n_dofs
    _, r64 = oracles(urdf_path(stem))
    q0, tpos, tquat = cuda(*IKM.problem(r64, links, 3, seed=11))
    one = m.compute_inverse_kinematics_multi(q0[1], links, tpos[:, 1], tquat[:, 1], max_iters=5)
    allr = m.compute_inverse_kinematics_multi(q0, links, tpos, tquat, max_iters=5)
    assert isinstance(one, drm.robot_model.InverseKinematicsResult)
    assert one.q.shape == (n,) and one.pos_error.shape == (4,) and one.converged.dtype == torch.bool
    for a, b in zip(one, rows(allr, 1)):
        assert torch.equal(a, b)
    empty = m.compute_inverse_kinematics_multi(q0[:0], links, tpos[:, :0], tquat[:, :0])
    assert empty.q.shape == (0, n) and empty.pos_error.shape == (4, 0) and empty.damping.shape == (0,)
    with pytest.raises(KeyError):
        m.compute_inverse_kinematics_multi(q0, ["no_such_link"], tpos[:1])
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics_multi(q0, links, tpos[:, :2])
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics_multi(q0, links, tpos[:3])
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics_multi(q0, links, tpos, tquat[:, :, :3])
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics_multi(q0, links, tpos, damping=torch.ones(2, device=DEV))
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics_multi(q0.cpu(), links, tpos.cpu())
    with pytest.raises(AssertionError):
        m.compute_inverse_kinematics_multi(q0[:, :5], links, tpos)
    topo, table = m._topology, m._link_table()
    idx = [m._name_to_idx_map[l] for l in links]
    lo, hi = m._joint_limit_tensors()
    bad = [dict(max_iters=-1), dict(pos_tol=-1e-4), dict(rot_tol=-1.0), dict(damping_init=0.0), dict(damping_init=-1.0)]
    for kw in bad:
        with pytest.raises(RuntimeError, match="drmb200_inverse_kinematics_multi failed"):
            engine.inverse_kinematics_multi_raw(topo, idx, table, q0, tpos, tquat, lo, hi, **kw)
    with pytest.raises(RuntimeError, match="both be given"):
        engine.inverse_kinematics_multi_raw(topo, idx, table, q0, tpos, tquat, lo, None)
    with pytest.raises(RuntimeError, match="n_ee=0"):
        engine.inverse_kinematics_multi_raw(topo, [], table, q0, tpos[:0], tquat[:0])
    nine = [i for i in range(1, topo.n_links)][:9]
    z9 = torch.zeros(9, 3, 3, device=DEV)
    with pytest.raises(RuntimeError, match="n_ee=9"):
        engine.inverse_kinematics_multi_raw(topo, nine, table, q0, z9)
    with pytest.raises(RuntimeError, match="requested twice"):
        engine.inverse_kinematics_multi_raw(topo, [idx[0], idx[0]], table, q0, tpos[:2], tquat[:2])
    with pytest.raises(RuntimeError, match="no movable joint"):
        engine.inverse_kinematics_multi_raw(topo, [idx[0], 0], table, q0, tpos[:2], tquat[:2])
    with pytest.raises(RuntimeError, match="fp32-only"):
        engine.inverse_kinematics_multi_raw(topo, idx, table, q0.double(), tpos, tquat)
    fixed = drm.DifferentiableRobotModel(S.build(S.families()["G_all_fixed"], model_dir), "G", device=DEV)
    z = torch.zeros(4, 0, device=DEV)
    with pytest.raises(RuntimeError, match="without movable joints"):
        engine.inverse_kinematics_multi_raw(fixed._topology, [fixed._topology.n_links - 1], fixed._link_table(), z,
                                            torch.zeros(1, 4, 3, device=DEV))
