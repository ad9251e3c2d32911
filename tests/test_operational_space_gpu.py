"""GPU: the operational-space dynamics (compute_operational_space_dynamics, csrc/operational_space.cu) against the fp64
oracle (tests/osd_oracle.py), the reference's goldens and compositions of the existing kernels; on every shipped robot and
the synthetic topology families.

Errors are per configuration, relative to that configuration's largest entry of the same output; the bound is
max(8 x the fp32 oracle's error on the same rows, 2e-5), per (robot, output), as for the dynamics derivatives."""
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor
from conftest import GOLDEN_DIR, URDFS, urdf_path
import derivatives_oracle as D
import osd_oracle as S
import synthetic_robots as SR
import tile_mirrors as TM
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL, LARGE = 131, 4099
LARGE_ROWS = torch.cat([torch.arange(SMALL, LARGE - 3, 97), torch.arange(LARGE - 3, LARGE)])
FLAGS = [(True, True), (True, False), (False, True), (False, False)]
NAMES = ("inv_inertia", "acceleration", "velocity", "bias_acceleration")
EE = {
    "2link_robot": "endEffector", "iiwa7": "iiwa_link_ee", "panda_no_gripper": "panda_virtual_ee_link",
    "panda": "panda_virtual_ee_link", "allegro_hand_description_left": "link_15.0_tip",
    "allegro_hand_description_left_small_damping": "link_3.0_tip", "trifinger_edu": "finger_tip_link_240",
    "jaco_clean": "j2n6s300_link_finger_tip_3", "jaco": "j2n6s300_link_6", "fetch_arm_no_gripper": "virtual_ee_link",
    "fetch_arm_no_gripper_small_damping": "virtual_ee_link", "iiwa7_allegro": "link_15.0_tip",
}
TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
_MODELS = {}


def model_of(stem):
    if stem not in _MODELS:
        _MODELS[stem] = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    return _MODELS[stem]


def per_config_error(got, want):
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
    assert np.isfinite(err) and err <= bound, f"{what}: per-configuration error {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def robots(stem_or_path, nonsym):
    path = urdf_path(stem_or_path) if stem_or_path in URDFS else stem_or_path
    r32 = O.load_robot(path, torch.float32)
    if nonsym:
        r32 = D.perturbed(r32)
    return r32, r32.to(torch.float64), O.link_table(r32).float().to(DEV).contiguous()


def inputs(robot, B, seed=3):
    q, qd, _ = O.sample_inputs(robot.to(torch.float64), B, seed=seed, dtype=torch.float32)
    f = torch.randn(B, robot.n_dofs, generator=torch.Generator().manual_seed(seed))
    return q, qd, f


def link_sets(stem, robot):
    """(single link, several links: the end effector -- a fixed-joint tip on most robots --, a middle link and the root)."""
    multi = [EE[stem], robot.names[len(robot.names) // 2], robot.names[0]]
    if stem in ("allegro_hand_description_left", "iiwa7_allegro"):
        multi = [EE[stem]] + [t for t in TIPS if t != EE[stem]] + [robot.names[0]]
    return [EE[stem]], list(dict.fromkeys(multi))


def pose_to_position(x, E):
    """Linear rows (and blocks) of pose-mode outputs: [B, 6E(, 6E)] -> [B, 3E(, 3E)]."""
    idx = torch.cat([torch.arange(6 * e, 6 * e + 3) for e in range(E)])
    return x[:, idx][:, :, idx] if x.ndim == 3 else x[:, idx]


class OraclePieces:
    """J / velocity / bias of a link set (pose mode), G and qdd per flag combination: each computed once per robot and rows."""

    def __init__(self, robot, q, qd, f, links):
        self.robot, self.q, self.qd, self.f, self.links = robot, q, qd, f, links
        self.J = S.stacked_jacobian(robot, q, links)
        self.bias = S.bias_acceleration(robot, q, qd, links).detach()
        self.G = S.force_response(robot, q)
        self.inv = self.J @ self.G @ self.J.transpose(1, 2)
        self.vel = torch.einsum("bmn,bn->bm", self.J, qd)

    def outputs(self, grav, damp, rows=None, position_only=False):
        qdd = O.forward_dynamics(self.robot, self.q, self.qd, self.f, grav, damp).detach()
        acc = torch.einsum("bmn,bn->bm", self.J, qdd) + self.bias
        out = [self.inv, acc, self.vel, self.bias]
        if rows is not None:
            idx = torch.cat([torch.arange(6 * e, 6 * e + 6) for e in rows])
            out = [o[:, idx][:, :, idx] if o.ndim == 3 else o[:, idx] for o in out]
        if position_only:
            out = [pose_to_position(o, o.shape[1] // 6) for o in out]
        return out


# ------------------------------------------------------------------------------------------------
# shipped robots against the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_shipped_robots_match_oracle(stem, nonsym):
    r32, r64, table = robots(stem, nonsym)
    topo = model_of(stem)._topology
    single, multi = link_sets(stem, r32)
    idx = [r32.index(nm) for nm in multi]
    for B in (SMALL, LARGE):
        q, qd, f = inputs(r32, B)
        rows = torch.arange(B) if B == SMALL else LARGE_ROWS
        sub = [t[rows] for t in (q, qd, f)]
        o64 = OraclePieces(r64, *(t.double() for t in sub), multi)
        o32 = OraclePieces(r32, *sub, multi)
        dev = [t.to(DEV) for t in (q, qd, f)]
        for grav, damp in FLAGS:
            flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
            for links, pick, pos in ((single, [0], False), (multi, None, False), (multi, None, True)):
                got = engine.operational_space_dynamics_raw(topo, [r32.index(nm) for nm in links] if links is single else idx,
                                                            table, *dev, flags, position_only=pos)
                w64 = o64.outputs(grav, damp, pick, pos)
                w32 = o32.outputs(grav, damp, pick, pos)
                for k, name in enumerate(NAMES):
                    # acceleration = J qdd + Jdot qd: on jaco_clean's light fingers qdd is large and the two terms largely
                    # cancel, so the fp32 rounding of qdd reaches about 4e-5 of the row's largest entry
                    floor = 1e-4 if name == "acceleration" else 2e-5
                    check(f"{stem} B={B} g{grav:d}d{damp:d} E={len(links)} pos={pos} {name}", got[k].cpu()[rows], w64[k], w32[k],
                          floor)


GOLDEN = ["2link_robot", "iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro"]


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".osd.npz"), allow_pickle=False)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=torch.float32)
        inertia[0] = r32.inertia[0]
        r32.inertia = inertia
    table = O.link_table(r32).float().to(DEV).contiguous()
    links = [str(s) for s in g["links"]]
    pos = bool(g["position_only"])
    q, qd, f = (torch.tensor(g[k]) for k in ("q", "qd", "f"))
    got = engine.operational_space_dynamics_raw(model_of(stem)._topology, [r32.index(nm) for nm in links], table,
                                                q.to(DEV), qd.to(DEV), f.to(DEV), engine.GRAVITY, position_only=pos)
    w64 = S.operational_space_dynamics(r32.to(torch.float64), q.double(), qd.double(), f.double(), links, True, False, pos)
    pre = "" if tag == "sym" else "nonsym."
    for k, (name, key) in enumerate(zip(NAMES, ("inv_inertia", "acceleration", "velocity", "bias"))):
        check(f"{stem} {pre}{name}", got[k].cpu(), torch.tensor(g[pre + key]), w64[k].float(), floor=2e-4)


# ------------------------------------------------------------------------------------------------
# compositions of the existing kernels
# ------------------------------------------------------------------------------------------------
CONSISTENCY = [("iiwa7", ["iiwa_link_ee"]), ("panda", ["panda_virtual_ee_link", "panda_link4"]),
               ("allegro_hand_description_left", TIPS), ("iiwa7_allegro", TIPS), ("trifinger_edu", ["finger_tip_link_0",
                                                                                              "finger_tip_link_120"])]


def stacked_jacobian_from_fk(m, q, links, position_only=False):
    out = m.compute_fk_and_jacobian_multi(q, links)
    return torch.cat([out[nm][2] if position_only else torch.cat([out[nm][2], out[nm][3]], dim=1) for nm in links], dim=1)


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem,links", CONSISTENCY)
def test_matches_compositions_of_existing_kernels(stem, links, nonsym):
    m = model_of(stem)
    r32, _, table = robots(stem, nonsym)
    topo = m._topology
    idx = [m._name_to_idx_map[nm] for nm in links]
    q, qd, f = (t.to(DEV) for t in inputs(r32, 1000, seed=5))
    for flags in (engine.GRAVITY | engine.DAMPING, 0):
        inv, acc, vel, bias = engine.operational_space_dynamics_raw(topo, idx, table, q, qd, f, flags)
        with torch.no_grad():
            J = engine.fk_jacobian_multi_raw(topo, idx, table, q)[2:]
            J = torch.cat([torch.cat([J[0][e], J[1][e]], dim=1) for e in range(len(idx))], dim=1).double()
            G = engine.forward_dynamics_derivatives_raw(topo, table, q, qd, f, flags, want_dq=False, want_dqd=False)[2].double()
            qdd = engine.forward_dynamics_raw(topo, table, q, qd, f, flags).double()
        assert per_config_error(inv, J @ G @ J.transpose(1, 2)) < 1e-4
        assert per_config_error(acc - bias, torch.einsum("bmn,bn->bm", J, qdd)) < 1e-4
        assert per_config_error(vel, torch.einsum("bmn,bn->bm", J, qd.double())) < 5e-5
    # velocity: the world-frame transport of the body-frame spatial velocities of update_kinematic_state
    if not nonsym:
        m.update_kinematic_state(q, qd)
        for e, nm in enumerate(links):
            body = m._bodies[m._name_to_idx_map[nm]]
            R = body.pose.rotation()
            lin = torch.einsum("bij,bj->bi", R, body.vel.lin)
            ang = torch.einsum("bij,bj->bi", R, body.vel.ang)
            assert per_config_error(vel[:, 6 * e:6 * e + 3], lin) < 1e-5
            assert per_config_error(vel[:, 6 * e + 3:6 * e + 6], ang) < 1e-5


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem,links", CONSISTENCY)
def test_affinity_and_structure(stem, links, nonsym):
    m = model_of(stem)
    r32, _, table = robots(stem, nonsym)
    topo = m._topology
    idx = [m._name_to_idx_map[nm] for nm in links]
    E = len(idx)
    q, qd, f = (t.to(DEV) for t in inputs(r32, 777, seed=6))
    inv, acc, vel, bias = engine.operational_space_dynamics_raw(topo, idx, table, q, qd, f, engine.GRAVITY)
    J = stacked_jacobian_from_fk(m, q, links) if not nonsym else None
    if J is not None:
        F = torch.randn(acc.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
        _, acc2, _, _ = engine.operational_space_dynamics_raw(topo, idx, table, q, qd, f + torch.einsum("bmn,bm->bn", J, F),
                                                              engine.GRAVITY)
        want = torch.einsum("bmk,bk->bm", inv.double(), F.double())
        assert per_config_error((acc2.double() - acc.double()), want) < 2e-3
    # position only = the linear rows and blocks of pose mode
    pos = engine.operational_space_dynamics_raw(topo, idx, table, q, qd, f, engine.GRAVITY, position_only=True)
    for a, b in zip(pos, (inv, acc, vel, bias)):
        assert per_config_error(a, pose_to_position(b, E)) < 1e-5
    # each diagonal block is the single-link call
    for e, l in enumerate(idx):
        one = engine.operational_space_dynamics_raw(topo, [l], table, q, qd, f, engine.GRAVITY)
        s = slice(6 * e, 6 * e + 6)
        assert per_config_error(inv[:, s, s], one[0]) < 1e-5
        for a, b in zip((acc, vel, bias), one[1:]):
            assert per_config_error(a[:, s], b) < 1e-5
    if not nonsym:                                          # J H^-1 J^T: symmetric, positive semi-definite
        sym = inv.double()
        assert per_config_error(sym, sym.transpose(1, 2)) < 1e-4
        ev = torch.linalg.eigvalsh(0.5 * (sym + sym.transpose(1, 2)))
        assert float((ev.min(1).values / ev.max(1).values.clamp_min(1e-30)).min()) > -1e-4


# ------------------------------------------------------------------------------------------------
# launch geometry, models, capture and edge cases
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem,links", [("iiwa7", ["iiwa_link_ee"]), ("iiwa7_allegro", TIPS), ("2link_robot", ["endEffector"])])
def test_rows_are_independent_of_batch_and_alignment(stem, links):
    m = model_of(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f = (t.to(DEV) for t in inputs(r32, 20011, seed=14))
    big = m.compute_operational_space_dynamics(q, qd, f, links)
    rows = torch.tensor([0, 1, 17, 5003, 20010], device=DEV)
    small = m.compute_operational_space_dynamics(q[rows], qd[rows], f[rows], links)
    for a, b in zip(big, small):
        assert torch.equal(a[rows], b)

    def shifted(t):                                     # the same values 4 bytes off 16-byte alignment
        buf = torch.empty(t.numel() + 1, device=DEV)
        v = buf[1:].view(t.shape)
        v.copy_(t)
        assert v.data_ptr() % 16 != 0
        return v
    for B in (1003, 1024):
        got = m.compute_operational_space_dynamics(shifted(q[:B]), shifted(qd[:B]), shifted(f[:B]), links)
        for a, b in zip(got, big):
            assert torch.equal(a, b[:B])


def test_learnable_and_fused_models_use_current_values():
    stem = "iiwa7"
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f = (t.to(DEV) for t in inputs(r32, 333, seed=13))
    init = torch.tensor([[0.3, 0.01, -0.02], [0.015, 0.25, 0.005], [-0.01, 0.02, 0.2]])
    models = []
    for fuse in (False, True):
        m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
        m.make_link_param_learnable("iiwa_link_3", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.clone()))
        m.make_link_param_learnable("iiwa_link_5", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.t().clone()))
        if fuse:
            m.fuse_learnable_parameters()
        models.append(m)
    table = models[0]._link_table().detach()
    links = ["iiwa_link_ee", "iiwa_link_4"]
    idx = [models[0]._name_to_idx_map[nm] for nm in links]
    want = engine.operational_space_dynamics_raw(models[0]._topology, idx, table, q, qd, f, engine.GRAVITY)
    const = model_of(stem).compute_operational_space_dynamics(q, qd, f, links)
    assert rel(want[0], const[0]) > 1e-4                 # the learnable values differ from the URDF ones
    for m in models:
        got = m.compute_operational_space_dynamics(q, qd, f, links)
        for a, b in zip(got, want):
            assert not a.requires_grad
            assert torch.equal(a, b)


def test_one_launch_per_call_and_cuda_graph_capture():
    m = model_of("iiwa7_allegro")
    r32 = O.load_robot(urdf_path("iiwa7_allegro"), torch.float32)
    q, qd, f = (t.to(DEV) for t in inputs(r32, 4099, seed=15))
    want = m.compute_operational_space_dynamics(q, qd, f, TIPS)
    torch.cuda.synchronize()
    before = engine.launch_count()
    m.compute_operational_space_dynamics(q, qd, f, TIPS, position_only=True)
    assert engine.launch_count() == before + 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_operational_space_dynamics(q, qd, f, TIPS)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = m.compute_operational_space_dynamics(q, qd, f, TIPS)
    for t in got:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_outputs_can_be_skipped():
    m = model_of("panda")
    topo = m._topology
    r32, _, table = robots("panda", False)
    q, qd, f = (t.to(DEV) for t in inputs(r32, 300, seed=18))
    idx = [m._name_to_idx_map["panda_virtual_ee_link"]]
    full = engine.operational_space_dynamics_raw(topo, idx, table, q, qd, f, engine.GRAVITY)
    for k in range(4):
        want = [j == k for j in range(4)]
        got = engine.operational_space_dynamics_raw(topo, idx, table, q, qd, f, engine.GRAVITY, False, *want)
        assert torch.equal(got[k], full[k]) and all(got[j] is None for j in range(4) if j != k)
    before = engine.launch_count()
    engine.operational_space_dynamics_raw(topo, idx, table, q, qd, f, engine.GRAVITY, False, False, False, False, False)
    assert engine.launch_count() == before


def test_edge_cases():
    m = model_of("iiwa7")
    n = m._n_dofs
    r32 = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd, f = (t.to(DEV) for t in inputs(r32, 3, seed=16))
    links = ["iiwa_link_ee", "iiwa_link_0"]
    empty = torch.zeros(0, n, device=DEV)
    out = m.compute_operational_space_dynamics(empty, empty, empty, links)
    assert out.inv_inertia.shape == (0, 12, 12) and out.acceleration.shape == (0, 12)
    one = m.compute_operational_space_dynamics(q[1], qd[1], f[1], links, False, True, True)
    full = m.compute_operational_space_dynamics(q, qd, f, links, False, True, True)
    assert one.inv_inertia.shape == (6, 6) and one.velocity.shape == (6,)
    for a, b in zip(one, full):
        assert torch.equal(a, b[1])
    # the root gets zero rows and columns
    pose = m.compute_operational_space_dynamics(q, qd, f, links)
    assert torch.all(pose.inv_inertia[:, 6:, :] == 0) and torch.all(pose.inv_inertia[:, :, 6:] == 0)
    for v in pose[1:]:
        assert torch.all(v[:, 6:] == 0)
    with pytest.raises(AssertionError):
        m.compute_operational_space_dynamics(q, qd, f, ["iiwa_link_ee", "iiwa_link_ee"])
    with pytest.raises(KeyError):
        m.compute_operational_space_dynamics(q, qd, f, ["no_such_link"])
    with pytest.raises(AssertionError):
        m.compute_operational_space_dynamics(q[:, :5], qd[:, :5], f[:, :5], links)
    with pytest.raises(AssertionError):
        m.compute_operational_space_dynamics(q, qd[:2], f, links)
    with pytest.raises(AssertionError):
        m.compute_operational_space_dynamics(q.cpu(), qd.cpu(), f.cpu(), links)
    table, topo = m._link_table(), m._topology
    for bad in ([], list(range(9)), [1, 1], [99], [-1]):
        with pytest.raises(RuntimeError, match="drmb200_operational_space_dynamics"):
            engine.operational_space_dynamics_raw(topo, bad, table, q, qd, f, 0)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        engine.operational_space_dynamics_raw(topo, [8], table, q.cpu(), qd.cpu(), f.cpu(), 0)
    with pytest.raises(RuntimeError, match="fp32-only"):
        engine.operational_space_dynamics_raw(topo, [8], table, q.double(), qd.double(), f.double(), 0)


# ------------------------------------------------------------------------------------------------
# synthetic topologies
# ------------------------------------------------------------------------------------------------
FAM = SR.families()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_osd"))


@pytest.mark.parametrize("name", sorted(FAM))
def test_synthetic_families_match_oracle_or_are_refused(name, model_dir):
    """Every flag combination, pose and position mode.  The expected outcome is the host code's (tests/tile_mirrors.py,
    pinned to it by tests/test_tile_choice.py): no family needs more than 227 KB for one row, so none is refused."""
    spec = FAM[name]
    path = SR.build(spec, model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    r32, r64, table = robots(path, True)
    names = r32.names
    links = list(dict.fromkeys([names[-1], names[len(names) // 2], names[0]]))
    idx = [r32.index(nm) for nm in links]
    par, mov = spec.doc()
    q, qd, f = inputs(r32, 37, seed=17)
    rows = torch.arange(0, 37, 4)
    sub = [t[rows] for t in (q, qd, f)]
    o64 = OraclePieces(r64, *(t.double() for t in sub), links) if r32.n_dofs else None
    o32 = OraclePieces(r32, *sub, links) if r32.n_dofs else None
    for pos in (False, True):
        tile, need = TM.osd_choice(par, mov, idx, not pos)
        assert tile is not None, f"{name}: the mirror expects a refusal ({need} B)"
        for grav, damp in FLAGS:
            flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
            got = engine.operational_space_dynamics_raw(m._topology, idx, table, q.to(DEV), qd.to(DEV), f.to(DEV), flags,
                                                        position_only=pos)
            if r32.n_dofs == 0:
                for t in got:
                    assert torch.all(t == 0)
                continue
            w64 = o64.outputs(grav, damp, None, pos)
            w32 = o32.outputs(grav, damp, None, pos)
            for k, nm in enumerate(NAMES):
                check(f"{name} T={tile} pos={pos} g{grav:d}d{damp:d} {nm}", got[k].cpu()[rows], w64[k], w32[k])
