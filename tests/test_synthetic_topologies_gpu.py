"""GPU: every entry point on the synthetic topology families of tests/synthetic_robots.py, against the fp64 oracle.

The shipped URDFs are all depth-first, have at most one live branch point and at most 29 links; these families reach
what the engine accepts beyond that: 8 live branch-point slots (breadth-first hands), nested branches in random
parents-first orders, runs and branch points of fixed links, massless links, unfoldable models, 64-link chains and
trees, and degenerate models.  Each family runs at a ragged batch (131) and a multi-tile one (4 099, checked on a
sample of rows); a third of the links carry non-symmetric inertias.

Tolerance: for each model and output the fp32 oracle is measured against the fp64 oracle on the same inputs, and the
kernel's family-relative error (max |err| / max |fp64 value| over the output) must be at most max(8 x that, 2e-5).
Models the engine must refuse are in REFUSALS, each with the outcome the host code gives for it.
"""
import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar, UnconstrainedTensor
import synthetic_robots as S
from rollout_oracle import forward_dynamics_rollout as oracle_rollout
from test_backward_gpu import shifted
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FAM = S.families()
SMALL, LARGE = 131, 4099
SMEM_CAP = 227 * 1024


# ------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------
class Model:
    """One family: the product model (topology), the fp64 / fp32 oracle robots with the same non-symmetric inertias,
    and the device table built from them."""

    def __init__(self, name, directory):
        self.spec = FAM[name]
        self.path = S.build(self.spec, directory)
        self.m = drm.DifferentiableRobotModel(self.path, name, device=DEV)
        self.topo = self.m._topology
        r32 = O.load_robot(self.path, torch.float32)
        for i, nm in enumerate(r32.names):                 # every third abstract link non-symmetric, in any document order
            k = int(nm[1:])
            if k % 3 == 1:
                gen = torch.Generator().manual_seed(k)
                r32.inertia[i] += 0.05 * r32.inertia[i].abs().max() * torch.randn(3, 3, generator=gen)
        self.r32, self.r64 = r32, r32.to(torch.float64)
        self.n, self.N = r32.n_dofs, len(r32.names)
        self.table = O.link_table(self.r32).float().to(DEV).contiguous()
        self.folded = engine.fold_link_table(self.topo, self.table)
        par, mov = self.spec.doc()
        self.slots, self.red_slots, self.foldable = S.live_slots(par), S.live_slots(S.reduced_parents(par, mov)), S.foldable(par, mov)
        self.leaves = S.leaves(par) or [0]

    def inputs(self, seed):
        """q, qd, qdd, f for LARGE rows (fp32 values); the SMALL batch is the first SMALL rows."""
        q, qd, qdd = O.sample_inputs(self.r64, LARGE, seed=seed, dtype=torch.float32)
        f = torch.randn(LARGE, self.n, generator=torch.Generator().manual_seed(seed))
        return q, qd, qdd, f


_MODELS = {}


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_gpu"))


def get(name, directory):
    if name not in _MODELS:
        _MODELS[name] = Model(name, directory)
    return _MODELS[name]


# rows of the LARGE batch compared with the oracle: a spread over every tile plus the ragged tail
LARGE_ROWS = torch.cat([torch.arange(SMALL, LARGE - 3, 61), torch.arange(LARGE - 3, LARGE)])
ORACLE_ROWS = torch.cat([torch.arange(SMALL), LARGE_ROWS])


def split(t, dim=0):
    """Kernel outputs of the SMALL and LARGE runs -> the rows the oracle evaluated (ORACLE_ROWS order)."""
    small, large = t
    return torch.cat([small.index_select(dim, torch.arange(SMALL, device=small.device)),
                      large.index_select(dim, LARGE_ROWS.to(large.device))], dim=dim)


def check(what, got, want64, want32, floor=2e-5):
    """Family-relative error of the kernel vs the fp64 oracle, bounded by max(8 x the fp32 oracle's, floor)."""
    got, want64, want32 = got.detach().double().cpu(), want64.detach().double().cpu(), want32.detach().double().cpu()
    assert got.shape == want64.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(want64.shape)}"
    if want64.numel() == 0:
        return
    scale = float(want64.abs().max())
    if scale == 0.0:                                   # e.g. the Jacobian of a joint's own origin: rounding only
        assert float(got.abs().max()) <= 1e-6, what
        return
    e32 = float((want32 - want64).abs().max()) / scale
    err = float((got - want64).abs().max()) / scale
    bound = max(8 * e32, floor)
    print(f"ERR {what}: {err:.2e} (bound {bound:.2e})")
    assert np.isfinite(err) and err <= bound, f"{what}: family-relative error {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"


def both(fn, r64, r32, *args):
    """fn evaluated by the fp64 and the fp32 oracle on the same (fp32-valued) inputs."""
    return fn(r64, *(a.double() if torch.is_tensor(a) else a for a in args)), fn(r32, *(a.float() if torch.is_tensor(a) else a for a in args))


def oracle_kinematics(robot, q, links):
    """pos, quat, lin / ang Jacobians of `links`, from one kinematic_state pass."""
    R, p, _, _, _ = O.kinematic_state(robot, q)
    B, n = q.shape[0], robot.n_dofs
    out = []
    for e in links:
        lin, ang = torch.zeros(B, 3, n, dtype=q.dtype), torch.zeros(B, 3, n, dtype=q.dtype)
        i = e
        while i > 0:
            if robot.dof[i] >= 0:
                z = R[i] @ robot.axis[i]
                lin[:, :, robot.dof[i]] = torch.cross(z, p[e] - p[i], dim=-1)
                ang[:, :, robot.dof[i]] = z
            i = robot.parent[i]
        out.append((p[e], O.quaternion(R[e]), lin, ang))
    return out


def oracle_mass_matrix(robot, q):
    """Column j = ID(q, 0, e_j) - ID(q, 0, 0) (robot_model.py:403-450), all columns in one stacked evaluation."""
    B, n = q.shape
    qq = q.repeat(n + 1, 1)
    qdd = torch.zeros(n + 1, B, n, dtype=q.dtype)
    idx = torch.arange(n)
    qdd[idx, :, idx] = 1
    tau = O.inverse_dynamics(robot, qq, torch.zeros_like(qq), qdd.reshape(-1, n), True, False).reshape(n + 1, B, n)
    return (tau[:n] - tau[n:]).permute(1, 2, 0)


def align_quat(quat, want):
    """Quaternions are defined up to sign: take the kernel's sign per row from the fp64 oracle's."""
    sign = torch.sign((quat.double().cpu() * want).sum(-1, keepdim=True))
    return quat.double().cpu() * torch.where(sign == 0, torch.ones_like(sign), sign)


def mm_smem_bytes(model):
    """Shared memory of the mass-matrix kernel (MmSmemLayout and the tile choice of mass_matrix_device_impl)."""
    folded = model.foldable
    N = 1 + model.n if folded else model.N
    slots = model.red_slots if folded else model.slots
    n = model.n

    def floats(T):
        o = T * n * n + T * n
        o = (o + 3) & ~3
        return o + N * 28 + N * 8 * T + slots * 6 * T
    return 4 * (floats(64) if 4 * floats(64) <= 113 * 1024 else floats(32))


RUNNABLE = sorted(FAM)


# ------------------------------------------------------------------------------------------------
# kinematics
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", RUNNABLE)
def test_kinematics_match_the_oracle(name, model_dir):
    M = get(name, model_dir)
    if M.n == 0:
        assert (name, "fk") in REFUSALS                        # checked there
        return
    q = M.inputs(1)[0]
    qo = q[ORACLE_ROWS]
    qg = q.to(DEV)
    links = M.leaves
    want64, want32 = both(oracle_kinematics, M.r64, M.r32, qo, links)
    for k, e in enumerate(links):                      # single-end-effector FK + Jacobian of every leaf
        outs = [engine.fk_jacobian_raw(M.topo, e, M.table, qg[:B].contiguous()) for B in (SMALL, LARGE)]
        pos, quat, jl, ja = (split([o[c] for o in outs]) for c in range(4))
        check(f"{name} fk pos l{e}", pos, want64[k][0], want32[k][0])
        check(f"{name} fk quat l{e}", align_quat(quat, want64[k][1]), want64[k][1], want32[k][1])
        check(f"{name} fk jac l{e}", torch.stack([jl, ja]), torch.stack(want64[k][2:]), torch.stack(want32[k][2:]))
    ee = links[:8]                                     # one multi-end-effector walk
    outs = [engine.fk_jacobian_multi_raw(M.topo, ee, M.table, qg[:B].contiguous()) for B in (SMALL, LARGE)]
    for c, tag in enumerate(("pos", "quat", "jlin", "jang")):
        got = split([o[c] for o in outs], dim=1)
        w64 = torch.stack([w[c] for w in want64[:len(ee)]])
        w32 = torch.stack([w[c] for w in want32[:len(ee)]])
        if tag == "quat":
            got = align_quat(got, w64)
        check(f"{name} fk_multi {tag}", got, w64, w32)


@pytest.mark.parametrize("name", RUNNABLE)
def test_kinematic_state_and_all_links_match_the_oracle(name, model_dir):
    M = get(name, model_dir)
    if M.n == 0:
        assert (name, "kinematic_state") in REFUSALS
        return
    q, qd = M.inputs(2)[:2]
    (R64, p64, w64, v64, _), (R32, p32, w32, v32, _) = both(O.kinematic_state, M.r64, M.r32, q[ORACLE_ROWS], qd[ORACLE_ROWS])
    outs = [engine.kinematic_state_raw(M.topo, M.table, q[:B].to(DEV), qd[:B].to(DEV), want_quats=True) for B in (SMALL, LARGE)]
    poses, quats, vels = (split([o[c] for o in outs], dim=2) for c in range(3))
    pose64 = torch.stack([torch.cat([R.reshape(-1, 9), p], 1).t() for R, p in zip(R64, p64)])
    pose32 = torch.stack([torch.cat([R.reshape(-1, 9), p], 1).t() for R, p in zip(R32, p32)])
    check(f"{name} kinematic_state poses", poses, pose64, pose32)
    vel64 = torch.stack([torch.cat([w, v], 1).t() for w, v in zip(w64, v64)])
    vel32 = torch.stack([torch.cat([w, v], 1).t() for w, v in zip(w32, v32)])
    check(f"{name} kinematic_state vels", vels, vel64, vel32)
    q64 = torch.stack([O.quaternion(R) for R in R64])
    q32 = torch.stack([O.quaternion(R) for R in R32])
    check(f"{name} kinematic_state quats", align_quat(quats.permute(0, 2, 1), q64), q64, q32)
    # the model-level entry points on the URDF (symmetric) inertias: all-links FK and update_kinematic_state
    r64 = O.load_robot(M.path, torch.float64)
    qs = q[:SMALL].to(DEV)
    allfk = M.m.compute_forward_kinematics_all_links(qs)
    R, p, w, v, _ = O.kinematic_state(r64, q[:SMALL].double(), qd[:SMALL].double())
    got = torch.stack([allfk[nm][0] for nm in M.m.get_link_names()])
    check(f"{name} all-links fk pos", got, torch.stack(p), torch.stack(p), floor=2e-6)
    M.m.update_kinematic_state(qs, qd[:SMALL].to(DEV))
    for i, body in enumerate(M.m._bodies):
        check(f"{name} body pose l{i}", body.pose.translation(), p[i], p[i], floor=2e-6)
        check(f"{name} body vel l{i}", torch.cat([body.vel.ang, body.vel.lin], 1), torch.cat([w[i], v[i]], 1),
              torch.cat([w[i], v[i]], 1), floor=1e-5)


# ------------------------------------------------------------------------------------------------
# dynamics
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", RUNNABLE)
def test_inverse_dynamics_matches_the_oracle(name, model_dir):
    M = get(name, model_dir)
    q, qd, qdd, _ = M.inputs(3)
    ins = [t[ORACLE_ROWS] for t in (q, qd, qdd)]
    dev = [t.to(DEV) for t in (q, qd, qdd)]
    try:
        for grav, damp in ((True, True), (False, True), (True, False)):
            flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
            w64, w32 = both(O.inverse_dynamics, M.r64, M.r32, *ins, grav, damp)
            for fold in (1, 0):
                engine.set_option("rnea_fold", fold)
                got = split([engine.inverse_dynamics_raw(M.topo, M.table, *(t[:B] for t in dev), flags) for B in (SMALL, LARGE)])
                check(f"{name} rnea g{int(grav)}d{int(damp)} fold{fold}", got, w64, w32)
            if M.folded is not None:
                engine.set_option("rnea_fold", 1)
                got = split([engine.inverse_dynamics_raw(M.topo, M.table, *(t[:B] for t in dev), flags, folded=M.folded)
                             for B in (SMALL, LARGE)])
                check(f"{name} rnea g{int(grav)}d{int(damp)} prefolded", got, w64, w32)
    finally:
        engine.set_option("rnea_fold", 1)
    assert (M.folded is not None) == M.foldable


@pytest.mark.parametrize("name", RUNNABLE)
def test_forward_dynamics_and_mass_matrix_match_the_oracle(name, model_dir):
    M = get(name, model_dir)
    q, qd, _, f = M.inputs(4)
    ins = [t[ORACLE_ROWS] for t in (q, qd, f)]
    dev = [t.to(DEV) for t in (q, qd, f)]
    if M.n == 0:                                               # nothing to compute: empty results
        assert engine.forward_dynamics_raw(M.topo, M.table, *dev, engine.GRAVITY).shape == (LARGE, 0)
        assert engine.mass_matrix_raw(M.topo, M.table, dev[0]).shape == (LARGE, 0, 0)
        return
    for grav, damp in ((True, True), (False, False)):
        flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
        w64, w32 = both(O.forward_dynamics, M.r64, M.r32, *ins, grav, damp)
        got = split([engine.forward_dynamics_raw(M.topo, M.table, *(t[:B] for t in dev), flags) for B in (SMALL, LARGE)])
        check(f"{name} aba g{int(grav)}d{int(damp)}", got, w64, w32)
        if M.folded is not None:
            got = split([engine.forward_dynamics_raw(M.topo, M.table, *(t[:B] for t in dev), flags, folded=M.folded)
                         for B in (SMALL, LARGE)])
            check(f"{name} aba g{int(grav)}d{int(damp)} prefolded", got, w64, w32)
    if mm_smem_bytes(M) > SMEM_CAP:
        assert (name, "mass_matrix") in REFUSALS                 # checked there
        return
    w64, w32 = both(oracle_mass_matrix, M.r64, M.r32, ins[0])
    got = split([engine.mass_matrix_raw(M.topo, M.table, dev[0][:B]) for B in (SMALL, LARGE)])
    check(f"{name} mass matrix", got, w64, w32)
    if M.folded is not None:
        got = split([engine.mass_matrix_raw(M.topo, M.table, dev[0][:B], folded=M.folded) for B in (SMALL, LARGE)])
        check(f"{name} mass matrix prefolded", got, w64, w32)


@pytest.mark.parametrize("name", RUNNABLE)
def test_rollout_matches_the_oracle(name, model_dir):
    M = get(name, model_dir)
    T, dt, rows = 8, 2.0 ** -10, 67
    if M.n == 0:
        return
    q, qd, _, _ = M.inputs(5)
    f = torch.randn(T, rows, M.n, generator=torch.Generator().manual_seed(5))
    q, qd = q[:rows], qd[:rows]
    (o64, o32) = (oracle_rollout(M.r64, q.double(), qd.double(), f.double(), dt, True, True),
                  oracle_rollout(M.r32, q, qd, f, dt, True, True))
    got = engine.forward_dynamics_rollout_raw(M.topo, M.table, q.to(DEV), qd.to(DEV), f.to(DEV), dt,
                                              engine.GRAVITY | engine.DAMPING)
    for k, tag in enumerate(("q", "qd", "qdd")):
        check(f"{name} rollout {tag}", got[k], o64[k], o32[k])


@pytest.mark.parametrize("name", ["A_bfs_movable_palm", "A_bfs_fixed_palm", "C_random", "C_dfs", "D_fixed", "F_tree64"])
def test_body_state_after_inverse_dynamics_matches_the_oracle(name, model_dir):
    """`_bodies[i].acc / .force` against drm_oracle.dynamic_state (the model's own URDF inertias)."""
    M = get(name, model_dir)
    q, qd, qdd, _ = (t[:SMALL] for t in M.inputs(6))
    r64, r32 = O.load_robot(M.path, torch.float64), O.load_robot(M.path, torch.float32)
    for grav in (True, False):
        s64, s32 = both(O.dynamic_state, r64, r32, q, qd, qdd, grav, True)
        M.m.compute_inverse_dynamics(q.to(DEV), qd.to(DEV), qdd.to(DEV), include_gravity=grav, use_damping=True)
        for key, attr in (("acc", "acc"), ("force", "force")):
            got = torch.stack([torch.cat([getattr(b, attr).ang, getattr(b, attr).lin], 1) for b in M.m._bodies])
            w64 = torch.cat([s64[f"{key}_ang"], s64[f"{key}_lin"]], 2)
            w32 = torch.cat([s32[f"{key}_ang"], s32[f"{key}_lin"]], 2)
            check(f"{name} body {key} g{int(grav)}", got, w64, w32)


def test_inputs_off_alignment_match_the_oracle(model_dir):
    """The 8-slot breadth-first hand with every input 4 bytes off 16-byte alignment (cooperative staging)."""
    M = get("A_bfs_fixed_palm", model_dir)
    q, qd, qdd, f = M.inputs(7)
    ins = [t[ORACLE_ROWS] for t in (q, qd, qdd, f)]
    flags = engine.GRAVITY | engine.DAMPING
    dev = [t.to(DEV) for t in (q, qd, qdd, f)]
    sh = lambda t, B: shifted(t[:B].contiguous())        # noqa: E731
    w64, w32 = both(O.inverse_dynamics, M.r64, M.r32, *ins[:3], True, True)
    got = split([engine.inverse_dynamics_raw(M.topo, M.table, *(sh(t, B) for t in dev[:3]), flags) for B in (SMALL, LARGE)])
    check("A_bfs_fixed_palm rnea unaligned", got, w64, w32)
    got = split([engine.inverse_dynamics_raw(M.topo, M.table, *(sh(t, B) for t in dev[:3]), flags, folded=M.folded)
                 for B in (SMALL, LARGE)])
    check("A_bfs_fixed_palm rnea prefolded unaligned", got, w64, w32)
    w64, w32 = both(O.forward_dynamics, M.r64, M.r32, ins[0], ins[1], ins[3], True, True)
    got = split([engine.forward_dynamics_raw(M.topo, M.table, sh(dev[0], B), sh(dev[1], B), sh(dev[3], B), flags)
                 for B in (SMALL, LARGE)])
    check("A_bfs_fixed_palm aba unaligned", got, w64, w32)
    w64, w32 = both(oracle_mass_matrix, M.r64, M.r32, ins[0])
    got = split([engine.mass_matrix_raw(M.topo, M.table, sh(dev[0], B)) for B in (SMALL, LARGE)])
    check("A_bfs_fixed_palm mass matrix unaligned", got, w64, w32)
    (R64, p64, _, _, _), (R32, p32, _, _, _) = both(O.kinematic_state, M.r64, M.r32, ins[0])
    got = split([engine.kinematic_state_raw(M.topo, M.table, sh(dev[0], B))[0] for B in (SMALL, LARGE)], dim=2)
    check("A_bfs_fixed_palm kinematic_state unaligned", got[:, 9:12], torch.stack(p64).permute(0, 2, 1),
          torch.stack(p32).permute(0, 2, 1))


# ------------------------------------------------------------------------------------------------
# metamorphic: the same robot in two document orders
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("a,b", [("A_bfs_movable_palm", "B_dfs_movable_palm"), ("A_bfs_fixed_palm", "B_dfs_fixed_palm"),
                                 ("C_dfs", "C_random")])
def test_document_orders_agree_after_permuting_columns(a, b, model_dir):
    Ma, Mb = get(a, model_dir), get(b, model_dir)
    # dof column of each movable link, by name
    col_a = {Ma.r32.names[i]: Ma.r32.dof[i] for i in Ma.r32.controlled}
    perm = torch.tensor([col_a[Mb.r32.names[i]] for i in Mb.r32.controlled])       # b's column k = a's column perm[k]
    q, qd, qdd, f = Ma.inputs(8)
    q, qd, qdd, f = (t[:SMALL] for t in (q, qd, qdd, f))
    ins_a = [t.to(DEV) for t in (q, qd, qdd, f)]
    ins_b = [t[:, perm].contiguous().to(DEV) for t in (q, qd, qdd, f)]
    flags = engine.GRAVITY | engine.DAMPING
    w64, w32 = both(O.inverse_dynamics, Ma.r64, Ma.r32, q, qd, qdd)
    ta = engine.inverse_dynamics_raw(Ma.topo, Ma.table, *ins_a[:3], flags)
    tb = engine.inverse_dynamics_raw(Mb.topo, Mb.table, *ins_b[:3], flags)
    bound = 2 * max(8 * float((w32.double() - w64).abs().max() / w64.abs().max()), 2e-5)
    assert float((ta[:, perm] - tb).abs().max() / w64.abs().max()) <= bound, "rnea"
    w64, w32 = both(O.forward_dynamics, Ma.r64, Ma.r32, q, qd, f, True, True)
    aa = engine.forward_dynamics_raw(Ma.topo, Ma.table, ins_a[0], ins_a[1], ins_a[3], flags)
    ab = engine.forward_dynamics_raw(Mb.topo, Mb.table, ins_b[0], ins_b[1], ins_b[3], flags)
    bound = 2 * max(8 * float((w32.double() - w64).abs().max() / w64.abs().max()), 2e-5)
    assert float((aa[:, perm] - ab).abs().max() / w64.abs().max()) <= bound, "aba"
    if mm_smem_bytes(Ma) <= SMEM_CAP:
        Ha = engine.mass_matrix_raw(Ma.topo, Ma.table, ins_a[0])
        Hb = engine.mass_matrix_raw(Mb.topo, Mb.table, ins_b[0])
        assert float((Ha[:, perm][:, :, perm] - Hb).abs().max() / Ha.abs().max()) <= 1e-4, "mass matrix"


# ------------------------------------------------------------------------------------------------
# gradients against autograd of the fp64 oracle (every link parameter learnable)
# ------------------------------------------------------------------------------------------------
ORACLE_PARAM = {"trans": "trans", "rot_angles": "rpy", "mass": "mass", "com": "com", "inertia_mat": "inertia",
                "joint_damping": "damping"}


def learnable_model_at(path, robot):
    """Every link parameter an unconstrained module initialised from `robot` (the oracle's values, non-symmetric
    inertias included); a path-based variant of test_backward_gpu.learnable_model."""
    m = drm.DifferentiableRobotModel(path, "learnable", device=DEV)
    params = {}
    for i, body in enumerate(m._bodies):
        if i == 0:
            continue
        inits = {"mass": UnconstrainedScalar(init_val=robot.mass[i].clone()),
                 "com": UnconstrainedTensor(1, 3, init_tensor=robot.com[i].clone().reshape(1, 3)),
                 "inertia_mat": UnconstrainedTensor(3, 3, init_tensor=robot.inertia[i].clone().reshape(3, 3))}
        if body.joint_idx is not None:
            inits["trans"] = UnconstrainedTensor(1, 3, init_tensor=robot.trans[i].clone().reshape(1, 3))
            inits["rot_angles"] = UnconstrainedTensor(1, 3, init_tensor=robot.rpy[i].clone().reshape(1, 3))
            inits["joint_damping"] = UnconstrainedScalar(init_val=robot.damping[i].clone())
        for pname, module in inits.items():
            m.make_link_param_learnable(body.name, pname, module)
            params[(i, pname)] = module.param
    return m, params


def oracle_grads(robot, loss_fn, inputs):
    rb = robot.to(robot.trans.dtype)
    for name in set(ORACLE_PARAM.values()):
        setattr(rb, name, getattr(rb, name).detach().clone().requires_grad_(True))
    ins = [t.detach().clone().requires_grad_(True) for t in inputs]
    loss = loss_fn(rb, *ins)
    names = sorted(set(ORACLE_PARAM.values()))
    grads = torch.autograd.grad(loss, ins + [getattr(rb, n) for n in names], allow_unused=True)
    by = {n: (torch.zeros_like(getattr(rb, n)) if g is None else g) for n, g in zip(names, grads[len(ins):])}
    return [torch.zeros_like(t) if g is None else g for t, g in zip(ins, grads[:len(ins)])], by


def check_grads(what, M, run, loss_fn, inputs):
    """run(model, device inputs) -> loss on the device; loss_fn(robot, *inputs) the same loss on the oracle."""
    m, params = learnable_model_at(M.path, M.r32)
    dev = [t.to(DEV).requires_grad_(True) for t in inputs]
    run(m, *dev).backward()
    g64, by64 = oracle_grads(M.r64, loss_fn, [t.double() for t in inputs])
    g32, by32 = oracle_grads(M.r32, loss_fn, [t.float() for t in inputs])

    def flat(gs, by, got=False):
        parts = [g.reshape(-1).double().cpu() for g in gs]
        for (i, pname), p in sorted(params.items()):
            if got:
                parts.append((torch.zeros_like(p) if p.grad is None else p.grad).reshape(-1).double().cpu())
            else:
                parts.append(by[ORACLE_PARAM[pname]][i].reshape(-1).double())
        return torch.cat(parts)
    check(what, flat([t.grad for t in dev], None, got=True), flat(g64, by64), flat(g32, by32))


GRAD_FAMILIES = ["A_bfs_fixed_palm", "A_bfs_movable_palm", "C_random", "D_fixed", "E_unfoldable", "F_chain64", "F_tree64",
                 "G_one_joint"]
GRAD_ROWS = 67


@pytest.mark.parametrize("name", GRAD_FAMILIES)
def test_kinematic_and_inverse_dynamics_gradients_match_oracle_autograd(name, model_dir):
    M = get(name, model_dir)
    q, qd, qdd, _ = (t[:GRAD_ROWS] for t in M.inputs(9))
    gen = torch.Generator().manual_seed(9)
    e = M.leaves[-1]
    Gp, Gl, Ga = torch.randn(GRAD_ROWS, 3, generator=gen), torch.randn(GRAD_ROWS, 3, M.n, generator=gen), torch.randn(GRAD_ROWS, 3, M.n, generator=gen)
    link = M.r32.names[e]

    def fk_run(m, qq):
        pos, _, jl, ja = m.compute_fk_and_jacobian(qq, link)
        return (Gp.to(DEV) * pos).sum() + (Gl.to(DEV) * jl).sum() + (Ga.to(DEV) * ja).sum()

    def fk_loss(rb, qq):
        pos, _, jl, ja = oracle_kinematics(rb, qq, [e])[0]
        return (Gp.to(qq.dtype) * pos).sum() + (Gl.to(qq.dtype) * jl).sum() + (Ga.to(qq.dtype) * ja).sum()
    check_grads(f"{name} fk grad", M, fk_run, fk_loss, [q])

    G = torch.randn(GRAD_ROWS, M.n, generator=gen)
    chain = all(p == i - 1 for i, p in enumerate(M.spec.doc()[0]) if i > 0)
    try:
        for bwd_chain in ((0, 1) if chain else (1,)):
            engine.set_option("rnea_bwd_chain", bwd_chain)
            check_grads(f"{name} rnea grad chain{bwd_chain}", M,
                        lambda m, a, b, c: (G.to(DEV) * m.compute_inverse_dynamics(a, b, c, True, True)).sum(),
                        lambda rb, a, b, c: (G.to(a.dtype) * O.inverse_dynamics(rb, a, b, c, True, True)).sum(), [q, qd, qdd])
    finally:
        engine.set_option("rnea_bwd_chain", 1)


@pytest.mark.parametrize("name", GRAD_FAMILIES)
def test_dynamics_gradients_match_oracle_autograd(name, model_dir):
    M = get(name, model_dir)
    q, qd, _, f = (t[:GRAD_ROWS] for t in M.inputs(10))
    gen = torch.Generator().manual_seed(10)
    G = torch.randn(GRAD_ROWS, M.n, generator=gen)
    check_grads(f"{name} aba grad", M,
                lambda m, a, b, c: (G.to(DEV) * m.compute_forward_dynamics(a, b, c, True, True)).sum(),
                lambda rb, a, b, c: (G.to(a.dtype) * O.forward_dynamics(rb, a, b, c, True, True)).sum(), [q, qd, f])
    if mm_smem_bytes(M) <= SMEM_CAP:
        GH = torch.randn(GRAD_ROWS, M.n, M.n, generator=gen)
        check_grads(f"{name} mass matrix grad", M, lambda m, a: (GH.to(DEV) * m.compute_lagrangian_inertia_matrix(a)).sum(),
                    lambda rb, a: (GH.to(a.dtype) * oracle_mass_matrix(rb, a)).sum(), [q])
    T, dt, rows = 4, 2.0 ** -10, 33
    fr = torch.randn(T, rows, M.n, generator=gen)
    Gq, Gqd = torch.randn(T, rows, M.n, generator=gen), torch.randn(T, rows, M.n, generator=gen)
    check_grads(f"{name} rollout grad", M,
                lambda m, a, b, c: sum((g.to(DEV) * o).sum() for g, o in zip((Gq, Gqd), m.compute_forward_dynamics_rollout(a, b, c, dt, True, True))),
                lambda rb, a, b, c: sum((g.to(a.dtype) * o).sum() for g, o in zip((Gq, Gqd), oracle_rollout(rb, a, b, c, dt, True, True))),
                [q[:rows], qd[:rows], fr])


# ------------------------------------------------------------------------------------------------
# models the engine refuses (family H, and the mass matrix beyond its shared-memory limit)
# ------------------------------------------------------------------------------------------------
def _entry(model, point, B=5):
    n = model._n_dofs
    z = torch.zeros(B, n, device=DEV)
    names = model.get_link_names()
    calls = {
        "inverse_dynamics": lambda: model.compute_inverse_dynamics(z, z, z),
        "forward_dynamics": lambda: model.compute_forward_dynamics(z, z, z),
        "mass_matrix": lambda: model.compute_lagrangian_inertia_matrix(z),
        "rollout": lambda: model.compute_forward_dynamics_rollout(z, z, z.expand(3, B, n).contiguous(), 1e-3),
        "kinematic_state": lambda: model.update_kinematic_state(z, z) or model._bodies[-1].pose,
        "all_links_fk": lambda: model.compute_forward_kinematics_all_links(z),
        "body_state": lambda: model.compute_inverse_dynamics(z, z, z) and model._bodies[-1].force,
        "fk": lambda: model.compute_fk_and_jacobian(z, names[-1]),
        "fk_multi": lambda: model.compute_fk_and_jacobian_multi(z, [names[k] for k in S.leaves(model._parent_idx)[:8]]),
    }
    return calls[point]()


# (model, entry point) -> expected outcome: None = computes, else (exception, message pattern).  Worked out from the
# host code: build_tree_program refuses more than DRM_MAX_SLOTS live branch points for every kernel that walks the tree
# program, the single-end-effector FK walks a root-to-link path and the multi-end-effector walk (fk_tree.cu) is
# depth-first, which needs one slot for the palm; compile_topology refuses more than 64 links; the mass-matrix kernel
# keeps a tile of n x n matrices in shared memory (mass_matrix_device_impl).
LIVE = (RuntimeError, "more than 8 live branch points")
NULL_Q = (RuntimeError, "table / q is null")
REFUSALS = {
    ("H_nine_slots", "inverse_dynamics"): LIVE,
    ("H_nine_slots", "forward_dynamics"): LIVE,
    ("H_nine_slots", "mass_matrix"): LIVE,
    ("H_nine_slots", "rollout"): LIVE,
    ("H_nine_slots", "kinematic_state"): LIVE,
    ("H_nine_slots", "all_links_fk"): LIVE,
    ("H_nine_slots", "body_state"): LIVE,
    ("H_nine_slots", "fk"): None,
    ("H_nine_slots", "fk_multi"): None,
    ("H_65_links", "construct"): (ValueError, "65 links exceed the engine limit of 64"),
    # the kinematic kernels take q by pointer, and the q of a model without movable joints is empty (a null pointer)
    ("G_root_only", "fk"): NULL_Q,
    ("G_root_only", "kinematic_state"): NULL_Q,
    ("G_root_only", "all_links_fk"): NULL_Q,
    ("G_all_fixed", "fk"): NULL_Q,
    ("G_all_fixed", "kinematic_state"): NULL_Q,
    ("G_all_fixed", "all_links_fk"): NULL_Q,
    ("F_chain64", "mass_matrix"): (RuntimeError, r"needs \d+ B of shared memory per CTA"),
    ("F_tree64", "mass_matrix"): (RuntimeError, r"needs \d+ B of shared memory per CTA"),
    ("C_dfs", "mass_matrix"): (RuntimeError, r"needs \d+ B of shared memory per CTA"),
    ("C_random", "mass_matrix"): (RuntimeError, r"needs \d+ B of shared memory per CTA"),
}


@pytest.mark.parametrize("name,point", sorted(REFUSALS))
def test_refusals(name, point, model_dir):
    spec = {**FAM, **S.refusal_families()}[name]
    path = S.build(spec, model_dir)
    want = REFUSALS[(name, point)]
    if point == "construct":
        with pytest.raises(want[0], match=want[1]):
            drm.DifferentiableRobotModel(path, name, device=DEV)
        return
    model = drm.DifferentiableRobotModel(path, name, device=DEV)
    if name in FAM and point == "mass_matrix":
        assert mm_smem_bytes(get(name, model_dir)) > SMEM_CAP
    model._link_table()
    model._folded_table()                                   # table build and fold are launches of their own
    before = engine.launch_count()
    if want is None:
        _entry(model, point)
        torch.cuda.synchronize()
        assert engine.launch_count() > before
        return
    with pytest.raises(want[0], match=want[1]):
        _entry(model, point)
    assert engine.launch_count() == before                  # refused on the host, before any launch


def test_nine_slot_model_fk_matches_the_oracle(model_dir):
    """The refused tree program does not concern the path and depth-first walks: they compute, and correctly."""
    spec = S.refusal_families()["H_nine_slots"]
    path = S.build(spec, model_dir)
    m = drm.DifferentiableRobotModel(path, "H", device=DEV)
    r64, r32 = O.load_robot(path, torch.float64), O.load_robot(path, torch.float32)
    q = O.sample_inputs(r64, SMALL, seed=12)[0]
    leaves = S.leaves(r32.parent)[:8]
    w64, w32 = both(oracle_kinematics, r64, r32, q, leaves)
    out = m.compute_fk_and_jacobian_multi(q.to(DEV), [r32.names[e] for e in leaves])
    for k, e in enumerate(leaves):
        pos, quat, jl, ja = out[r32.names[e]]
        check(f"H_nine_slots fk_multi l{e}", torch.stack([jl, ja]), torch.stack(w64[k][2:]), torch.stack(w32[k][2:]))
        p1, _, jl1, _ = m.compute_fk_and_jacobian(q.to(DEV), r32.names[e])
        check(f"H_nine_slots fk pos l{e}", p1, w64[k][0], w32[k][0])
        check(f"H_nine_slots fk jlin l{e}", jl1, w64[k][2], w32[k][2])


# ------------------------------------------------------------------------------------------------
# mass-matrix gradients of the shipped robots against the fp64 oracle (not only against the stacked RNEA path, which
# runs the same adjoint kernel)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem,nonsymmetric", [("iiwa7", True), ("iiwa7", False), ("panda", False), ("trifinger_edu", False),
                                               ("iiwa7_allegro", False), ("jaco_clean", False)])
def test_mass_matrix_gradients_of_shipped_robots_match_oracle_autograd(stem, nonsymmetric):
    from types import SimpleNamespace
    from conftest import urdf_path
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if nonsymmetric:
        gen = torch.Generator().manual_seed(3)
        scale = r32.inertia.abs().amax(dim=(1, 2), keepdim=True)
        r32.inertia = r32.inertia + 0.05 * scale * torch.randn(r32.inertia.shape, generator=gen)
        assert float((r32.inertia - r32.inertia.transpose(1, 2)).abs().max()) > 1e-4
    M = SimpleNamespace(path=urdf_path(stem), r32=r32, r64=r32.to(torch.float64))
    q = O.sample_inputs(r32, 130, seed=8)[0]
    GH = torch.randn(130, r32.n_dofs, r32.n_dofs, generator=torch.Generator().manual_seed(4))
    check_grads(f"{stem} mass matrix grad{' nonsymmetric' if nonsymmetric else ''}", M,
                lambda m, a: (GH.to(DEV) * m.compute_lagrangian_inertia_matrix(a)).sum(),
                lambda rb, a: (GH.to(a.dtype) * oracle_mass_matrix(rb, a)).sum(), [q])
