"""GPU: contact-constrained rollouts (compute_contact_rollout / engine.contact_rollout_raw, csrc/contact_rollout.cu).

* omega = 0: bit-identical to the stepwise loop of compute_contact_dynamics(accel_ref=None) + semi-implicit Euler, on every
  robot and link set of the contact tests, every flag combination, outputs given or NULL;
* omega > 0, teacher-forced: compute_contact_dynamics at every stored (q_t, qd_t) with the kernel's own a_ref reproduces
  qdd[t] and force[t] bit for bit, and that a_ref matches the fp64 oracle's Baumgarte term at the same state;
* against the fp64 oracle (tests/contact_rollout_oracle.py) and the reference's goldens (<robot>.contact_rollout.npz)
  within max(8 x the fp32 oracle's deviation over the same loop, a floor);
* physics (the pinned-end-effector example's setting, energy), launch geometry, robustness, graphs and refusals."""
import ctypes
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor
from conftest import GOLDEN_DIR, urdf_path
import contact_oracle as C
import contact_rollout_oracle as CR
import test_contact_dynamics_gpu as CDT
import test_operational_space_gpu as OSDT
import tile_mirrors as TM
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TIPS = OSDT.TIPS
TRI = CDT.TRI
EE = OSDT.EE
EINVAL, ELIMIT = -1, -3             # DRMB200_EINVAL, DRMB200_ELIMIT
same_bits = CDT.same_bits
STATIC_SMEM = 128                       # the two mbarriers (-Xptxas -v)
# (robot, links, position_only, redundant: needs mu > 0)
CASES = [("2link_robot", ["endEffector"], False, True), ("iiwa7_allegro", TIPS, False, True),
         ("iiwa7", ["iiwa_link_ee"], False, False), ("panda_no_gripper", ["panda_virtual_ee_link"], False, False),
         ("trifinger_edu", TRI, True, False), ("allegro_hand_description_left", TIPS, True, False)]
CASE_IDS = [f"{c[0]}-{len(c[1])}{'pos' if c[2] else 'pose'}" for c in CASES]
FLAGS = [(True, False), (True, True), (False, False), (False, True)]


def model_of(stem):
    return OSDT.model_of(stem)


def inputs(stem, B, T, seed, fscale=0.1):
    r = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, _ = O.sample_inputs(r, B, seed=seed, dtype=torch.float32)
    qd = 0.2 * qd
    f = fscale * torch.randn(T, B, r.n_dofs, generator=torch.Generator().manual_seed(seed + 1))
    return q.to(DEV), qd.to(DEV), f.to(DEV)


def mu_for(m, links, q, pos, redundant):
    """1e-3 max_k A_kk for redundant sets (as the contact goldens), else 0."""
    if not redundant:
        return 0.0
    inv = engine.operational_space_dynamics_raw(m._topology, links, m._link_table().detach(), q, torch.zeros_like(q),
                                                torch.zeros_like(q), 0, pos, True, False, False, False)[0]
    return 1e-3 * float(torch.diagonal(inv, dim1=1, dim2=2).max())


def loop(m, names, q, qd, f, dt, flags, pos, mu, omega=0.0, targets=None):
    """The stepwise loop in torch: compute_contact_dynamics plus a torch Baumgarte term plus the integrate."""
    grav, damp = flags
    qs, qds, qdds, forces, oks = [], [], [], [], []
    if omega and targets is None:
        targets = fk_targets(m, names, q, pos)
    for t in range(f.shape[0]):
        a_ref = None
        if omega:
            a_ref = torch_baumgarte(m, names, q, qd, pos, omega, targets)
        out = m.compute_contact_dynamics(q, qd, f[t], names, a_ref, include_gravity=grav, use_damping=damp,
                                         position_only=pos, regularization=mu)
        qd = qd + dt * out.qdd
        q = q + dt * qd
        for lst, v in zip((qs, qds, qdds, forces, oks), (q, qd, out.qdd, out.force, out.solved)):
            lst.append(v)
    return torch.stack(qs), torch.stack(qds), torch.stack(qdds), torch.stack(forces), torch.stack(oks).all(0)


def fk_targets(m, names, q, pos):
    multi = m.compute_fk_and_jacobian_multi(q, names)
    tp = torch.stack([multi[n][0] for n in names])
    tq = None if pos else torch.stack([multi[n][1] for n in names])
    return tp, tq


def torch_baumgarte(m, names, q, qd, pos, omega, targets):
    multi = m.compute_fk_and_jacobian_multi(q, names)
    blocks, vel = [], []
    for l, n in enumerate(names):
        p, quat, jl, ja = multi[n]
        blocks.append(p - targets[0][l])
        vel.append(torch.einsum("bmn,bn->bm", jl, qd))
        if not pos:
            blocks.append(CR.rotvec_error(quat.double().cpu(), targets[1][l].double().cpu()).float().to(DEV))
            vel.append(torch.einsum("bmn,bn->bm", ja, qd))
    e, v = torch.cat(blocks, 1), torch.cat(vel, 1)
    return -(2 * omega) * v - (omega * omega) * e


def rollout(m, links, q, qd, f, dt, flags, pos, mu, omega=0.0, tp=None, tq=None, **want):
    fl = (engine.GRAVITY if flags[0] else 0) | (engine.DAMPING if flags[1] else 0)
    return engine.contact_rollout_raw(m._topology, links, m._link_table().detach(), q, qd, f, dt, fl, tp, tq, pos, mu, omega,
                                      **want)


# ------------------------------------------------------------------------------------------------
# 1. bit identity at omega = 0
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_bit_identical_to_the_stepwise_loop_at_zero_omega(case):
    stem, names, pos, redundant = case
    m = model_of(stem)
    links = m._contact_links(names)
    q, qd, f = inputs(stem, 37, 6, seed=31)
    mu = mu_for(m, links, q, pos, redundant)
    for flags in FLAGS:
        want = loop(m, names, q, qd, f, 1e-3, flags, pos, mu)
        got = rollout(m, links, q, qd, f, 1e-3, flags, pos, mu, want_accel_ref=True)
        for name, g, w in zip(("q", "qd", "qdd", "force"), got[:4], want[:4]):
            assert same_bits(g, w), f"{stem} {flags}: {name} differs from the loop"
        assert torch.equal(got[5], want[4])
        assert torch.equal(got[4], torch.zeros_like(got[4])) and not bool(torch.signbit(got[4]).any())
        bare = rollout(m, links, q, qd, f, 1e-3, flags, pos, mu, want_qdd=False, want_force=False)
        assert bare[2] is None and bare[3] is None and bare[4] is None
        assert same_bits(bare[0], want[0]) and same_bits(bare[1], want[1]) and torch.equal(bare[5], want[4])


# ------------------------------------------------------------------------------------------------
# 2. teacher-forced bit identity at omega > 0, and the Baumgarte term against the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("explicit", [False, True], ids=["default-targets", "explicit-targets"])
@pytest.mark.parametrize("case", [CASES[2], CASES[1], CASES[4]], ids=[CASE_IDS[2], CASE_IDS[1], CASE_IDS[4]])
def test_teacher_forced_steps_and_baumgarte_term(case, explicit):
    stem, names, pos, redundant = case
    m = model_of(stem)
    links = m._contact_links(names)
    B, T, dt, omega = 19, 5, 1e-3, 50.0
    q, qd, f = inputs(stem, B, T, seed=41)
    mu = mu_for(m, links, q, pos, redundant)
    tp = tq = None
    if explicit:                                  # off the start poses, so that e is not small
        tp, tq = fk_targets(m, names, q, pos)
        tp = tp + 0.01 * torch.randn(tp.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
        if tq is not None:
            tq = 3.0 * (tq + 0.05 * torch.randn(tq.shape, generator=torch.Generator().manual_seed(4)).to(DEV))
    got = rollout(m, links, q, qd, f, dt, (True, True), pos, mu, omega, tp, tq, want_accel_ref=True)
    qs = torch.cat([q[None], got[0][:-1]])
    qds = torch.cat([qd[None], got[1][:-1]])
    for t in range(T):
        out = m.compute_contact_dynamics(qs[t], qds[t], f[t], names, got[4][t], include_gravity=True, use_damping=True,
                                         position_only=pos, regularization=mu)
        assert same_bits(out.qdd, got[2][t]) and same_bits(out.force, got[3][t]), f"{stem} step {t}"
    r64 = O.load_robot(urdf_path(stem), torch.float64)
    if tp is None:
        tp64, tq64 = CR.poses(r64, q.double().cpu(), names)
        tq64 = None if pos else tq64
    else:
        tp64 = tp.double().cpu()
        tq64 = None if tq is None else tq.double().cpu()
    rows = got[5].cpu()                           # rows some step left unsolved (near-singular samples) are NaN
    assert bool(rows.any())
    if tp64 is not None:
        tp64 = tp64[:, rows]
        tq64 = None if tq64 is None else tq64[:, rows]
    for t in range(T):
        qt, qdt = qs[t].double().cpu()[rows], qds[t].double().cpu()[rows]
        want = CR.baumgarte(r64, qt, qdt, names, pos, omega, tp64, tq64)
        v = torch.einsum("bmn,bn->bm", CR.S.stacked_jacobian(r64, qt, names, pos), qdt)
        scale = 2 * omega * float(v.abs().max()) + omega * omega * float(((want + 2 * omega * v) / (omega * omega)).abs().max())
        err = float((got[4][t].double().cpu()[rows] - want).abs().max())
        bound = 1e-5 * scale + omega * omega * 2e-6
        print(f"ERR {stem} t={t} a_ref {err:.2e} (bound {bound:.2e})")
        assert err <= bound, f"{stem} step {t}: a_ref error {err:.3e} > {bound:.3e}"


# ------------------------------------------------------------------------------------------------
# 3. the fp64 oracle and the reference's goldens
# ------------------------------------------------------------------------------------------------
GOLDEN = ["2link_robot", "iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro", "trifinger_edu"]


def traj_error(got, want):
    """Largest per-(step, row) error relative to that step and row's largest entry."""
    g, w = got.double().cpu(), want.double().cpu()
    scale = w.abs().amax(-1, keepdim=True).clamp_min(1e-30)
    return float(((g - w).abs() / scale).max())


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_matches_reference_goldens_and_oracle(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".contact_rollout.npz"), allow_pickle=False)
    names = [str(s) for s in g["links"]]
    pos, mu, dt, omega = bool(g["position_only"]), float(g["mu"]), float(g["dt"]), float(g["omega"])
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=torch.float32)
        inertia[0] = r32.inertia[0]
        r32.inertia = inertia
    table = O.link_table(r32).float().to(DEV).contiguous()
    idx = [r32.index(nm) for nm in names]
    q0, qd0, f = (torch.tensor(g[k]) for k in ("q0", "qd0", "f"))
    got = engine.contact_rollout_raw(model_of(stem)._topology, idx, table, q0.to(DEV), qd0.to(DEV), f.to(DEV), dt,
                                     engine.GRAVITY, None, None, pos, mu, omega)
    o32 = CR.contact_rollout(r32, q0, qd0, f, names, dt, omega, include_gravity=True, position_only=pos, mu=mu)
    o64 = CR.contact_rollout(r32.to(torch.float64), q0.double(), qd0.double(), f.double(), names, dt, omega,
                             include_gravity=True, position_only=pos, mu=mu)
    # the rows every path solves at every step (TriFinger's stretched fingers leave a few near-singular at mu = 0)
    pre = "" if tag == "sym" else "nonsym."
    gold = {k: torch.tensor(g[pre + k]) for k in ("q", "qd", "qdd", "force")}
    # the rows whose every step is well conditioned in all paths (smallest fp64 scaled pivot >= 500x the threshold):
    # TriFinger's stretched fingers make some near-singular, and the reference's fp32 loop parts ways with fp64 there
    rows = got[5].cpu() & o32[5] & o64[5] & (o64[6] >= 500 * C.PIVOT_MIN) & torch.isfinite(gold["q"]).all(2).all(0)
    assert int(rows.sum()) >= 2, f"{stem}: only {int(rows.sum())} of 8 rows well conditioned"
    for i, k in enumerate(("q", "qd", "qdd", "force")):
        e32 = traj_error(o32[i][:, rows], o64[i][:, rows])
        err = traj_error(got[i].cpu()[:, rows], o64[i][:, rows])
        bound = max(8 * e32, 1e-5 if k in ("q", "qd") else 2e-4)
        # the goldens solve the reference's fp32 pieces (as the contact goldens): the bound adds their own distance from
        # the fp64 oracle
        gerr = traj_error(got[i].cpu()[:, rows], gold[k][:, rows])
        g64 = traj_error(o64[i][:, rows], gold[k][:, rows])
        print(f"ERR {stem} {tag} {k}: {err:.2e} vs fp64 (fp32 oracle {e32:.2e}, bound {bound:.2e}), {gerr:.2e} vs golden "
              f"(golden vs fp64 {g64:.2e})")
        assert err <= bound, f"{stem} {tag} {k}: {err:.3e} > {bound:.3e}"
        assert gerr <= bound + g64, f"{stem} {tag} {k}: {gerr:.3e} off the reference's golden (> {bound + g64:.3e})"


# ------------------------------------------------------------------------------------------------
# 4. physics
# ------------------------------------------------------------------------------------------------
def kuka_example(B=16, T=1000, accel=2.0):
    """The inputs of examples/pinned_end_effector_iiwa.py."""
    torch.manual_seed(0)
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    lim = m.get_joint_limits()
    lo = torch.tensor([l["lower"] for l in lim], device=DEV)
    hi = torch.tensor([l["upper"] for l in lim], device=DEV)
    n = m._n_dofs
    q0 = lo + (hi - lo) * (0.3 + 0.4 * torch.rand(B, n, device=DEV))
    inertia = torch.diagonal(m.compute_lagrangian_inertia_matrix(q0), dim1=1, dim2=2)
    amp = accel * inertia * torch.randn(3, B, n, device=DEV)
    freq = 2 * torch.pi * (0.5 + 2 * torch.rand(B, n, device=DEV))
    ts = (torch.arange(T, device=DEV, dtype=torch.float32) * 1e-3).view(T, 1, 1)
    f = amp[0] + amp[1] * torch.sin(freq * ts) + amp[2] * torch.cos(0.7 * freq * ts)
    return m, q0, f


def drift(m, q, p0):
    return float(max((m.compute_forward_kinematics(q[t], "iiwa_link_ee")[0] - p0).norm(dim=1).max() for t in range(q.shape[0])))


def test_pinned_end_effector_drift_matches_the_stepwise_loop():
    m, q0, f = kuka_example()
    qd0 = torch.zeros_like(q0)
    p0 = m.compute_forward_kinematics(q0, "iiwa_link_ee")[0]
    out = m.compute_contact_rollout(q0, qd0, f, ["iiwa_link_ee"], 1e-3, stabilization=200.0, use_damping=True,
                                    position_only=True)
    assert bool(out.solved.all())
    ours = drift(m, out.q, p0)
    ref = drift(m, loop(m, ["iiwa_link_ee"], q0, qd0, f, 1e-3, (True, True), True, 0.0, 200.0)[0], p0)
    print(f"ERR pinned drift kernel {ours * 1e3:.4f} mm, loop {ref * 1e3:.4f} mm")
    assert ours < 1e-3 and ours <= 2 * ref
    tp = p0[None]
    same = m.compute_contact_rollout(q0, qd0, f, ["iiwa_link_ee"], 1e-3, target_pos=tp, stabilization=200.0, use_damping=True,
                                     position_only=True)
    assert float((same.q - out.q).abs().max()) < 1e-4, "explicit FK-at-q0 targets differ from the default ones"


@pytest.mark.parametrize("pos", [True, False], ids=["pos", "pose"])
def test_default_and_explicit_targets_agree(pos):
    m = model_of("iiwa7")
    names = ["iiwa_link_ee"]
    q, qd, f = inputs("iiwa7", 23, 50, seed=5)
    tp, tq = fk_targets(m, names, q, pos)
    a = m.compute_contact_rollout(q, qd, f, names, 1e-3, stabilization=100.0, position_only=pos)
    b = m.compute_contact_rollout(q, qd, f, names, 1e-3, target_pos=tp, target_quat=tq, stabilization=100.0,
                                  position_only=pos)
    err = float((a.q - b.q).abs().max())
    print(f"ERR default vs explicit targets pos={pos}: {err:.2e}")
    assert err < 1e-4


def test_energy_drift_without_damping_is_no_worse_than_the_loop():
    m = model_of("iiwa7")
    names = ["iiwa_link_ee"]
    q, qd, _ = inputs("iiwa7", 16, 1, seed=9)
    f = torch.zeros(300, 16, 7, device=DEV)
    out = m.compute_contact_rollout(q, qd, f, names, 1e-3, stabilization=100.0, position_only=True)
    lq = loop(m, names, q, qd, f, 1e-3, (True, False), True, 0.0, 100.0)

    def energy_drift(qs, qds):
        e0 = m.compute_energy_and_momentum(q, qd)
        E0 = e0.kinetic_energy + e0.potential_energy
        worst = 0.0
        for t in range(qs.shape[0]):
            e = m.compute_energy_and_momentum(qs[t], qds[t])
            worst = max(worst, float((e.kinetic_energy + e.potential_energy - E0).abs().max()))
        return worst
    ours, ref = energy_drift(out.q, out.qd), energy_drift(lq[0], lq[1])
    print(f"ERR energy drift kernel {ours:.3e} J, loop {ref:.3e} J")
    assert ours <= 1.1 * ref + 1e-4


# ------------------------------------------------------------------------------------------------
# 5. launch geometry and robustness
# ------------------------------------------------------------------------------------------------
def rollout_floats(T, n, n_links, tree_slots, n_u, M, n_jslots, n_state_slots, E, pose):
    """ContactRolloutSmem(T, tree program, walk, M).total_floats."""
    aba = 4 * T * n + n_links * TM.TABLE_STRIDE + n_links * 14 * T + tree_slots * 42 * T
    return TM.up4(aba) + T * (4 * n + M + M * n_u + 6 * n_jslots + 24 * n_state_slots + 4 * M + M * M + n + 15 * E
                              + (4 * E if pose else 0))


def rollout_choice(parents, movable, links, pose):
    n = sum(movable[1:])
    _, n_u, n_jslots, n_slots = TM.multi_program(parents, movable, links)
    M = (6 if pose else 3) * len(links)
    return TM.ladder(lambda T: rollout_floats(T, n, len(parents), CDT.SR.live_slots(parents), n_u, M, n_jslots, n_slots,
                                              len(links), pose), STATIC_SMEM)


def _tile_cases():
    import test_launch_geometry_solvers_gpu as LG
    cases = {}
    for name in sorted(CDT.FAM):
        par, mov = CDT.FAM[name].doc()
        if sum(mov[1:]) == 0:
            continue
        for k in range(1, 9):
            links = LG.deepest(par, mov, k)
            if not CDT._solvable(par, mov, links):
                continue
            for pose in (True, False):
                tile, _ = rollout_choice(par, mov, links, pose)
                cases.setdefault((tile, pose), (name, links))
    return cases


TILE_CASES = _tile_cases()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_contact_rollout"))


def shifted(t):
    return CDT.shifted(t)


def abi_call(topo, links, table, q0, qd0, f, dt, flags, pos, mu, omega, tp=None, tq=None, misaligned=False, want=True):
    """One C-ABI call with caller-allocated outputs (optionally 4 bytes off 16-byte alignment, inputs and outputs)."""
    T, B, n = f.shape
    M = (3 if pos else 6) * len(links)
    q, qd = torch.empty((T, B, n), device=DEV), torch.empty((T, B, n), device=DEV)
    qdd = torch.empty((T, B, n), device=DEV) if want else None
    force = torch.empty((T, B, M), device=DEV) if want else None
    aref = torch.empty((T, B, M), device=DEV) if want else None
    ok = torch.empty(B, device=DEV, dtype=torch.uint8)
    if misaligned:
        q0, qd0, f, tp, tq, q, qd, qdd, force, aref = (shifted(t) for t in (q0, qd0, f, tp, tq, q, qd, qdd, force, aref))
    idx = (ctypes.c_int32 * len(links))(*links)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = CDT.ptr
    rc = engine.lib().drmb200_contact_rollout(ctypes.byref(topo), len(links), idx, p(table), p(q0), p(qd0), p(f), p(tp), p(tq),
                                              B, T, ctypes.c_float(dt), flags, int(pos), ctypes.c_float(mu),
                                              ctypes.c_float(omega), p(q), p(qd), p(qdd), p(force), p(aref), p(ok), s)
    return rc, (q, qd, qdd, force, aref, ok.bool())


def test_static_shared_memory_is_what_the_mirror_adds():
    lib = engine.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    for t in TM.LADDER:
        sym = f"_ZN3drm22contact_rollout_kernelILi{t}EEEvNS_11TreeProgramENS_12UnionProgramENS_18ContactRolloutArgsE"
        attr = (ctypes.c_size_t * 64)()
        assert cudart.cudaFuncGetAttributes(attr, ctypes.cast(getattr(lib, sym), ctypes.c_void_p)) == 0, sym
        assert attr[0] == STATIC_SMEM, (sym, attr[0])


def test_every_reachable_rung_has_a_case():
    assert {64, 32, 16, 8, 4} <= {k[0] for k in TILE_CASES}, sorted(TILE_CASES, key=str)


@pytest.mark.parametrize("key", sorted(TILE_CASES, key=str), ids=[f"T{t}-{'pose' if p else 'pos'}" for (t, p) in
                                                                  sorted(TILE_CASES, key=str)])
def test_rows_are_independent_of_tile_batch_and_alignment(key, model_dir):
    tile, pose = key
    name, links = TILE_CASES[key]
    m, r32, _, table = CDT.family(name, model_dir)
    topo = m._topology
    pos = not pose
    B, T = 3 * tile + 3, 3
    q, qd, f = OSDT.inputs(r32, B, seed=22)
    f = torch.stack([f, 0.5 * f, -f]).to(DEV)
    q, qd = q.to(DEV), qd.to(DEV)
    mu = 1e-2 * max(1e-6, mu_for(m, links, q, pos, True) * 1e3)
    fl = engine.GRAVITY | engine.DAMPING
    rc, big = abi_call(topo, links, table, q, qd, f, 1e-3, fl, pos, mu, 20.0)
    assert rc == 0, engine.lib().drmb200_last_error()
    # the loop at omega = 0 on the same rows
    rc0, zero = abi_call(topo, links, table, q, qd, f, 1e-3, fl, pos, mu, 0.0)
    want, qs, qds = [], q, qd                     # the stepwise loop on the same table
    for t in range(T):
        qdd, force, _ = engine.contact_dynamics_raw(topo, links, table, qs, qds, f[t], fl, None, pos, mu)
        qds = qds + 1e-3 * qdd
        qs = qs + 1e-3 * qds
        want.append((qs, qds, qdd, force))
    want = [torch.stack(w) for w in zip(*want)]
    for g, w in zip(zero[:4], want):
        assert same_bits(g, w), f"{name} T={tile}: omega = 0 differs from the loop"
    for Bs in sorted({1, max(1, tile - 1), tile, tile + 1, B - 1}):
        rc, small = abi_call(topo, links, table, q[:Bs], qd[:Bs], f[:, :Bs].contiguous(), 1e-3, fl, pos, mu, 20.0)
        assert rc == 0
        for a, b in zip(small, big):
            assert same_bits(a, b[:, :Bs] if a.ndim == 3 else b[:Bs]), f"{name} T={tile} B={Bs}: rows differ"
    rc, mis = abi_call(topo, links, table, q, qd, f, 1e-3, fl, pos, mu, 20.0, misaligned=True)
    assert rc == 0 and all(same_bits(a, b) for a, b in zip(mis, big)), f"{name} T={tile}: misaligned views differ"
    rc, bare = abi_call(topo, links, table, q, qd, f, 1e-3, fl, pos, mu, 20.0, misaligned=True, want=False)
    assert rc == 0 and same_bits(bare[0], big[0]) and same_bits(bare[1], big[1]) and torch.equal(bare[5], big[5])


def test_one_step_is_one_contact_call_and_empty_calls_are_no_ops():
    m = model_of("iiwa7")
    names = ["iiwa_link_ee"]
    links = m._contact_links(names)
    q, qd, f = inputs("iiwa7", 9, 1, seed=2)
    out = m.compute_contact_rollout(q, qd, f, names, 1e-3)
    c = m.compute_contact_dynamics(q, qd, f[0], names)
    qd1 = qd + 1e-3 * c.qdd
    assert same_bits(out.qdd[0], c.qdd) and same_bits(out.force[0], c.force)
    assert same_bits(out.qd[0], qd1) and same_bits(out.q[0], q + 1e-3 * qd1)
    before = engine.launch_count()
    e = rollout(m, links, q, qd, f[:0], 1e-3, (True, False), False, 0.0, 5.0)
    assert e[0].shape == (0, 9, 7)
    e = rollout(m, links, q[:0], qd[:0], f[:, :0], 1e-3, (True, False), False, 0.0, 5.0)
    assert e[0].shape == (1, 0, 7) and e[5].shape == (0,)
    assert engine.launch_count() == before
    one = m.compute_contact_rollout(q[0], qd[0], f[:, 0], names, 1e-3)
    assert same_bits(one.q, out.q[:, 0]) and same_bits(one.force, out.force[:, 0]) and bool(one.solved) == bool(out.solved[0])


def nan_from_one_step_on(out, b):
    """Row b's q and qdd are finite up to some step t0 and NaN from t0 on (force too)."""
    nan = torch.isnan(out[2][:, b]).all(1)
    assert bool(nan.any()), f"row {b}: unsolved but never NaN"
    t0 = int(torch.nonzero(nan)[0])
    assert bool(nan[t0:].all()) and bool(torch.isfinite(out[2][:t0, b]).all()), f"row {b}: NaN must start at one step"
    assert bool(torch.isnan(out[0][t0:, b]).all()) and bool(torch.isnan(out[3][t0:, b]).all())


def test_redundant_pose_set_at_zero_mu_is_unsolved():
    stem, names = "iiwa7_allegro", TIPS          # 24 pose rows on 23 joints: redundant, unsolvable at mu = 0
    m = model_of(stem)
    links = m._contact_links(names)
    q, qd, f = inputs(stem, 64, 4, seed=12)
    out = rollout(m, links, q, qd, f, 1e-3, (True, False), False, 0.0, 10.0)
    bad = torch.nonzero(~out[5]).flatten().tolist()
    assert len(bad) >= 60, f"only {len(bad)} of 64 rows unsolved"      # fp32 lets a few rows through (DESIGN.md)
    for b in bad:
        nan_from_one_step_on(out, b)


def test_unsolved_rows_leave_the_others_alone():
    """Kuka end-effector pose: a few rows start at singular configurations (q = 0 lines up joints 1, 3, 5, 7; a 1e-3 bend
    of joint 4 leaves a scaled pivot of about 1e-9), the rest are random.  Solved and unsolved rows share the 64-row
    tiles; the unsolved ones are NaN from their failing step on and every other row is bit-identical to itself run
    without them."""
    m = model_of("iiwa7")
    names = ["iiwa_link_ee"]
    links = m._contact_links(names)
    q, qd, f = inputs("iiwa7", 130, 4, seed=14)
    singular = [2, 33, 63, 64, 129]
    q[singular] = 0.0
    q[64, 3] = 1e-3
    qd[singular] = 0.0
    out = rollout(m, links, q, qd, f, 1e-3, (True, False), False, 0.0, 10.0)
    bad = ~out[5]
    assert bool(bad[singular].all()), f"singular rows solved: {out[5][singular].tolist()}"
    for b in torch.nonzero(bad).flatten().tolist():
        nan_from_one_step_on(out, b)
    good = torch.nonzero(out[5]).flatten()
    assert len(good) >= 100, f"only {len(good)} of 130 rows solved"
    alone = rollout(m, links, q[good], qd[good], f[:, good].contiguous(), 1e-3, (True, False), False, 0.0, 10.0)
    for a, b in zip(alone[:4], out[:4]):
        assert same_bits(a, b[:, good])
    assert bool(alone[5].all())


def test_learnable_and_fused_parameters_are_used():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    names = ["iiwa_link_ee"]
    q, qd, f = inputs("iiwa7", 11, 4, seed=8)
    base = m.compute_contact_rollout(q, qd, f, names, 1e-3, stabilization=30.0)
    init = torch.diag(torch.tensor([0.09, 0.02, 0.07])).to(DEV)
    m.make_link_param_learnable("iiwa_link_3", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.clone()))
    for fused in (False, True):
        if fused:
            m.fuse_learnable_parameters()
        out = m.compute_contact_rollout(q, qd, f, names, 1e-3, stabilization=30.0)
        want = loop(m, names, q, qd, f, 1e-3, (True, False), False, 0.0)
        zero = m.compute_contact_rollout(q, qd, f, names, 1e-3)
        assert same_bits(zero.q, want[0]) and same_bits(zero.force, want[3])
        assert not torch.equal(out.q, base.q) and out.q.grad_fn is None


def test_one_launch_and_graph_capture():
    m = model_of("trifinger_edu")
    q, qd, f = inputs("trifinger_edu", 40, 8, seed=3)
    before = engine.launch_count()
    want = m.compute_contact_rollout(q, qd, f, TRI, 1e-3, stabilization=40.0, position_only=True)
    assert engine.launch_count() - before == 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_contact_rollout(q, qd, f, TRI, 1e-3, stabilization=40.0, position_only=True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = m.compute_contact_rollout(q, qd, f, TRI, 1e-3, stabilization=40.0, position_only=True)
    g.replay()
    torch.cuda.synchronize()
    assert same_bits(got.q, want.q) and same_bits(got.force, want.force) and torch.equal(got.solved, want.solved)


def test_refusals():
    m = model_of("iiwa7")
    names = ["iiwa_link_ee"]
    links = m._contact_links(names)
    topo, table = m._topology, m._link_table().detach()
    q, qd, f = inputs("iiwa7", 4, 2, seed=1)
    tp, tq = fk_targets(m, names, q, False)
    fl = engine.GRAVITY
    for omega in (-1.0, float("inf"), float("nan")):
        assert abi_call(topo, links, table, q, qd, f, 1e-3, fl, False, 0.0, omega)[0] == EINVAL
    assert abi_call(topo, links, table, q, qd, f, 1e-3, fl, True, 0.0, 1.0, tp, tq)[0] == EINVAL     # quat in position mode
    assert abi_call(topo, links, table, q, qd, f, 1e-3, fl, False, 0.0, 1.0, tp, None)[0] == EINVAL  # one of two
    assert abi_call(topo, links, table, q, qd, f, 1e-3, fl, False, 0.0, 1.0, None, tq)[0] == EINVAL
    assert abi_call(topo, links, table, q, qd, f, 1e-3, fl, False, -1.0, 1.0)[0] == EINVAL            # mu < 0
    assert abi_call(topo, [0], table, q, qd, f, 1e-3, fl, False, 0.0, 1.0)[0] == EINVAL               # the root
    assert abi_call(topo, links + links, table, q, qd, f, 1e-3, fl, False, 0.0, 1.0)[0] == EINVAL     # twice
    assert abi_call(topo, links, table, q, qd, f, 1e-3, fl, False, 0.0, 1.0)[0] == 0
    with pytest.raises(AssertionError):
        m.compute_contact_rollout(q, qd, f, names, 1e-3, stabilization=-1.0)
    with pytest.raises(AssertionError):
        m.compute_contact_rollout(q, qd, f, names, 1e-3, target_pos=tp)
    with pytest.raises(AssertionError):
        m.compute_contact_rollout(q, qd, f, names, 1e-3, target_pos=tp, target_quat=tq, position_only=True)
    with pytest.raises(AssertionError):
        m.compute_contact_rollout(q, qd, f[0], names, 1e-3)
    with pytest.raises(AssertionError):
        m.compute_contact_rollout(q, qd, f, names, 1e-3, target_pos=tp[:, :2], target_quat=tq[:, :2])
    with pytest.raises(KeyError):
        m.compute_contact_rollout(q, qd, f, ["nope"], 1e-3)


def test_branch_point_limit_is_refused_with_elimit(model_dir):
    """The articulated-body code holds at most 8 live branch points: a hand of 8 fingers on an arm (9) is refused on the
    host with ELIMIT, before any launch."""
    spec = CDT.SR.refusal_families()["H_nine_slots"]
    path = CDT.SR.build(spec, model_dir)
    m = drm.DifferentiableRobotModel(path, "H_nine_slots", device=DEV)
    r32 = O.load_robot(path, torch.float32)
    q, qd, f = OSDT.inputs(r32, 4, seed=1)
    links = [len(r32.names) - 1]
    table = m._link_table().detach()                # the table build is a launch of its own
    before = engine.launch_count()
    rc, _ = abi_call(m._topology, links, table, q.to(DEV), qd.to(DEV), f[None].to(DEV), 1e-3, 0, True, 0.0, 1.0)
    assert rc == ELIMIT, (rc, engine.lib().drmb200_last_error())
    assert engine.launch_count() == before


def test_one_row_ctas_stay_far_below_the_shared_memory_limit():
    """The ELIMIT for a one-row CTA over 227 KB guards the layout, but no model the engine accepts reaches it: at its
    limits (64 links and joints, 8 links in pose mode, M = 48, 8 live branch points) a row needs about 40 KB.  So the
    refusal is checked by the bound, not by a model."""
    n = L = n_u = n_jslots = 64
    E, M, slots = 8, 48, 8
    need = 4 * rollout_floats(1, n, L, slots, n_u, M, n_jslots, slots, E, True) + STATIC_SMEM
    assert need < 48 * 1024 < TM.SMEM_CAP, need
    for name in sorted(CDT.FAM):                   # and the mirror finds a tile for every family's deepest 8 pose links
        par, mov = CDT.FAM[name].doc()
        if sum(mov[1:]) == 0:
            continue
        import test_launch_geometry_solvers_gpu as LG
        links = LG.deepest(par, mov, min(8, sum(mov[1:])))
        if CDT._solvable(par, mov, links):
            assert rollout_choice(par, mov, links, True)[0] is not None, name
