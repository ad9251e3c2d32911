"""GPU: contact dynamics and contact impulses (compute_contact_dynamics / compute_contact_impulse, csrc/contact_dynamics.cu)
against the fp64 oracle (tests/contact_oracle.py), the reference's goldens and compositions of the existing kernels; on
every shipped robot, every tile the host rule chooses, the synthetic topology families, learnable and fused models.

Errors are per configuration, relative to that configuration's largest entry of the same output; the bound is
max(8 x the fp32 oracle's error on the same rows, 2e-5).  Values are compared on the rows all three (kernel, fp64 and fp32
oracle) solve whose fp64 smallest scaled pivot is at least 100x the threshold: below that the solution's fp32 error is
set by how each path rounds A, which differs between the kernel's sweeps and the oracle's autograd.  `solved` is compared
on every row except those fp32 arithmetic cannot decide: the fp64 smallest pivot within 10x of the threshold, the fp32
oracle deciding differently from the fp64 one, or a system singular in exact arithmetic (fp64 pivot below 1e-9), whose
fp32 pivot is rounding noise that can exceed the threshold.  Unsolved rows must be NaN."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor
from conftest import GOLDEN_DIR, URDFS, urdf_path
import contact_oracle as C
import osd_oracle as S
import synthetic_robots as SR
import test_operational_space_gpu as OSDT
import tile_mirrors as TM
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL, LARGE = 131, 4099
LARGE_ROWS = torch.cat([torch.arange(SMALL, LARGE - 3, 97), torch.arange(LARGE - 3, LARGE)])
TIPS = OSDT.TIPS
TRI = ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"]
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -1                            # DRMB200_EINVAL
model_of = OSDT.model_of


def bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def per_config_error(got, want):
    return OSDT.per_config_error(got, want) if want.shape[0] else 0.0


def check_contact(what, got, w64, w32, floors=(1e-4, 2e-5), slack=8):
    """got: the kernel's (joint output, lambda, solved); w64 / w32: the oracle's (joint output, lambda, solved, min pivot).
    The bound is max(slack x the fp32 oracle's error, floor)."""
    out, lam, ok = (t.cpu() for t in got)
    o64, l64, ok64, piv = w64
    o32, l32, ok32, _ = w32
    undecidable = ((piv > C.PIVOT_MIN / 10) & (piv < C.PIVOT_MIN * 10)) | (ok32 != ok64) | (piv < 1e-9)
    wrong = (ok != ok64) & ~undecidable
    assert not bool(wrong.any()), f"{what}: solved {ok[wrong].tolist()} where the fp64 oracle says {ok64[wrong].tolist()} " \
                                  f"(min pivots {piv[wrong].tolist()})"
    assert bool(torch.isnan(out[~ok]).all()) and bool(torch.isnan(lam[~ok]).all()), f"{what}: unsolved rows are not NaN"
    assert bool(torch.isfinite(out[ok]).all()) and bool(torch.isfinite(lam[ok]).all()), f"{what}: solved rows not finite"
    rows = ok & ok64 & ok32 & (piv >= 100 * C.PIVOT_MIN)
    for name, g, a, b, floor in (("joints", out, o64, o32, floors[0]), ("lambda", lam, l64, l32, floors[1])):
        e32 = per_config_error(b[rows], a[rows])
        err = per_config_error(g[rows], a[rows])
        bound = max(slack * e32, floor)
        print(f"ERR {what} {name}: {err:.2e} (bound {bound:.2e}) rows {int(rows.sum())}/{len(rows)}")
        assert np.isfinite(err) and err <= bound, f"{what} {name}: per-configuration error {err:.3e} > {bound:.3e} (fp32 {e32:.2e})"
    return int(rows.sum())


def robots(stem_or_path, nonsym):
    return OSDT.robots(stem_or_path, nonsym)


class Pieces:
    """The oracle's J (pose), G, Jdot qd (pose) and qdd_free per flag combination, computed once per robot and rows."""

    def __init__(self, robot, q, qd, f, links):
        self.robot, self.q, self.qd, self.f = robot, q, qd, f
        self.J = S.stacked_jacobian(robot, q, links).detach()
        self.G = S.force_response(robot, q)
        self.bias = S.bias_acceleration(robot, q, qd, links).detach()

    def _sel(self, pos):
        if not pos:
            return self.J, self.bias
        idx = torch.cat([torch.arange(6 * e, 6 * e + 3) for e in range(self.J.shape[1] // 6)])
        return self.J[:, idx], self.bias[:, idx]

    def max_diag(self, pos):
        J, _ = self._sel(pos)
        return float(torch.diagonal(J @ self.G @ J.transpose(1, 2), dim1=1, dim2=2).max())

    def dynamics(self, grav, damp, pos, mu, a_ref):
        J, bias = self._sel(pos)
        qdd = O.forward_dynamics(self.robot, self.q, self.qd, self.f, grav, damp).detach()
        ref = torch.zeros_like(bias) if a_ref is None else a_ref.to(bias.dtype)
        return C.respond(J, self.G, qdd, ref - torch.einsum("bmn,bn->bm", J, qdd) - bias, mu)

    def impulse(self, pos, mu, v_ref):
        J, _ = self._sel(pos)
        vel = torch.einsum("bmn,bn->bm", J, self.qd)
        ref = torch.zeros_like(vel) if v_ref is None else v_ref.to(vel.dtype)
        return C.respond(J, self.G, self.qd, ref - vel, mu)


def link_sets(stem, robot):
    """(links, position_only): the end effector's pose, and several links' positions."""
    if "allegro" in stem:
        multi = TIPS
    elif stem == "trifinger_edu":
        multi = TRI
    else:
        multi = list(dict.fromkeys([OSDT.EE[stem], robot.names[len(robot.names) // 2]]))
    return [([OSDT.EE[stem]], False), (multi, True)]


def refs(B, M, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, M, generator=g), 0.1 * torch.randn(B, M, generator=g)


# ------------------------------------------------------------------------------------------------
# shipped robots against the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_shipped_robots_match_oracle(stem, nonsym):
    r32, r64, table = robots(stem, nonsym)
    topo = model_of(stem)._topology
    compared = 0
    # jaco_clean's finger links weigh grams: the kernel's A (articulated-body sweeps) and the oracle's (autograd) round
    # differently by more than the fp32 oracle's own error on the fingertip-plus-hand set, as the operational-space
    # acceleration does there (its test allows 1e-4)
    slack = 32 if stem == "jaco_clean" else 8
    for links, pos in link_sets(stem, r32):
        idx = [r32.index(nm) for nm in links]
        M = (3 if pos else 6) * len(links)
        for B in (SMALL, LARGE):
            q, qd, f = OSDT.inputs(r32, B)
            a_ref, v_ref = refs(B, M, 8)
            rows = torch.arange(B) if B == SMALL else LARGE_ROWS
            sub = [t[rows] for t in (q, qd, f)]
            p64 = Pieces(r64, *(t.double() for t in sub), links)
            p32 = Pieces(r32, *sub, links)
            dev = [t.to(DEV) for t in (q, qd, f, a_ref, v_ref)]
            for mu in (0.0, 1e-3 * p64.max_diag(pos)):
                for grav, damp in ((True, False), (False, True)):
                    flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
                    got = engine.contact_dynamics_raw(topo, idx, table, *dev[:3], flags, dev[3], pos, mu)
                    what = f"{stem} B={B} {links} pos={pos} mu={mu:.3g} g{grav:d}d{damp:d} dynamics"
                    compared += check_contact(what, [t[rows] for t in got], p64.dynamics(grav, damp, pos, mu, a_ref[rows]),
                                              p32.dynamics(grav, damp, pos, mu, a_ref[rows]), slack=slack)
                got = engine.contact_impulse_raw(topo, idx, table, dev[0], dev[1], dev[4], pos, mu)
                compared += check_contact(f"{stem} B={B} {links} pos={pos} mu={mu:.3g} impulse", [t[rows] for t in got],
                                          p64.impulse(pos, mu, v_ref[rows]), p32.impulse(pos, mu, v_ref[rows]), slack=slack)
    assert compared > 0


GOLDEN = ["2link_robot", "iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro", "trifinger_edu"]


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".contact.npz"), allow_pickle=False)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"], dtype=torch.float32)
        inertia[0] = r32.inertia[0]
        r32.inertia = inertia
    table = O.link_table(r32).float().to(DEV).contiguous()
    links = [str(s) for s in g["links"]]
    pos, mu = bool(g["position_only"]), float(g["mu"])
    q, qd, f, a_ref, v_ref = (torch.tensor(g[k]) for k in ("q", "qd", "f", "a_ref", "v_ref"))
    idx = [r32.index(nm) for nm in links]
    topo = model_of(stem)._topology
    dyn = engine.contact_dynamics_raw(topo, idx, table, q.to(DEV), qd.to(DEV), f.to(DEV), engine.GRAVITY, a_ref.to(DEV), pos, mu)
    imp = engine.contact_impulse_raw(topo, idx, table, q.to(DEV), qd.to(DEV), v_ref.to(DEV), pos, mu)
    r64 = r32.to(torch.float64)
    w_dyn = C.contact_dynamics(r64, q.double(), qd.double(), f.double(), links, a_ref.double(), True, False, pos, mu)
    w_imp = C.contact_impulse(r64, q.double(), qd.double(), links, v_ref.double(), pos, mu)
    assert bool(dyn[2].all()) and bool(imp[2].all())
    w32_dyn = C.contact_dynamics(r32, q, qd, f, links, a_ref, True, False, pos, mu)
    w32_imp = C.contact_impulse(r32, q, qd, links, v_ref, pos, mu)
    check_contact(f"{stem} {tag} dynamics", dyn, w_dyn, w32_dyn, floors=(2e-4, 2e-4))      # 8 rows: the floor of the OSD goldens
    check_contact(f"{stem} {tag} impulse", imp, w_imp, w32_imp, floors=(2e-4, 2e-4))
    pre = "" if tag == "sym" else "nonsym."
    for got, name in ((dyn[0], "qdd"), (dyn[1], "force"), (imp[0], "qd_plus"), (imp[1], "impulse")):
        # the goldens solve the reference's fp32 pieces: on TriFinger's light fingers they carry ~1e-2 of that rounding
        gold = torch.tensor(g[pre + name])
        assert per_config_error(got.cpu(), gold) < 2e-2, (name, per_config_error(got.cpu(), gold))


# ------------------------------------------------------------------------------------------------
# identities with the existing kernels
# ------------------------------------------------------------------------------------------------
CONSISTENCY = [("iiwa7", ["iiwa_link_ee"], False, 0.0), ("panda", ["panda_virtual_ee_link"], False, 0.0),
               ("allegro_hand_description_left", TIPS, True, 0.0), ("trifinger_edu", TRI, True, 0.0),
               ("iiwa7_allegro", TIPS, True, 0.0), ("iiwa7_allegro", TIPS, False, 50.0)]


def stacked_jacobian_from_fk(m, q, links, position_only):
    return OSDT.stacked_jacobian_from_fk(m, q, links, position_only)


@pytest.mark.parametrize("stem,links,pos,mu", CONSISTENCY)
def test_identities_with_existing_kernels(stem, links, pos, mu):
    m = model_of(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f = (t.to(DEV) for t in OSDT.inputs(r32, 1000, seed=5))
    M = (3 if pos else 6) * len(links)
    a_ref, v_ref = (t.to(DEV) for t in refs(1000, M, 9))
    qdd, lam, ok = m.compute_contact_dynamics(q, qd, f, links, a_ref, True, True, pos, mu)
    assert float(ok.float().mean()) > 0.9
    with torch.no_grad():
        J = stacked_jacobian_from_fk(m, q, links, pos).double()
        osd = m.compute_operational_space_dynamics(q, qd, f, links, True, True, pos)
        fd = m.compute_forward_dynamics(q, qd, f + torch.einsum("bmn,bm->bn", J, lam.double()).float(), True, True)
    # both paths round in fp32: compare on the rows whose equilibrated system is well conditioned
    A = osd.inv_inertia.double() + mu * torch.eye(M, device=DEV, dtype=torch.float64)
    s = torch.diagonal(A, dim1=1, dim2=2).abs().rsqrt()
    well = torch.linalg.cond(s[:, :, None] * A * s[:, None, :]) < 1e3
    assert int(well.sum()) >= 100
    ok = ok & well
    k = ok
    assert per_config_error(qdd[k], fd[k]) < 2e-3
    lam_osd = torch.linalg.solve(A[k], a_ref.double()[k] - osd.acceleration.double()[k])
    assert per_config_error(lam[k], lam_osd) < 2e-3
    # relative to the terms that cancel: light fingers reach 1e5 rad/s^2 while a_ref is O(1)
    Jqdd, bias = torch.einsum("bmn,bn->bm", J[k], qdd.double()[k]), osd.bias_acceleration.double()[k]
    terms = torch.einsum("bmn,bn->bm", J[k].abs(), qdd.double()[k].abs())
    scale = torch.maximum(terms.amax(1), bias.abs().amax(1)).clamp_min(1.0)
    err = (Jqdd + bias - (a_ref.double()[k] - mu * lam.double()[k])).abs().amax(1)
    assert float((err / scale).max()) < 2e-3
    # the impulse: inelastic contact does not add kinetic energy; the constrained velocity is v_ref - mu Lambda
    qp, imp, ok = m.compute_contact_impulse(q, qd, links, None, pos, mu)
    ok = ok & well
    k = ok
    T0 = m.compute_energy_and_momentum(q, qd).kinetic_energy.double()
    T1 = m.compute_energy_and_momentum(q, qp.nan_to_num()).kinetic_energy.double()
    assert bool((T1[k] <= T0[k] * (1 + 1e-4) + 1e-6).all())
    assert per_config_error(torch.einsum("bmn,bn->bm", J[k], qp.double()[k]), -mu * imp.double()[k]) < 2e-3 or mu == 0
    if mu == 0:
        assert float(torch.einsum("bmn,bn->bm", J[k], qp.double()[k]).abs().max()) < 1e-3 * float(qd.abs().max())
        # elastic: kinetic energy kept
        v = torch.einsum("bmn,bn->bm", J, qd.double()).float()
        qe, _, ok = m.compute_contact_impulse(q, qd, links, -v, pos, 0.0)
        ok = ok & well
        Te = m.compute_energy_and_momentum(q, qe.nan_to_num()).kinetic_energy.double()
        assert float(((Te - T0).abs() / T0)[ok].max()) < 1e-3


# ------------------------------------------------------------------------------------------------
# launch geometry: every tile the host rule chooses
# ------------------------------------------------------------------------------------------------
STATIC_SMEM = 128                      # the mbarrier, as for the operational-space kernel (-Xptxas -v)


def contact_floats(T, n, n_links, tree_slots, n_u, M, n_jslots, n_state_slots):
    """ContactSmemLayout(T, tree program, walk, M).total_floats."""
    aba = 4 * T * n + n_links * TM.TABLE_STRIDE + n_links * 14 * T + tree_slots * 42 * T
    return TM.up4(aba) + T * (M + M * n_u + 6 * n_jslots + 24 * n_state_slots + 4 * M + M * M + n)


def contact_choice(parents, movable, links, pose):
    n = sum(movable[1:])
    _, n_u, n_jslots, n_slots = TM.multi_program(parents, movable, links)
    M = (6 if pose else 3) * len(links)
    tree_slots = SR.live_slots(parents)
    return TM.ladder(lambda T: contact_floats(T, n, len(parents), tree_slots, n_u, M, n_jslots, n_slots), STATIC_SMEM)


FAM = SR.families()


def _solvable(par, mov, links):
    """Links that each have a movable joint on their root path."""
    def movable_path(l):
        while l > 0:
            if mov[l]:
                return True
            l = par[l]
        return False
    return all(movable_path(l) for l in links)


def _tile_cases():
    import test_launch_geometry_solvers_gpu as LG
    cases = {}
    for name in sorted(FAM):
        par, mov = FAM[name].doc()
        if sum(mov[1:]) == 0:
            continue
        for k in range(1, 9):
            links = LG.deepest(par, mov, k)
            if not _solvable(par, mov, links):
                continue
            _, n_u, _, _ = TM.multi_program(par, mov, links)
            for pose in (True, False):
                M = (6 if pose else 3) * len(links)
                branch = "task" if M <= n_u else "joint"
                tile, _ = contact_choice(par, mov, links, pose)
                cases.setdefault((tile, pose, branch), (name, links))
    return cases


TILE_CASES = _tile_cases()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_contact"))


def family(name, model_dir):
    import test_launch_geometry_solvers_gpu as LG
    return LG.family(name, model_dir)


def shifted(t):
    if t is None:
        return None
    buf = torch.empty(t.numel() + 1, device=DEV, dtype=t.dtype) if t.dtype == torch.float32 else \
        torch.empty(t.numel() + 4, device=DEV, dtype=t.dtype)
    off = 1 if t.dtype == torch.float32 else 4
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def contact_call(topo, links, table, x, flags, pos, mu, impulse=False, want_lambda=True, misaligned=False):
    """One C-ABI call with caller-allocated outputs (optionally 4 bytes off 16-byte alignment, inputs and outputs)."""
    q, qd, f, ref = x
    B, n = q.shape
    M = (3 if pos else 6) * len(links)
    out = torch.empty((B, n), device=DEV)
    lam = torch.empty((B, M), device=DEV) if want_lambda else None
    ok = torch.empty(B, device=DEV, dtype=torch.uint8)
    if misaligned:
        q, qd, f, ref, out, lam = (shifted(t) for t in (q, qd, f, ref, out, lam))
    idx = (ctypes.c_int32 * len(links))(*links)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    lib = engine.lib()
    if impulse:
        rc = lib.drmb200_contact_impulse(ctypes.byref(topo), len(links), idx, ptr(table), ptr(q), ptr(qd), ptr(ref), B, int(pos),
                                         ctypes.c_float(mu), ptr(out), ptr(lam), ptr(ok), s)
    else:
        rc = lib.drmb200_contact_dynamics(ctypes.byref(topo), len(links), idx, ptr(table), ptr(q), ptr(qd), ptr(f), ptr(ref), B,
                                          flags, int(pos), ctypes.c_float(mu), ptr(out), ptr(lam), ptr(ok), s)
    assert rc == 0, lib.drmb200_last_error()
    return out, lam, ok.bool()


def same_rows(what, small, big):
    for a, b in zip(small, big):
        if a is not None:
            assert same_bits(a, b[:a.shape[0]]), f"{what}: rows differ from the {LARGE}-row batch"


@pytest.mark.parametrize("key", sorted(TILE_CASES, key=str),
                         ids=[f"T{t}-{'pose' if p else 'pos'}-{b}" for (t, p, b) in sorted(TILE_CASES, key=str)])
def test_contact_at_every_tile(key, model_dir):
    tile, pose, branch = key
    name, links = TILE_CASES[key]
    m, r32, r64, table = family(name, model_dir)
    topo = m._topology
    pos = not pose
    M = (3 if pos else 6) * len(links)
    q, qd, f = OSDT.inputs(r32, LARGE, seed=22)
    a_ref, v_ref = refs(LARGE, M, 23)
    rows = torch.unique(torch.cat([torch.arange(min(3 * tile + 4, LARGE)), torch.arange(3 * tile + 4, LARGE - 3, 211),
                                   torch.arange(LARGE - 3, LARGE)]))
    names = [r32.names[l] for l in links]
    sub = [t[rows] for t in (q, qd, f)]
    p64 = Pieces(r64, *(t.double() for t in sub), names)
    p32 = Pieces(r32, *sub, names)
    mu = 1e-3 * p64.max_diag(pos)
    xd = [t.to(DEV) for t in (q, qd, f, a_ref)]
    xi = [t.to(DEV) for t in (q, qd, f, v_ref)]
    for impulse, x in ((False, xd), (True, xi)):
        big = contact_call(topo, links, table, x, engine.GRAVITY | engine.DAMPING, pos, mu, impulse)
        w64 = p64.impulse(pos, mu, v_ref[rows]) if impulse else p64.dynamics(True, True, pos, mu, a_ref[rows])
        w32 = p32.impulse(pos, mu, v_ref[rows]) if impulse else p32.dynamics(True, True, pos, mu, a_ref[rows])
        check_contact(f"{name} {len(links)} links T={tile} {branch} pos={pos} impulse={impulse}", [t[rows] for t in big], w64, w32)
        for B in sorted({1, max(1, tile - 1), tile, tile + 1, 3 * tile + 3}):
            same_rows(f"{name} B={B}", contact_call(topo, links, table, [t[:B] for t in x], engine.GRAVITY | engine.DAMPING,
                                                    pos, mu, impulse), big)
        same_rows(f"{name} misaligned", contact_call(topo, links, table, x, engine.GRAVITY | engine.DAMPING, pos, mu, impulse,
                                                     misaligned=True), big)
        part = contact_call(topo, links, table, x, engine.GRAVITY | engine.DAMPING, pos, mu, impulse, want_lambda=False,
                            misaligned=True)
        assert part[1] is None and same_bits(part[0], big[0]) and torch.equal(part[2], big[2])


def test_every_reachable_rung_has_a_case():
    tiles = {k[0] for k in TILE_CASES}
    assert {64, 32, 16, 8, 4} <= tiles, tiles
    assert {k[2] for k in TILE_CASES} == {"task", "joint"}


def test_static_shared_memory_is_what_the_mirror_adds():
    lib = engine.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    for t in TM.LADDER:
        for b in (0, 1):
            sym = f"_ZN3drm23contact_dynamics_kernelILi{t}ELb{b}EEEvNS_11TreeProgramENS_12UnionProgramENS_11ContactArgsE"
            attr = (ctypes.c_size_t * 64)()
            rc = cudart.cudaFuncGetAttributes(attr, ctypes.cast(getattr(lib, sym), ctypes.c_void_p))
            assert rc == 0, (sym, rc)
            assert attr[0] == STATIC_SMEM, (sym, attr[0])


# ------------------------------------------------------------------------------------------------
# synthetic topologies
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(FAM))
def test_synthetic_families_match_oracle_or_are_refused(name, model_dir):
    spec = FAM[name]
    path = SR.build(spec, model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    r32, r64, table = robots(path, True)
    par, mov = spec.doc()
    names = r32.names
    links = [l for l in dict.fromkeys([len(names) - 1, len(names) // 2]) if l > 0] or [0]
    q, qd, f = OSDT.inputs(r32, 37, seed=17)
    dev = [t.to(DEV) for t in (q, qd, f)]
    if r32.n_dofs == 0 or not _solvable(par, mov, links):
        before = engine.launch_count()
        with pytest.raises(RuntimeError, match="no movable joint"):
            engine.contact_dynamics_raw(m._topology, links, table, *dev, 0, None, True, 0.1)
        assert engine.launch_count() == before
        return
    rows = torch.arange(0, 37, 4)
    sub = [t[rows] for t in (q, qd, f)]
    lnames = [names[l] for l in links]
    p64 = Pieces(r64, *(t.double() for t in sub), lnames)
    p32 = Pieces(r32, *sub, lnames)
    for pos in (False, True):
        tile, need = contact_choice(par, mov, links, not pos)
        assert tile is not None, f"{name}: the mirror expects a refusal ({need} B)"
        mu = 1e-3 * p64.max_diag(pos)
        got = engine.contact_dynamics_raw(m._topology, links, table, *dev, engine.GRAVITY, None, pos, mu)
        check_contact(f"{name} T={tile} pos={pos} dynamics", [t.cpu()[rows] for t in got],
                      p64.dynamics(True, False, pos, mu, None), p32.dynamics(True, False, pos, mu, None))
        got = engine.contact_impulse_raw(m._topology, links, table, dev[0], dev[1], None, pos, mu)
        check_contact(f"{name} T={tile} pos={pos} impulse", [t.cpu()[rows] for t in got], p64.impulse(pos, mu, None),
                      p32.impulse(pos, mu, None))


@pytest.mark.parametrize("name", ["H_nine_slots"])
def test_too_many_branch_points_give_the_forward_dynamics_message_without_a_launch(name, model_dir):
    spec = SR.refusal_families()[name]
    path = SR.build(spec, model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    r32, _, table = robots(path, False)
    q, qd, f = (t.to(DEV) for t in OSDT.inputs(r32, 4, seed=1))
    with pytest.raises(RuntimeError) as fd:
        engine.forward_dynamics_raw(m._topology, table, q, qd, f, 0)
    msg = str(fd.value).split("): ", 1)[1]
    par, mov = spec.doc()
    import test_launch_geometry_solvers_gpu as LG
    links = LG.deepest(par, mov, 1)
    before = engine.launch_count()
    with pytest.raises(RuntimeError, match=r"code -3\): ") as got:
        engine.contact_dynamics_raw(m._topology, links, table, q, qd, f, 0)
    assert str(got.value).split("): ", 1)[1] == msg
    with pytest.raises(RuntimeError, match=r"code -3\): ") as got:
        engine.contact_impulse_raw(m._topology, links, table, q, qd)
    assert str(got.value).split("): ", 1)[1] == msg
    assert engine.launch_count() == before


# ------------------------------------------------------------------------------------------------
# models, capture and edge cases
# ------------------------------------------------------------------------------------------------
def test_learnable_and_fused_models_use_current_values():
    stem = "iiwa7"
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f = (t.to(DEV) for t in OSDT.inputs(r32, 333, seed=13))
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
    links = ["iiwa_link_ee"]
    idx = [models[0]._name_to_idx_map[nm] for nm in links]
    want_d = engine.contact_dynamics_raw(models[0]._topology, idx, table, q, qd, f, engine.GRAVITY)
    want_i = engine.contact_impulse_raw(models[0]._topology, idx, table, q, qd)
    const = model_of(stem).compute_contact_dynamics(q, qd, f, links)
    assert OSDT.rel(want_d[0].nan_to_num(), const[0].nan_to_num()) > 1e-4
    for m in models:
        for got, want in ((m.compute_contact_dynamics(q, qd, f, links), want_d), (m.compute_contact_impulse(q, qd, links), want_i)):
            for a, b in zip(got, want):
                assert not a.requires_grad
                assert same_bits(a, b)


def test_one_launch_per_call_and_cuda_graph_capture():
    m = model_of("iiwa7_allegro")
    r32 = O.load_robot(urdf_path("iiwa7_allegro"), torch.float32)
    q, qd, f = (t.to(DEV) for t in OSDT.inputs(r32, 4099, seed=15))
    a_ref = torch.randn(4099, 24, device=DEV)
    want = m.compute_contact_dynamics(q, qd, f, TIPS, a_ref, regularization=50.0)
    want_i = m.compute_contact_impulse(q, qd, TIPS, regularization=50.0)
    torch.cuda.synchronize()
    for call in (lambda: m.compute_contact_dynamics(q, qd, f, TIPS, position_only=True),
                 lambda: m.compute_contact_impulse(q, qd, TIPS, position_only=True)):
        before = engine.launch_count()
        call()
        assert engine.launch_count() == before + 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_contact_dynamics(q, qd, f, TIPS, a_ref, regularization=50.0)
        m.compute_contact_impulse(q, qd, TIPS, regularization=50.0)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = m.compute_contact_dynamics(q, qd, f, TIPS, a_ref, regularization=50.0)
        got_i = m.compute_contact_impulse(q, qd, TIPS, regularization=50.0)
    for t in (*got, *got_i):
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip((*got, *got_i), (*want, *want_i)):
        assert same_bits(a, b)
    assert bool(want.solved.all())


def test_force_can_be_skipped():
    m = model_of("panda")
    r32, _, table = robots("panda", False)
    q, qd, f = (t.to(DEV) for t in OSDT.inputs(r32, 300, seed=18))
    idx = [m._name_to_idx_map["panda_virtual_ee_link"]]
    topo = m._topology
    full = engine.contact_dynamics_raw(topo, idx, table, q, qd, f, engine.GRAVITY)
    part = engine.contact_dynamics_raw(topo, idx, table, q, qd, f, engine.GRAVITY, want_force=False)
    assert part[1] is None and same_bits(part[0], full[0]) and torch.equal(part[2], full[2])
    full = engine.contact_impulse_raw(topo, idx, table, q, qd)
    part = engine.contact_impulse_raw(topo, idx, table, q, qd, want_impulse=False)
    assert part[1] is None and same_bits(part[0], full[0]) and torch.equal(part[2], full[2])


def test_edge_cases_and_argument_errors():
    m = model_of("iiwa7")
    n = m._n_dofs
    r32 = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd, f = (t.to(DEV) for t in OSDT.inputs(r32, 3, seed=16))
    links = ["iiwa_link_ee"]
    empty = torch.zeros(0, n, device=DEV)
    before = engine.launch_count()
    out = m.compute_contact_dynamics(empty, empty, empty, links)
    assert out.qdd.shape == (0, n) and out.force.shape == (0, 6) and out.solved.shape == (0,)
    out = m.compute_contact_impulse(empty, empty, links, position_only=True)
    assert out.qd_plus.shape == (0, n) and out.impulse.shape == (0, 3)
    assert engine.launch_count() == before
    one = m.compute_contact_dynamics(q[1], qd[1], f[1], links, None, False, True, True, 0.01)
    full = m.compute_contact_dynamics(q, qd, f, links, None, False, True, True, 0.01)
    assert one.qdd.shape == (n,) and one.force.shape == (3,) and one.solved.dtype == torch.bool and one.solved.ndim == 0
    for a, b in zip(one, full):
        assert same_bits(a, b[1])
    onei = m.compute_contact_impulse(q[1], qd[1], links, torch.ones(3, device=DEV), True)
    assert onei.qd_plus.shape == (n,) and onei.impulse.shape == (3,)
    with pytest.raises(AssertionError):
        m.compute_contact_dynamics(q, qd, f, ["iiwa_link_ee", "iiwa_link_ee"])
    with pytest.raises(KeyError):
        m.compute_contact_impulse(q, qd, ["no_such_link"])
    with pytest.raises(AssertionError):
        m.compute_contact_dynamics(q, qd, f, links, torch.zeros(3, 5, device=DEV))
    table, topo = m._link_table().detach(), m._topology
    ee = m._name_to_idx_map["iiwa_link_ee"]
    einval = [([], 0.0, "n_ee"), (list(range(1, 10)), 0.0, "n_ee"), ([ee, ee], 0.0, "twice"), ([99], 0.0, "range"),
              ([-1], 0.0, "range"), ([0], 0.0, "no movable joint"), ([ee], -1.0, "regularization"),
              ([ee], float("nan"), "regularization"), ([ee], float("inf"), "regularization")]
    before = engine.launch_count()
    for bad, mu, _ in einval:
        with pytest.raises(RuntimeError, match=r"drmb200_contact_dynamics failed \(code -"):
            engine.contact_dynamics_raw(topo, bad, table, q, qd, f, 0, regularization=mu)
        with pytest.raises(RuntimeError, match=r"drmb200_contact_impulse failed \(code -"):
            engine.contact_impulse_raw(topo, bad, table, q, qd, regularization=mu)
    # null required pointers and a negative batch, through the C ABI
    lib = engine.lib()
    idx = (ctypes.c_int32 * 1)(ee)
    out, lam, ok = torch.empty(3, n, device=DEV), torch.empty(3, 6, device=DEV), torch.empty(3, device=DEV, dtype=torch.uint8)
    args = [ptr(table), ptr(q), ptr(qd), ptr(f)]
    for k in range(len(args) + 2):
        a = list(args) + [ptr(out), ptr(ok)]
        a[k] = None
        rc = lib.drmb200_contact_dynamics(ctypes.byref(topo), 1, idx, a[0], a[1], a[2], a[3], None, 3, 0, 0,
                                          ctypes.c_float(0.0), a[4], ptr(lam), a[5], None)
        assert rc == EINVAL
    for k in range(5):
        a = [ptr(table), ptr(q), ptr(qd), ptr(out), ptr(ok)]
        a[k] = None
        rc = lib.drmb200_contact_impulse(ctypes.byref(topo), 1, idx, a[0], a[1], a[2], None, 3, 0, ctypes.c_float(0.0), a[3],
                                         ptr(lam), a[4], None)
        assert rc == EINVAL
    rc = lib.drmb200_contact_impulse(ctypes.byref(topo), 1, idx, ptr(table), ptr(q), ptr(qd), None, -1, 0, ctypes.c_float(0.0),
                                     ptr(out), ptr(lam), ptr(ok), None)
    assert rc == EINVAL and b"batch" in lib.drmb200_last_error()
    torch.cuda.synchronize()
    assert engine.launch_count() == before
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        engine.contact_dynamics_raw(topo, [ee], table, q.cpu(), qd.cpu(), f.cpu(), 0)
    with pytest.raises(RuntimeError, match="fp32-only"):
        engine.contact_impulse_raw(topo, [ee], table, q.double(), qd.double())


def test_redundant_sets_are_unsolved_without_regularisation():
    m = model_of("iiwa7_allegro")
    r32 = O.load_robot(urdf_path("iiwa7_allegro"), torch.float32)
    q, qd, f = (t.to(DEV) for t in OSDT.inputs(r32, 500, seed=19))
    # 24 rows, 23 joints: singular in exact arithmetic.  In fp32 the last pivot is rounding noise, which stays below the
    # threshold on most rows but not all: `solved` is not a rank test, and such sets need regularisation
    out = m.compute_contact_dynamics(q, qd, f, TIPS)
    print(f"redundant, mu = 0: {float(out.solved.float().mean()):.3f} of the rows solved")
    assert float(out.solved.float().mean()) < 0.5
    assert bool(torch.isnan(out.qdd[~out.solved]).all()) and bool(torch.isnan(out.force[~out.solved]).all())
    out = m.compute_contact_impulse(q, qd, TIPS)
    print(f"redundant impulse, mu = 0: {float(out.solved.float().mean()):.3f} of the rows solved")
    assert float(out.solved.float().mean()) < 0.5
    assert bool(m.compute_contact_dynamics(q, qd, f, TIPS, regularization=100.0).solved.all())


# ------------------------------------------------------------------------------------------------
# the example
# ------------------------------------------------------------------------------------------------
def test_pinned_end_effector_example(tmp_path):
    """1 s at dt = 1e-3 under random torques: the pinned point drifts < 1 mm; the same rollout without the contact moves
    it more than 1 cm."""
    out = subprocess.run([sys.executable, os.path.join(REPO, "examples", "pinned_end_effector_iiwa.py"), "--steps", "1000",
                          "--json"], capture_output=True, text=True, cwd=str(tmp_path), timeout=900,
                         env=dict(os.environ, PYTHONPATH=os.pathsep.join([REPO, os.environ.get("PYTHONPATH", "")])))
    assert out.returncode == 0, out.stderr[-3000:]
    import json
    res = json.loads(out.stdout.strip().splitlines()[-1])
    assert res["max_drift_m"] < 1e-3, res
    assert res["free_drift_m"] > 1e-2, res
    assert res["joint_motion_rad"] > 1e-2, res
