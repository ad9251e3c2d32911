"""GPU: the dynamics-derivatives, inverse-kinematics, multi-link inverse-kinematics and operational-space kernels at every
tile size their host code can choose, and every kernel on joint angles beyond the fast sin / cos range.

The tile a model lands on comes from the mirrors of tests/tile_mirrors.py (pinned to the host code by
tests/test_tile_choice.py); each case asserts its tile before it runs.  Per case:
  * the fp64 oracle at batch sizes 1, T - 1, T, T + 1, 3T + 3 and a ragged multi-wave batch of 4 099 rows (checked on a
    spread of rows from every tile plus the tail), bound max(8 x the fp32 oracle's error, 2e-5) per configuration;
  * every row bit-identical across those batch sizes, and with every input and output 4 bytes off 16-byte alignment
    (through the C ABI);
  * every flag combination and both modes; for the derivatives the unfolded program ("rnea_fold" = 0) and every subset of
    the outputs, for the IK kernels per-row damping without joint limits.
"""
import ctypes

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
import derivatives_oracle as D
import ik_multi_oracle as IKM
import ik_oracle as IK
import rollout_oracle as RO
import synthetic_robots as S
import tile_mirrors as TM
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LARGE = 4099
FLAGS = [(True, True), (True, False), (False, True), (False, False)]
FAM = S.families()
_MODELS = {}


# ------------------------------------------------------------------------------------------------
# cases: the first family / link set (k deepest links, k = 1..8) that lands on each tile
# ------------------------------------------------------------------------------------------------
def deepest(par, mov, k):
    def depth(l):
        d = 0
        while l > 0:
            d, l = d + mov[l], par[l]
        return d
    return sorted(range(1, len(par)), key=lambda l: (-depth(l), l))[:k]


def _solver_cases():
    ikm, osd = {}, {}
    for name in sorted(FAM):
        par, mov = FAM[name].doc()
        if sum(mov[1:]) == 0:
            continue
        for k in range(1, 9):
            links = deepest(par, mov, k)
            _, n_u, _, _ = TM.multi_program(par, mov, links)
            for pose in (True, False):
                M = (6 if pose else 3) * len(links)
                branch = "task" if M <= n_u else "joint"
                ikm.setdefault((TM.ikm_choice(par, mov, links, pose)[0], pose, branch), (name, links))
                osd.setdefault((TM.osd_choice(par, mov, links, pose)[0], pose, branch), (name, links))
    return ikm, osd


IKM_CASES, OSD_CASES = _solver_cases()
IK_CASES = {64: "D_fixed", 32: "C_dfs"}
# (family, rnea_fold): TC = 128 (n = 1), lowered tiles (14 / 8, 9 / 4 and 4 / 2 unfolded), TC = 1 with TC n and TC n^2
# odd (bulk and cooperative copies alternate between tiles)
DERIV_CASES = [("G_one_joint", 1), ("E_unfoldable", 1), ("D_fixed", 1), ("D_fixed", 0), ("B_dfs_fixed_palm", 1),
               ("B_dfs_fixed_palm", 0)]


def ids(cases):
    return [f"T{t}-{'pose' if p else 'pos'}-{b}" for (t, p, b) in cases]


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("solver_geometry"))


def family(name, model_dir):
    if name not in _MODELS:
        path = S.build(FAM[name], model_dir)
        r32 = O.load_robot(path, torch.float32)
        _MODELS[name] = (drm.DifferentiableRobotModel(path, name, device=DEV), r32, r32.to(torch.float64),
                         O.link_table(r32).float().to(DEV).contiguous())
    return _MODELS[name]


def batches(T):
    return sorted({1, max(1, T - 1), T, T + 1, 3 * T + 3})


def checked_rows(T):
    """Rows the oracle checks in the LARGE batch: the first 3T + 4 (every small batch), a spread, the tail."""
    return torch.unique(torch.cat([torch.arange(min(3 * T + 4, LARGE)), torch.arange(3 * T + 4, LARGE - 3, 97),
                                   torch.arange(LARGE - 3, LARGE)]))


def shifted(t):
    """The same values 4 bytes off 16-byte alignment (None stays None)."""
    if t is None:
        return None
    buf = torch.empty(t.numel() + 1, device=DEV, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def per_config_error(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, f"shape {tuple(got.shape)} vs {tuple(want.shape)}"
    B = want.shape[0]
    scale = want.reshape(B, -1).abs().amax(1)
    err = (got - want).reshape(B, -1).abs().amax(1)
    return float(torch.where(scale > 0, err / scale.clamp_min(1e-300), err).max())


def check(what, got, want64, want32, floor=2e-5):
    e32 = per_config_error(want32, want64)
    err = per_config_error(got, want64)
    bound = max(8 * e32, floor)
    print(f"ERR {what}: {err:.2e} (bound {bound:.2e}, ratio {err / bound:.3f})")
    assert np.isfinite(err) and err <= bound, f"{what}: per-configuration error {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"


def same_rows(what, small, big):
    for a, b in zip(small, big):
        if a is not None:
            assert torch.equal(a, b[:a.shape[0]]), f"{what}: rows differ from the {LARGE}-row batch"


def inputs(r32, B, seed):
    q, qd, qdd = O.sample_inputs(r32.to(torch.float64), B, seed=seed, dtype=torch.float32)
    f = torch.randn(B, r32.n_dofs, generator=torch.Generator().manual_seed(seed))
    return q, qd, qdd, f


# ------------------------------------------------------------------------------------------------
# dynamics derivatives
# ------------------------------------------------------------------------------------------------
def deriv_call(topo, table, x, flags, fd, wants=(True, True, True), misaligned=False):
    """Through the C ABI; `misaligned`: every input and output 4 bytes off 16-byte alignment."""
    q, qd, x3 = x
    B, n = q.shape
    outs = [torch.empty(B, n, n, device=DEV) if w else None for w in wants[:3 if fd else 2]]
    if misaligned:
        q, qd, x3 = (shifted(t) for t in (q, qd, x3))
        outs = [shifted(o) for o in outs]
    if fd:
        rc = engine.lib().drmb200_forward_dynamics_derivatives(ctypes.byref(topo), ptr(table), ptr(q), ptr(qd), ptr(x3), B, flags,
                                                               *[ptr(o) for o in outs], stream())
    else:
        rc = engine.lib().drmb200_inverse_dynamics_derivatives(ctypes.byref(topo), ptr(table), ptr(q), ptr(qd), ptr(x3), B, flags,
                                                               *[ptr(o) for o in outs], stream())
    assert rc == 0, engine.lib().drmb200_last_error()
    return outs


@pytest.mark.parametrize("fd", [False, True], ids=["ID", "FD"])
@pytest.mark.parametrize("name,fold", DERIV_CASES)
def test_derivatives_at_every_tile(name, fold, fd, model_dir):
    m, r32, r64, table = family(name, model_dir)
    par, mov = FAM[name].doc()
    tile, need = TM.deriv_choice(*TM.deriv_program(par, mov, bool(fold)), fd)
    if tile is None:
        pytest.skip(f"refused ({need} B): pinned in test_dynamics_derivatives_gpu.py")
    old = engine.get_option("rnea_fold")
    engine.set_option("rnea_fold", fold)
    try:
        topo = m._topology
        q, qd, qdd, f = inputs(r32, LARGE, seed=21)
        x = [t.to(DEV) for t in (q, qd, f if fd else qdd)]
        rows = checked_rows(tile)
        sub = [t[rows] for t in (q, qd, f if fd else qdd)]
        fn = D.forward_dynamics_derivatives if fd else D.inverse_dynamics_derivatives
        for grav, damp in FLAGS:
            flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
            big = deriv_call(topo, table, x, flags, fd)
            w64 = fn(r64, *(t.double() for t in sub), grav, damp)
            w32 = fn(r32, *sub, grav, damp)
            for k in range(len(big)):
                check(f"{name} fold={fold} {'FD' if fd else 'ID'} TC={tile} g{grav:d}d{damp:d} out{k}", big[k].cpu()[rows], w64[k],
                      w32[k])
            for B in batches(tile):
                same_rows(f"{name} B={B}", deriv_call(topo, table, [t[:B] for t in x], flags, fd), big)
            same_rows(f"{name} misaligned", deriv_call(topo, table, x, flags, fd, misaligned=True), big)
        # every subset of the outputs: the same matrices, bit for bit; nothing wanted: no launch
        n_out = 3 if fd else 2
        for mask in range(1 << n_out):
            wants = [bool(mask >> k & 1) for k in range(n_out)] + [False] * (3 - n_out)
            before = engine.launch_count()
            part = deriv_call(topo, table, x, flags, fd, wants, misaligned=True)
            torch.cuda.synchronize()
            assert engine.launch_count() == before + (1 if mask else 0)
            for k in range(n_out):
                assert (part[k] is None) != wants[k]
                if wants[k]:
                    assert torch.equal(part[k], big[k]), (mask, k)
    finally:
        engine.set_option("rnea_fold", old)


# ------------------------------------------------------------------------------------------------
# operational-space dynamics
# ------------------------------------------------------------------------------------------------
OSD_NAMES = ("inv_inertia", "acceleration", "velocity", "bias_acceleration")


def osd_call(topo, links, table, x, flags, pos, wants=(True,) * 4, misaligned=False):
    q, qd, f = x
    B = q.shape[0]
    M = (3 if pos else 6) * len(links)
    outs = [torch.empty((B, M, M) if k == 0 else (B, M), device=DEV) if w else None for k, w in enumerate(wants)]
    if misaligned:
        q, qd, f = (shifted(t) for t in (q, qd, f))
        outs = [shifted(o) for o in outs]
    idx = (ctypes.c_int32 * len(links))(*links)
    rc = engine.lib().drmb200_operational_space_dynamics(ctypes.byref(topo), len(links), idx, ptr(table), ptr(q), ptr(qd), ptr(f), B,
                                                         flags, int(pos), *[ptr(o) for o in outs], stream())
    assert rc == 0, engine.lib().drmb200_last_error()
    return outs


@pytest.mark.parametrize("key", sorted(OSD_CASES, key=str), ids=ids(sorted(OSD_CASES, key=str)))
def test_operational_space_at_every_tile(key, model_dir):
    import test_operational_space_gpu as OSDT
    tile, pose, branch = key
    name, links = OSD_CASES[key]
    m, r32, r64, table = family(name, model_dir)
    par, mov = FAM[name].doc()
    assert TM.osd_choice(par, mov, links, pose)[0] == tile
    topo = m._topology
    q, qd, _, f = inputs(r32, LARGE, seed=22)
    x = [t.to(DEV) for t in (q, qd, f)]
    rows = checked_rows(tile)
    sub = [t[rows] for t in (q, qd, f)]
    names = [r32.names[l] for l in links]
    o64 = OSDT.OraclePieces(r64, *(t.double() for t in sub), names)
    o32 = OSDT.OraclePieces(r32, *sub, names)
    for grav, damp in FLAGS:
        flags = (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)
        big = osd_call(topo, links, table, x, flags, not pose)
        w64, w32 = o64.outputs(grav, damp, None, not pose), o32.outputs(grav, damp, None, not pose)
        for k, nm in enumerate(OSD_NAMES):
            check(f"{name} {len(links)} links T={tile} {branch} pose={pose} g{grav:d}d{damp:d} {nm}", big[k].cpu()[rows], w64[k], w32[k],
                  1e-4 if nm == "acceleration" else 2e-5)
        for B in batches(tile):
            same_rows(f"{name} B={B}", osd_call(topo, links, table, [t[:B] for t in x], flags, not pose), big)
        same_rows(f"{name} misaligned", osd_call(topo, links, table, x, flags, not pose, misaligned=True), big)
    for mask in range(16):
        wants = [bool(mask >> k & 1) for k in range(4)]
        before = engine.launch_count()
        part = osd_call(topo, links, table, x, flags, not pose, wants, misaligned=True)
        torch.cuda.synchronize()
        assert engine.launch_count() == before + (1 if mask else 0)
        for k in range(4):
            assert (part[k] is None) != wants[k]
            if wants[k]:
                assert torch.equal(part[k], big[k]), (mask, k)


# ------------------------------------------------------------------------------------------------
# inverse kinematics: one step against the fp64 oracle, per-row damping, no joint limits
# ------------------------------------------------------------------------------------------------
def ik_call(topo, links, table, q0, tpos, tquat, damp, misaligned=False, multi=True, max_iters=1):
    B, n = q0.shape
    E = len(links)
    outs = [torch.zeros(B, n, device=DEV), torch.zeros((E, B) if multi else (B,), device=DEV),
            torch.zeros((E, B) if multi else (B,), device=DEV), torch.zeros(B, device=DEV, dtype=torch.uint8),
            torch.zeros(B, device=DEV)]
    ins = [q0, tpos, tquat, None, None, damp]
    if misaligned:
        ins, outs = [shifted(t) for t in ins], [shifted(t) for t in outs]
    args = [ptr(t) for t in ins] + [B, max_iters, ctypes.c_float(IK.DAMPING_INIT), ctypes.c_float(1e-4), ctypes.c_float(1e-3)]
    if multi:
        idx = (ctypes.c_int32 * E)(*links)
        rc = engine.lib().drmb200_inverse_kinematics_multi(ctypes.byref(topo), E, idx, ptr(table), *args, *[ptr(t) for t in outs],
                                                           stream())
    else:
        rc = engine.lib().drmb200_inverse_kinematics(ctypes.byref(topo), links[0], ptr(table), *args, *[ptr(t) for t in outs],
                                                     stream())
    assert rc == 0, engine.lib().drmb200_last_error()
    return outs


def compare_ik_step(what, got_q, got_damp, w64, w32, rows):
    """One step against the fp64 oracle, as compare_one_step in test_inverse_kinematics_multi_gpu.py."""
    keep = w64["margin"] >= 1e-3
    assert int((~keep).sum()) <= max(3, len(rows) // 100), f"{what}: {int((~keep).sum())} rows within the accept margin"
    assert torch.allclose(got_damp.cpu()[rows][keep].double(), w64["damping"][keep], rtol=1e-6, atol=0), f"{what}: damping differs"
    q = got_q.cpu()[rows].double()[keep]
    e32 = float((w32["q"].double()[keep] - w64["q"][keep]).abs().max())
    err = float((q - w64["q"][keep]).abs().max())
    bound = max(8 * e32, 2e-5)
    print(f"ERR {what}: q {err:.2e} (bound {bound:.2e}, ratio {err / bound:.3f})")
    assert np.isfinite(err) and err <= bound, f"{what}: q error {err:.3e} > {bound:.3e}"


def run_ik_case(what, m, r32, r64, table, links, pose, tile, multi):
    topo = m._topology
    names = [r32.names[l] for l in links]
    if multi:
        q0, tpos, tquat = IKM.problem(r64, names, LARGE, seed=23)
    else:
        q0, tpos, tquat = IK.problem(r64, names[0], LARGE, seed=23)
    tquat = tquat if pose else None
    damp = (10.0 ** (-3 * torch.rand(LARGE, generator=torch.Generator().manual_seed(24)) - 1)).float()
    dev = [None if t is None else t.to(DEV).contiguous() for t in (q0, tpos, tquat, damp)]
    big = ik_call(topo, links, table, *dev, multi=multi)
    rows = checked_rows(tile)
    sel = (lambda t: None if t is None else t[:, rows]) if multi else (lambda t: None if t is None else t[rows])
    solve = (lambda r, q, tp, tq, d: IKM.solve(r, q, names, tp, tq, None, None, d, max_iters=1)) if multi else \
        (lambda r, q, tp, tq, d: IK.solve(r, q, names[0], tp, tq, None, None, d, max_iters=1))
    w64 = solve(r64, q0[rows].double(), sel(tpos), sel(tquat), damp[rows].double())
    w32 = solve(r32, q0[rows], sel(tpos), sel(tquat), damp[rows])
    compare_ik_step(what, big[0], big[4], w64, w32, rows)
    for B in batches(tile):
        cut = (lambda t: None if t is None else t[:, :B].contiguous()) if multi else (lambda t: None if t is None else t[:B])
        small = ik_call(topo, links, table, dev[0][:B], cut(dev[1]), cut(dev[2]), dev[3][:B], multi=multi)
        for k, (a, b) in enumerate(zip(small, big)):
            assert torch.equal(a, b[:, :B] if (multi and k in (1, 2)) else b[:B]), f"{what} B={B} output {k}"
    for a, b in zip(ik_call(topo, links, table, *dev, misaligned=True, multi=multi), big):
        assert torch.equal(a, b), f"{what} misaligned"


@pytest.mark.parametrize("key", sorted(IKM_CASES, key=str), ids=ids(sorted(IKM_CASES, key=str)))
def test_multi_link_ik_at_every_tile(key, model_dir):
    tile, pose, branch = key
    name, links = IKM_CASES[key]
    m, r32, r64, table = family(name, model_dir)
    par, mov = FAM[name].doc()
    assert TM.ikm_choice(par, mov, links, pose)[0] == tile
    run_ik_case(f"{name} {len(links)} links T={tile} {branch} pose={pose}", m, r32, r64, table, links, pose, tile, True)


@pytest.mark.parametrize("pose", [True, False], ids=["pose", "pos"])
@pytest.mark.parametrize("tile", sorted(IK_CASES))
def test_single_link_ik_at_every_tile(tile, pose, model_dir):
    name = IK_CASES[tile]
    m, r32, r64, table = family(name, model_dir)
    par, mov = FAM[name].doc()
    link = deepest(par, mov, 1)
    assert TM.ik_choice(sum(mov[1:]), TM.path_len(par, link[0]))[0] == tile
    run_ik_case(f"{name} ik T={tile} pose={pose}", m, r32, r64, table, link, pose, tile, False)


def test_every_reachable_rung_has_a_case():
    for T in TM.LADDER[:-1]:
        for pose in (True, False):
            if pose or T > 2:
                assert any(k[:2] == (T, pose) for k in OSD_CASES), ("osd", T, pose)
                assert any(k[:2] == (T, pose) for k in IKM_CASES), ("ikm", T, pose)
    for table in (IKM_CASES, OSD_CASES):
        assert {k[2] for k in table} == {"task", "joint"}


def test_static_shared_memory_is_what_the_mirrors_add():
    """cudaFuncGetAttributes(...).sharedSizeBytes of every instantiation, through the library's own CUDA runtime."""
    lib = engine.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    symbols = {"deriv": ["_ZN3drm27dynamics_derivatives_kernelILb0EEEvNS_11TreeProgramENS_11FoldProgramENS_9DerivArgsE",
                         "_ZN3drm27dynamics_derivatives_kernelILb1EEEvNS_11TreeProgramENS_11FoldProgramENS_9DerivArgsE"],
               "ik": [f"_ZN3drm25inverse_kinematics_kernelILb{b}EEEvNS_11PathProgramENS_6IkArgsE" for b in (0, 1)],
               "ikm": [f"_ZN3drm31inverse_kinematics_multi_kernelILb{b}EEEvNS_12UnionProgramENS_7IkmArgsE" for b in (0, 1)],
               "osd": [f"_ZN3drm24operational_space_kernelILi{t}EEEvNS_11TreeProgramENS_12UnionProgramENS_7OsdArgsE"
                       for t in TM.LADDER]}
    for kernel, syms in symbols.items():
        for sym in syms:
            attr = (ctypes.c_size_t * 64)()
            rc = cudart.cudaFuncGetAttributes(attr, ctypes.cast(getattr(lib, sym), ctypes.c_void_p))
            assert rc == 0, (sym, rc)
            assert attr[0] == TM.STATIC_SMEM[kernel], (sym, attr[0])


# ------------------------------------------------------------------------------------------------
# the slow sin / cos path (|q| > 105 615) in every kernel
# ------------------------------------------------------------------------------------------------
def large_angle_rows(r32, B, seed):
    """Sampled inputs whose q mixes, in every warp, ordinary angles with ones just below and just above the fast path's
    limit and at 1e6 and 3e7 rad."""
    q, qd, qdd, f = inputs(r32, B, seed)
    lim = 105615.0
    vals = torch.tensor([np.nextafter(np.float32(lim), np.float32(0)), lim, np.nextafter(np.float32(lim), np.float32(1e9)),
                         lim + 3.0, -lim - 0.5, 1e6, -1e6 - 0.25, 3e7, -3e7], dtype=torch.float32)
    g = torch.Generator().manual_seed(seed)
    pick = torch.rand(q.shape, generator=g) < 0.5
    q = torch.where(pick, vals[torch.randint(len(vals), q.shape, generator=g)] + 0 * q, q)
    return q, qd, qdd, f


def test_large_angles_in_every_forward_kernel(model_dir):
    import test_operational_space_gpu as OSDT
    name = "D_fixed"
    m, r32, r64, table = family(name, model_dir)
    topo = m._topology
    B = 256
    q, qd, qdd, f = large_angle_rows(r32, B, seed=30)
    assert bool((q.abs() > 105615).any()) and bool((q.abs() < 10).any())
    dq, dqd, dqdd, df = (t.to(DEV) for t in (q, qd, qdd, f))
    q64 = q.double()
    leaves = [r32.names[l] for l in deepest(*FAM[name].doc(), 3)]
    # FK + Jacobian, single and multi-link
    for link in leaves:
        p, _, jl, ja = m.compute_fk_and_jacobian(dq, link)
        check(f"large-angle fk pos {link}", p, O.forward_kinematics(r64, q64, link)[0], O.forward_kinematics(r32, q, link)[0])
        check(f"large-angle fk jac {link}", torch.cat([jl, ja], 1), torch.cat(O.jacobian(r64, q64, link), 1),
              torch.cat(O.jacobian(r32, q, link), 1))
    multi = m.compute_fk_and_jacobian_multi(dq, leaves)
    for link in leaves:
        check(f"large-angle fk_multi {link}", multi[link][2], O.jacobian(r64, q64, link)[0], O.jacobian(r32, q, link)[0])
    # kinematic state of every link: poses [B, N, 12] and body velocities [B, N, 6]
    poses, _, vels = engine.kinematic_state_raw(topo, table, dq, dqd)
    kin = []
    for r, qq in ((r64, q64), (r32, q)):
        R, p, w, v, _ = O.kinematic_state(r, qq, qd.to(qq.dtype))
        kin.append((torch.stack([torch.cat([Ri.reshape(-1, 9), pi], 1) for Ri, pi in zip(R, p)], 1),
                    torch.stack([torch.cat([wi, vi], 1) for wi, vi in zip(w, v)], 1)))
    check("large-angle kinematic_state poses", poses.permute(2, 0, 1), kin[0][0], kin[1][0])
    check("large-angle kinematic_state vels", vels.permute(2, 0, 1), kin[0][1], kin[1][1])
    # one rollout step (later steps move q by dt qd, which fp32 rounds to its spacing at |q|: up to 2 rad at 3e7, so
    # they would compare the rounding of q, not the kernel)
    for grav, damp in FLAGS[:2]:
        got = m.compute_forward_dynamics_rollout(dq, dqd, df[None], 0.01, grav, damp)
        w64 = RO.forward_dynamics_rollout(r64, q64, qd.double(), f.double()[None], 0.01, grav, damp)
        w32 = RO.forward_dynamics_rollout(r32, q, qd, f[None], 0.01, grav, damp)
        for k, nm in enumerate(("q", "qd", "qdd")):
            check(f"large-angle rollout g{grav:d}d{damp:d} {nm}", got[k][0], w64[k][0], w32[k][0])
    # inverse dynamics, forward dynamics, mass matrix
    for grav, damp in FLAGS[:2]:
        check("large-angle rnea", m.compute_inverse_dynamics(dq, dqd, dqdd, grav, damp),
              O.inverse_dynamics(r64, q64, qd.double(), qdd.double(), grav, damp), O.inverse_dynamics(r32, q, qd, qdd, grav, damp))
        check("large-angle aba", m.compute_forward_dynamics(dq, dqd, df, grav, damp),
              O.forward_dynamics(r64, q64, qd.double(), f.double(), grav, damp), O.forward_dynamics(r32, q, qd, f, grav, damp))
    H = m.compute_lagrangian_inertia_matrix(dq)
    eye = torch.eye(r32.n_dofs)

    def mass(r, qq):
        z = torch.zeros_like(qq)
        return torch.stack([O.inverse_dynamics(r, qq, z, eye[j].to(qq.dtype).expand_as(qq), False, False)
                            for j in range(r32.n_dofs)], dim=2)
    check("large-angle mass matrix", H, mass(r64, q64), mass(r32, q))
    # both derivative kernels
    got = engine.inverse_dynamics_derivatives_raw(topo, table, dq, dqd, dqdd, 3)
    w64, w32 = D.inverse_dynamics_derivatives(r64, q64, qd.double(), qdd.double(), True, True), \
        D.inverse_dynamics_derivatives(r32, q, qd, qdd, True, True)
    for k in range(2):
        check(f"large-angle ID derivatives {k}", got[k], w64[k], w32[k])
    got = engine.forward_dynamics_derivatives_raw(topo, table, dq, dqd, df, 3)
    w64, w32 = D.forward_dynamics_derivatives(r64, q64, qd.double(), f.double(), True, True), \
        D.forward_dynamics_derivatives(r32, q, qd, f, True, True)
    for k in range(3):
        check(f"large-angle FD derivatives {k}", got[k], w64[k], w32[k])
    # operational-space dynamics, pose mode
    idx = deepest(*FAM[name].doc(), 3)
    got = engine.operational_space_dynamics_raw(topo, idx, table, dq, dqd, df, engine.GRAVITY)
    o64, o32 = OSDT.OraclePieces(r64, q64, qd.double(), f.double(), leaves), OSDT.OraclePieces(r32, q, qd, f, leaves)
    w64, w32 = o64.outputs(True, False), o32.outputs(True, False)
    for k, nm in enumerate(OSD_NAMES):
        check(f"large-angle osd {nm}", got[k], w64[k], w32[k], 1e-4 if nm == "acceleration" else 2e-5)
    # adjoints of FK, RNEA and ABA against oracle autograd
    G = torch.randn(B, 3, generator=torch.Generator().manual_seed(31))
    Gt = torch.randn(B, r32.n_dofs, generator=torch.Generator().manual_seed(32))

    def loss(fk, rnea, aba, qq, dt):
        return (fk(qq) * G.to(dt)).sum() + (rnea(qq) * Gt.to(dt)).sum() + (aba(qq) * Gt.to(dt)).sum()
    qa = dq.clone().requires_grad_(True)
    loss(lambda a: m.compute_forward_kinematics(a, leaves[0])[0], lambda a: m.compute_inverse_dynamics(a, dqd, dqdd, True, True),
         lambda a: m.compute_forward_dynamics(a, dqd, df, True, True), qa, DEV).backward()
    want = []
    for r, qq in ((r64, q64), (r32, q)):
        qo = qq.clone().requires_grad_(True)
        dt = qq.dtype
        l = loss(lambda a: O.forward_kinematics(r, a, leaves[0])[0],
                 lambda a: O.inverse_dynamics(r, a, qd.to(dt), qdd.to(dt), True, True),
                 lambda a: O.forward_dynamics(r, a, qd.to(dt), f.to(dt), True, True), qo, dt)
        want.append(torch.autograd.grad(l, qo)[0])
    check("large-angle adjoints dq", qa.grad, want[0], want[1])


def ulp32(x):
    """The spacing of fp32 numbers at |x| (float64 tensor of the same shape)."""
    a = x.abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


@pytest.mark.parametrize("multi", [False, True], ids=["ik", "ik_multi"])
def test_large_angles_in_one_ik_step(multi, model_dir):
    """The IK kernels' walk at large angles, where the multi-link kernel's only stack frame (around the slow sin / cos
    call) is live.  Per row:
      * max_iters = 0 reports the errors at the start: pos_err / rot_err against the oracle's evaluation at q0;
      * one step: dq = q - q0 of every element against the fp64 oracle's, on rows where the fp64 and fp32 oracles take the
        same accept decision outside the 1e-3 margin.  q0 + dq is rounded to fp32's spacing at |q0| (2 rad at 3e7), which
        decides the trial point; so an element may differ by that spacing plus max(8 x the fp32 oracle's largest error on
        the compared rows once its own rounding is removed, 2e-5) rad."""
    name = "D_fixed"
    m, r32, r64, table = family(name, model_dir)
    links = deepest(*FAM[name].doc(), 3 if multi else 1)
    names = [r32.names[l] for l in links]
    B = 256
    q0, tpos, tquat = IKM.problem(r64, names, B, seed=33) if multi else IK.problem(r64, names[0], B, seed=33)
    q0 = large_angle_rows(r32, B, seed=34)[0]
    path = IKM.union_dofs(r64, names)
    big = q0[:, path].abs() > 105615
    assert bool(big.any(1).float().mean() > 0.5) and bool((q0[:, path].abs() < 10).any())
    damp = torch.full((B,), IK.DAMPING_INIT)
    dev = [t.to(DEV).contiguous() for t in (q0, tpos, tquat, damp)]
    what = f"large-angle {'multi-link ' if multi else ''}ik"
    # errors at the start: the walk and its sin / cos alone
    start = ik_call(m._topology, links, table, *dev, multi=multi, max_iters=0)
    ev = (lambda r, q: IKM.evaluate(r, q, names, tpos.to(q.dtype), tquat.to(q.dtype))[3:]) if multi else \
        (lambda r, q: [t[None] for t in IK.evaluate(r, q, names[0], tpos.to(q.dtype), tquat.to(q.dtype))[3:]])
    s64, s32 = ev(r64, q0.double()), ev(r32, q0)
    for k, nm in ((1, "pos_err"), (2, "rot_err")):
        got = start[k] if multi else start[k][None]
        check(f"{what} {nm} at q0", got.t(), s64[k - 1].t(), s32[k - 1].t())
    # one step
    out = ik_call(m._topology, links, table, *dev, multi=multi)
    solve = IKM.solve if multi else IK.solve
    tgt = names if multi else names[0]
    w64 = solve(r64, q0.double(), tgt, tpos, tquat, None, None, damp.double(), max_iters=1)
    w32 = solve(r32, q0, tgt, tpos, tquat, None, None, damp, max_iters=1)
    keep = (w64["accepted"] == w32["accepted"]) & (w64["margin"] >= 1e-3) & (w32["margin"] >= 1e-3)
    acc = keep & w64["accepted"]
    print(f"{what}: {int(keep.sum())} of {B} rows compared, {int(acc.sum())} of them accepted, "
          f"{int((acc & big.any(1)).sum())} accepted with a joint beyond the fast range")
    assert int(keep.sum()) >= 3 * B // 4 and int((acc & big.any(1)).sum()) >= B // 8
    q = out[0].cpu()
    assert torch.equal(out[4].cpu()[keep].double(), w64["damping"][keep]), f"{what}: accept decisions differ"
    r = ulp32(torch.maximum(torch.maximum(q0.abs(), q.abs()), w32["q"].abs()).double())
    d64 = w64["q"] - q0.double()
    d32 = (w32["q"].double() - q0.double() - d64).abs()
    e32 = float((d32 - r).clamp_min(0)[keep].max())
    bound = max(8 * e32, 2e-5) + r
    err = (q.double() - q0.double() - d64).abs()
    ratio = float((err / bound)[keep].max())
    small = err[keep][q0[keep].abs() < 10]
    print(f"ERR {what} step: max per-element error / bound {ratio:.3f} (fp32 oracle {e32:.2e} rad); elements with |q0| < 10: max error {float(small.max()):.2e} rad")
    assert ratio <= 1.0, f"{what}: step error {ratio:.2f} x the per-element bound"
