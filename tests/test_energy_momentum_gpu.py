"""GPU: energy, generalized momentum and centre of mass (compute_energy_and_momentum / drmb200_energy_momentum,
csrc/energy_momentum.cu) against the fp64 oracle (tests/energy_oracle.py), the reference's per-body state, and the other
kernels (mass matrix, kinematic state, RNEA gravity torque, multi-link Jacobians); on every shipped robot, the synthetic
topology families and every tile the host rule can choose.

Errors are per configuration, relative to that configuration's largest entry of the output; the bound is
max(8 x the fp32 oracle's error on the same rows, 2e-5), as in test_dynamics_regressor_gpu.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedTensor
from conftest import GOLDEN_DIR, URDFS, urdf_path
import derivatives_oracle as D
import energy_oracle as E
import synthetic_robots as S
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL, LARGE = 131, 4099
LARGE_ROWS = torch.cat([torch.arange(SMALL, LARGE - 3, 97), torch.arange(LARGE - 3, LARGE)])
NAMES = ("kinetic", "potential", "momentum", "com", "com_velocity", "com_jacobian")
EINVAL, ELIMIT = -1, -3

# ------------------------------------------------------------------------------------------------
# mirror of the host tile rule (csrc/energy_momentum.cu: EmSmemLayout, energy_momentum_tile)
# ------------------------------------------------------------------------------------------------
KERNEL_SYMBOL = "_ZN3drm22energy_momentum_kernelENS_11TreeProgramENS_6EmArgsE"
STATIC_SMEM = 0                   # the kernel declares none (pinned by test_static_shared_memory_matches_the_mirror)
TWO_CTAS, CTA_MAX = 113 * 1024, 227 * 1024


def layout_bytes(T, n, N, slots):
    up4 = lambda x: (x + 3) & ~3  # noqa: E731
    return 4 * (2 * up4(T * n) + N * 28 + slots * 18 * T + N * 16 * T + T * (8 + 4 * n))


def tile_choice(n, N, slots):
    """(T, dynamic bytes), or (None, bytes needed) when even one row per CTA exceeds 227 KB."""
    T = 64
    while T > 1 and layout_bytes(T, n, N, slots) + STATIC_SMEM > TWO_CTAS:
        T //= 2
    b = layout_bytes(T, n, N, slots)
    return (T, b) if b + STATIC_SMEM <= CTA_MAX else (None, b + STATIC_SMEM)


def tile_of(robot):
    return tile_choice(robot.n_dofs, len(robot.names), S.live_slots(robot.parent))[0]


# ------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------
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
    print(f"ERR {what}: {err:.2e} (bound {bound:.2e})")
    assert np.isfinite(err) and err <= bound, f"{what}: per-configuration error {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"


def check_all(what, got, r64, r32, q, qd, rows=None, floor=2e-5):
    """Every output of one kernel call (rows: the checked subset) against the fp64 and fp32 oracles."""
    if rows is not None:
        got = [None if g is None else g.cpu()[rows] for g in got]
        q, qd = q[rows], qd[rows]
    w64 = E.energy_momentum(r64, q.double(), qd.double())
    w32 = E.energy_momentum(r32, q, qd)
    for name, g, a, b in zip(NAMES, got, w64, w32):
        check(f"{what} {name}", g, a, b, floor)


def robots(path, nonsym):
    r32 = O.load_robot(path, torch.float32)
    if nonsym:
        r32 = D.perturbed(r32)
    return r32, r32.to(torch.float64), O.link_table(r32).float().to(DEV).contiguous()


def inputs(robot, B, seed=3):
    q, qd, _ = O.sample_inputs(robot.to(torch.float64), B, seed=seed, dtype=torch.float32)
    return q, qd


def model_of(stem):
    return drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def raw_call(topo, table, q, qd, B, outs):
    return engine.lib().drmb200_energy_momentum(ctypes.byref(topo), ptr(table), ptr(q), ptr(qd), B, *[ptr(o) for o in outs],
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def empty_outs(B, n):
    return [torch.empty(s, device=DEV) for s in ((B,), (B,), (B, n), (B, 3), (B, 3), (B, 3, n))]


def shifted(t):
    """The same values 4 bytes off 16-byte alignment."""
    buf = torch.empty(t.numel() + 1, device=DEV, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def assert_equal(a, b, what=""):
    for name, x, y in zip(NAMES, a, b):
        assert (x is None) == (y is None), (what, name)
        if x is not None:
            assert torch.equal(x, y), (what, name)


# ------------------------------------------------------------------------------------------------
# shipped robots against the fp64 oracle and the reference
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_shipped_robots_match_oracle(stem, nonsym):
    r32, r64, table = robots(urdf_path(stem), nonsym)
    topo = model_of(stem)._topology
    for B in (SMALL, LARGE):
        q, qd = inputs(r32, B)
        got = engine.energy_momentum_raw(topo, table, q.to(DEV), qd.to(DEV))
        check_all(f"{stem} B={B}", got, r64, r32, q, qd, None if B == SMALL else LARGE_ROWS)


GOLDEN = ["iiwa7", "panda_no_gripper", "fetch_arm_no_gripper", "2link_robot", "allegro_hand_description_left_small_damping"]


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".energy.npz"), allow_pickle=False)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"])
        inertia[0] = r32.inertia[0]
        r32.inertia = inertia
    r64 = r32.to(torch.float64)
    table = O.link_table(r32).float().to(DEV).contiguous()
    q, qd = torch.tensor(g["q"]), torch.tensor(g["qd"])
    pre = "" if tag == "sym" else "nonsym."
    got = engine.energy_momentum_raw(model_of(stem)._topology, table, q.to(DEV), qd.to(DEV))
    w64 = E.energy_momentum(r64, q.double(), qd.double())
    # the goldens are the reference's fp32 evaluation: the bound is the fp64 oracle's distance from them
    for name, k, o in zip(NAMES, got, w64):
        check(f"{stem} {pre}{name}", k.cpu(), torch.tensor(g[pre + name]), o.float(), floor=2e-4)


# ------------------------------------------------------------------------------------------------
# identities with the other kernels
# ------------------------------------------------------------------------------------------------
IDENTITY = ["iiwa7", "panda", "trifinger_edu", "allegro_hand_description_left", "iiwa7_allegro"]


def rel(got, want, scale):
    """Largest per-configuration error relative to a per-configuration scale [B]."""
    B = got.shape[0]
    return float(((got - want).reshape(B, -1).abs().amax(1) / scale.clamp_min(1e-30)).max())


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", IDENTITY)
def test_identities_with_the_other_kernels(stem, nonsym):
    r32, _, table = robots(urdf_path(stem), nonsym)
    m = model_of(stem)
    topo, n, N = m._topology, r32.n_dofs, len(r32.names)
    q, qd = (t.to(DEV) for t in inputs(r32, 257, seed=8))
    kin, pot, mom, com, comv, jcom = (t.double() for t in engine.energy_momentum_raw(topo, table, q, qd))
    t = table.double()
    mass, mc, Io = t[:, 24], t[:, 21:24], t[:, 12:21].reshape(N, 3, 3)
    M = float(mass.sum())

    # momentum = H qd with the mass-matrix kernel
    H = engine.mass_matrix_raw(topo, table, q).double()
    want = (H @ qd.double().unsqueeze(2)).squeeze(2)
    assert rel(mom, want, (H.abs() @ qd.double().abs().unsqueeze(2)).squeeze(2).amax(1)) < 1e-5
    # kinetic = 1/2 qd . momentum
    assert rel(kin, 0.5 * (qd.double() * mom).sum(1), 0.5 * (qd.double().abs() * mom.abs()).sum(1)) < 1e-5

    # com, potential, com velocity and kinetic energy from kinematic_state's poses and velocities plus the table
    poses, _, vels = engine.kinematic_state_raw(topo, table, q, qd)
    R = poses[:, :9].double().reshape(N, 3, 3, -1).permute(3, 0, 1, 2)         # [B, N, 3, 3]
    p = poses[:, 9:12].double().permute(2, 0, 1)                              # [B, N, 3]
    w, v = vels[:, :3].double().permute(2, 0, 1), vels[:, 3:].double().permute(2, 0, 1)
    Rmc = (R @ mc.unsqueeze(2)).squeeze(-1)
    h = mass[:, None] * p + Rmc
    hscale = (mass[:, None] * p.abs() + Rmc.abs()).sum(1).amax(1)
    assert rel(com, h.sum(1) / M, hscale / M) < 1e-5
    assert rel(pot, 9.81 * h.sum(1)[:, 2], 9.81 * hscale) < 1e-5
    f_lin = mass[:, None] * v - torch.cross(mc.expand_as(w), w, dim=-1)
    f_ang = (Io @ w.unsqueeze(-1)).squeeze(-1) + torch.cross(mc.expand_as(v), v, dim=-1)
    L = (R @ f_lin.unsqueeze(-1)).squeeze(-1)
    assert rel(comv, L.sum(1) / M, L.abs().sum(1).amax(1) / M) < 1e-5
    k2 = (v * f_lin).sum(-1) + (w * f_ang).sum(-1)
    assert rel(kin, 0.5 * k2.sum(1), 0.5 * k2.abs().sum(1)) < 1e-5

    # 9.81 M J_com[2] is the RNEA kernel's gravity torque
    z = torch.zeros_like(q)
    tau_g = engine.inverse_dynamics_raw(topo, table, q, z, z, engine.GRAVITY).double()
    assert rel(9.81 * M * jcom[:, 2], tau_g, tau_g.abs().amax(1)) < 1e-5

    # J_com from the multi-link Jacobians of every massive link: sum_i m_i J_lin,i + J_ang,i x (R_i mc_i), over M
    links = [l for l in range(1, N) if float(mass[l]) != 0 or bool((mc[l] != 0).any())]
    want = torch.zeros_like(jcom)
    scale = torch.zeros(q.shape[0], dtype=torch.float64, device=DEV)
    for g in range(0, len(links), 8):
        group = links[g:g + 8]
        _, _, jl, ja = engine.fk_jacobian_multi_raw(topo, group, table, q, want_pos=False, want_quat=False)
        for e, l in enumerate(group):
            term = mass[l] * jl[e].double() + torch.cross(ja[e].double(), Rmc[:, l, :, None].expand_as(ja[e]), dim=1)
            want += term / M
            scale = torch.maximum(scale, term.abs().amax((1, 2)) / M)
    assert rel(jcom, want, scale) < 1e-5


# ------------------------------------------------------------------------------------------------
# exact zeros and skipped outputs
# ------------------------------------------------------------------------------------------------
def test_exact_zeros():
    m = model_of("iiwa7")
    r32 = O.load_robot(urdf_path("iiwa7"), torch.float32)
    topo, n = m._topology, r32.n_dofs
    table = m._link_table().detach().clone()
    q, qd = (t.to(DEV) for t in inputs(r32, 131, seed=5))
    kin, _, mom, _, comv, _ = engine.energy_momentum_raw(topo, table, q, torch.zeros_like(qd))
    for t in (kin, mom, comv):
        assert torch.equal(t, torch.zeros_like(t))
    # massless subtree of the last joint: its column of J_com is exactly zero, the others are not
    last = r32.controlled[-1]
    sub = E.subtrees(r32)[last]
    light = table.clone()
    light[sub, 21:25] = 0
    jcom = engine.energy_momentum_raw(topo, light, q, qd)[5]
    assert torch.equal(jcom[:, :, r32.dof[last]], torch.zeros_like(jcom[:, :, 0]))
    assert bool((jcom[:, :, r32.dof[last] - 1] != 0).any())
    # a massless model: no NaN; com, its velocity and its Jacobian are zeros
    massless = table.clone()
    massless[:, 21:25] = 0
    out = engine.energy_momentum_raw(topo, massless, q, qd)
    assert all(bool(torch.isfinite(t).all()) for t in out)
    for t in (out[1], out[3], out[4], out[5]):
        assert torch.equal(t, torch.zeros_like(t))


@pytest.mark.parametrize("stem", ["iiwa7", "allegro_hand_description_left"])
def test_skipped_outputs_and_missing_qd_leave_the_rest_bit_identical(stem):
    m = model_of(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    topo, table, n = m._topology, m._link_table(), r32.n_dofs
    q, qd = (t.to(DEV) for t in inputs(r32, 333, seed=6))
    full = engine.energy_momentum_raw(topo, table, q, qd)
    no_qd = engine.energy_momentum_raw(topo, table, q)
    assert no_qd[0] is None and no_qd[2] is None and no_qd[4] is None
    for k in (1, 3, 5):
        assert torch.equal(no_qd[k], full[k]), NAMES[k]
    for k in range(6):
        wants = [j == k for j in range(6)]
        one = engine.energy_momentum_raw(topo, table, q, qd, *wants)
        assert torch.equal(one[k], full[k]), NAMES[k]
        assert all(one[j] is None for j in range(6) if j != k)
    res = m.compute_energy_and_momentum(q)
    assert res.kinetic_energy is None and res.momentum is None and res.com_velocity is None
    assert torch.equal(res.com_jacobian, full[5])


def test_batch_sizes_alignment_and_large_angles():
    stem = "iiwa7_allegro"
    r32, r64, table = robots(urdf_path(stem), nonsym=True)
    m = model_of(stem)
    topo, n = m._topology, r32.n_dofs
    q, qd = inputs(r32, LARGE, seed=9)
    q[::3, 1] = torch.tensor([2.0e5, -3.3e5, 1.1e6, 7.5e7] * 400)[: q[::3].shape[0]]
    q[1::5, 4] += 12345.678
    x = [t.to(DEV) for t in (q, qd)]
    big = engine.energy_momentum_raw(topo, table, *x)
    check_all("large angles", big, r64, r32, q, qd, torch.arange(0, LARGE, 13))
    for B in (1, 63, 64, 65, LARGE):
        assert_equal(engine.energy_momentum_raw(topo, table, *(t[:B] for t in x)), tuple(o[:B] for o in big), B)
    outs = [shifted(torch.empty_like(o)) for o in big]
    assert raw_call(topo, table, *(shifted(t) for t in x), LARGE, outs) == 0
    assert_equal(tuple(outs), big, "unaligned")


# ------------------------------------------------------------------------------------------------
# launch geometry
# ------------------------------------------------------------------------------------------------
def test_static_shared_memory_matches_the_mirror():
    lib = engine.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    torch.zeros(1, device=DEV)                         # a current context
    attr = (ctypes.c_size_t * 64)()
    rc = cudart.cudaFuncGetAttributes(attr, ctypes.cast(getattr(lib, KERNEL_SYMBOL), ctypes.c_void_p))
    assert rc == 0
    assert attr[0] == STATIC_SMEM                      # cudaFuncAttributes.sharedSizeBytes


_FAM = S.families()


def _tile_cases():
    """The first shipped robot or synthetic family (in that order) that lands on each tile the host rule can choose."""
    cases = {}
    for stem in sorted(URDFS):
        cases.setdefault(tile_of(O.load_robot(urdf_path(stem), torch.float32)), ("urdf", stem))
    for name in sorted(_FAM):
        par, mov = _FAM[name].doc()
        if S.live_slots(par) <= 8:
            cases.setdefault(tile_choice(sum(mov[1:]), len(par), S.live_slots(par))[0], ("family", name))
    cases.pop(None, None)
    return cases


TILE_CASES = _tile_cases()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_energy"))


def _load(kind, name, model_dir):
    path = urdf_path(name) if kind == "urdf" else S.build(_FAM[name], model_dir)
    return drm.DifferentiableRobotModel(path, name, device=DEV), path


def test_no_model_within_the_link_limit_is_refused():
    # the largest footprint: 64 links, 63 joints and 8 branch slots still run 16 rows per CTA; the 64-link chain's rows need
    # 4 KB of link records and 5.6 KB in all
    assert tile_choice(63, 64, 8)[0] == 16
    assert layout_bytes(2, 63, 64, 0) - layout_bytes(1, 63, 64, 0) < 6 * 1024


@pytest.mark.parametrize("tile", sorted(TILE_CASES))
def test_every_tile_the_host_rule_chooses(tile, model_dir):
    kind, name = TILE_CASES[tile]
    m, path = _load(kind, name, model_dir)
    r32, r64, table = robots(path, nonsym=True)
    assert tile_of(r32) == tile
    topo = m._topology
    q, qd = inputs(r32, LARGE, seed=21)
    x = [t.to(DEV) for t in (q, qd)]
    rows = torch.unique(torch.cat([torch.arange(min(3 * tile + 4, LARGE)), torch.arange(3 * tile + 4, LARGE - 3, 97),
                                   torch.arange(LARGE - 3, LARGE)]))
    big = engine.energy_momentum_raw(topo, table, *x)
    check_all(f"{name} T={tile}", big, r64, r32, q, qd, rows)
    for B in sorted({1, max(1, tile - 1), tile, tile + 1, 3 * tile + 3}):
        assert_equal(engine.energy_momentum_raw(topo, table, *(t[:B] for t in x)), tuple(o[:B] for o in big), B)
    outs = [shifted(torch.empty_like(o)) for o in big]
    assert raw_call(topo, table, *(shifted(t) for t in x), LARGE, outs) == 0
    assert_equal(tuple(outs), big, "unaligned")


# ------------------------------------------------------------------------------------------------
# synthetic topologies and refusals
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(_FAM))
def test_synthetic_families_match_oracle(name, model_dir):
    m, path = _load("family", name, model_dir)
    r32, r64, table = robots(path, nonsym=True)
    assert tile_of(r32) is not None
    q, qd = inputs(r32, SMALL, seed=17)
    got = engine.energy_momentum_raw(m._topology, table, q.to(DEV), qd.to(DEV))
    check_all(f"{name}", got, r64, r32, q, qd)


@pytest.mark.parametrize("name", sorted(S.refusal_families()))
def test_refusal_families_are_refused_like_rnea(name, model_dir):
    path = S.build(S.refusal_families()[name], model_dir)
    try:
        m = drm.DifferentiableRobotModel(path, name, device=DEV)
    except ValueError:
        return                                         # refused before any kernel exists (more links than the engine holds)
    z = torch.zeros(5, m._n_dofs, device=DEV)
    with pytest.raises(RuntimeError) as rnea:
        m.compute_inverse_dynamics(z, z, z)
    before = engine.launch_count()
    with pytest.raises(RuntimeError) as em:
        m.compute_energy_and_momentum(z, z)
    assert engine.launch_count() == before
    assert f"code {ELIMIT})" in str(em.value)
    assert "more than 8 live branch points" in str(em.value)
    assert str(em.value).split("failed ", 1)[1] == str(rnea.value).split("failed ", 1)[1]


# ------------------------------------------------------------------------------------------------
# learnable and fused link parameters, launches, capture, edge cases
# ------------------------------------------------------------------------------------------------
def test_learnable_and_fused_models_equal_a_constant_model():
    stem = "iiwa7"
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd = (t.to(DEV) for t in inputs(r32, 333, seed=13))
    init = torch.tensor([[0.3, 0.01, -0.02], [0.015, 0.25, 0.005], [-0.01, 0.02, 0.2]])
    learn, fused = model_of(stem), model_of(stem)
    for m in (learn, fused):
        m.make_link_param_learnable("iiwa_link_3", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.clone()))
        m.make_link_param_learnable("iiwa_link_5", "trans", UnconstrainedTensor(1, 3, init_tensor=torch.tensor([[0.0, 0.02, 0.21]])))
    fused.fuse_learnable_parameters()
    table = learn._link_table().detach().clone()
    want = engine.energy_momentum_raw(learn._topology, table, q, qd)
    assert not torch.equal(want[2], engine.energy_momentum_raw(learn._topology, model_of(stem)._link_table(), q, qd)[2])
    for m in (learn, fused):
        got = m.compute_energy_and_momentum(q, qd)
        assert not any(t.requires_grad for t in got)
        assert_equal(tuple(got), want)


def test_one_launch_per_call_and_cuda_graph_capture():
    m = model_of("panda")
    r32 = O.load_robot(urdf_path("panda"), torch.float32)
    q, qd = (t.to(DEV) for t in inputs(r32, 4099, seed=15))
    want = m.compute_energy_and_momentum(q, qd)
    torch.cuda.synchronize()
    before = engine.launch_count()
    m.compute_energy_and_momentum(q, qd)
    assert engine.launch_count() == before + 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_energy_and_momentum(q, qd)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = m.compute_energy_and_momentum(q, qd)
    for t in got:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert_equal(tuple(got), tuple(want))


def test_edge_cases(model_dir):
    m = model_of("iiwa7")
    n = m._n_dofs
    r32 = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd = (t.to(DEV) for t in inputs(r32, 3, seed=16))
    topo, table = m._topology, m._link_table()
    empty = torch.zeros(0, n, device=DEV)
    res = m.compute_energy_and_momentum(empty, empty)
    assert [tuple(t.shape) for t in res] == [(0,), (0,), (0, n), (0, 3), (0, 3), (0, 3, n)]
    one = m.compute_energy_and_momentum(q[1], qd[1])
    assert [tuple(t.shape) for t in one] == [(), (), (n,), (3,), (3,), (3, n)]
    assert_equal(tuple(one), tuple(t[1] for t in m.compute_energy_and_momentum(q, qd)))
    outs = empty_outs(3, n)
    fixed, fpath = _load("family", "G_all_fixed", model_dir)
    fixed._link_table()                                # the model's table is built (one launch) before counting
    before = engine.launch_count()
    assert raw_call(topo, None, q, qd, 3, outs) == EINVAL
    assert raw_call(topo, table, None, qd, 3, outs) == EINVAL
    assert raw_call(topo, table, q, None, 3, outs) == EINVAL
    for k in (0, 2, 4):                                # each velocity-dependent output needs qd
        assert raw_call(topo, table, q, None, 3, [o if j == k else None for j, o in enumerate(outs)]) == EINVAL
    assert raw_call(topo, table, q, qd, -1, outs) == EINVAL
    assert raw_call(topo, table, q, qd, 0, outs) == 0
    assert raw_call(topo, None, None, None, 0, [None] * 6) == 0
    assert raw_call(topo, table, q, qd, 3, [None] * 6) == 0
    assert engine.launch_count() == before
    # a model without movable joints still has a potential energy and a centre of mass
    fr32, fr64, ftable = robots(fpath, nonsym=False)
    z = torch.zeros(4, 0)
    got = fixed.compute_energy_and_momentum(z.to(DEV), z.to(DEV))
    assert engine.launch_count() == before + 1
    check_all("all fixed", got, fr64, fr32, z, z)
    with pytest.raises(AssertionError):
        m.compute_energy_and_momentum(q[:, :5], qd[:, :5])
    with pytest.raises(AssertionError):
        m.compute_energy_and_momentum(q, qd[:2])
    with pytest.raises(AssertionError):
        m.compute_energy_and_momentum(q.cpu(), qd.cpu())
    with pytest.raises(AssertionError):
        m.compute_energy_and_momentum(q.double(), qd.double())
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        engine.energy_momentum_raw(topo, table, q.cpu(), qd.cpu())
    with pytest.raises(RuntimeError, match="fp32-only"):
        engine.energy_momentum_raw(topo, table, q.double(), qd.double())
