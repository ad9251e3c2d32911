"""GPU: the joint-torque regressor (compute_dynamics_regressor / drmb200_dynamics_regressor, csrc/dynamics_regressor.cu)
against the fp64 oracle (tests/regressor_oracle.py), the reference's autograd Jacobians, the inverse-dynamics kernel and
its adjoint; on every shipped robot, the synthetic topology families and every tile the host rule can choose.

Errors are per configuration, relative to that configuration's largest entry of Y; the bound is
max(8 x the fp32 oracle's error on the same rows, 2e-5), as in test_dynamics_derivatives_gpu.py."""
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
import regressor_oracle as R
import synthetic_robots as S
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL, LARGE = 131, 4099
LARGE_ROWS = torch.cat([torch.arange(SMALL, LARGE - 3, 97), torch.arange(LARGE - 3, LARGE)])
FLAGS = [(True, True), (True, False), (False, True), (False, False)]
EINVAL, ELIMIT = -1, -3


# ------------------------------------------------------------------------------------------------
# mirror of the host tile rule (csrc/dynamics_regressor.cu: RegSmemLayout, regressor_tile)
# ------------------------------------------------------------------------------------------------
KERNEL_SYMBOL = "_ZN3drm25dynamics_regressor_kernelENS_11TreeProgramENS_7RegArgsE"
STATIC_SMEM = 128                 # the mbarrier, as the kernel declares it (pinned by test_static_shared_memory_matches_the_mirror)
TWO_CTAS, CTA_MAX = 113 * 1024, 227 * 1024


def layout_bytes(tc, n, N):
    up4 = lambda x: (x + 3) & ~3  # noqa: E731
    return 4 * (3 * up4(tc * n) + up4(tc * n * N * 14) + N * 28)


def tile_choice(n, N):
    """(TC, dynamic bytes), or (None, bytes needed) when even one configuration per CTA exceeds 227 KB."""
    tc = 1 if N >= 128 else 128 // N
    while tc > 1 and layout_bytes(tc, n, N) + STATIC_SMEM > TWO_CTAS:
        tc -= 1
    b = layout_bytes(tc, n, N)
    return (tc, b) if b + STATIC_SMEM <= CTA_MAX else (None, b + STATIC_SMEM)


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


def robots(path, nonsym):
    r32 = O.load_robot(path, torch.float32)
    if nonsym:
        r32 = D.perturbed(r32)
    return r32, r32.to(torch.float64), O.link_table(r32).float().to(DEV).contiguous()


def inputs(robot, B, seed=3):
    return O.sample_inputs(robot.to(torch.float64), B, seed=seed, dtype=torch.float32)


def flags_of(grav, damp):
    return (engine.GRAVITY if grav else 0) | (engine.DAMPING if damp else 0)


def model_of(stem):
    return drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def raw_call(topo, table, q, qd, qdd, B, flags, Y):
    return engine.lib().drmb200_dynamics_regressor(ctypes.byref(topo), ptr(table), ptr(q), ptr(qd), ptr(qdd), B, flags, ptr(Y),
                                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def shifted(t):
    """The same values 4 bytes off 16-byte alignment."""
    buf = torch.empty(t.numel() + 1, device=DEV, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


# ------------------------------------------------------------------------------------------------
# shipped robots against the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", sorted(URDFS))
def test_shipped_robots_match_oracle(stem, nonsym):
    r32, r64, table = robots(urdf_path(stem), nonsym)
    topo = model_of(stem)._topology
    for B in (SMALL, LARGE):
        q, qd, qdd = inputs(r32, B)
        rows = torch.arange(B) if B == SMALL else LARGE_ROWS
        dev = [t.to(DEV) for t in (q, qd, qdd)]
        sub = [t[rows] for t in (q, qd, qdd)]
        for grav, damp in FLAGS:
            got = engine.dynamics_regressor_raw(topo, table, *dev, flags_of(grav, damp))
            w64 = R.regressor(r64, *(t.double() for t in sub), grav, damp)
            w32 = R.regressor(r32, *sub, grav, damp)
            check(f"{stem} B={B} g{grav:d}d{damp:d}", got.cpu()[rows], w64, w32)


# ------------------------------------------------------------------------------------------------
# the reference's own autograd Jacobians, through the chain rule
# ------------------------------------------------------------------------------------------------
GOLDEN = ["iiwa7", "panda_no_gripper", "fetch_arm_no_gripper", "2link_robot", "allegro_hand_description_left_small_damping"]


@pytest.mark.parametrize("tag", ["sym", "nonsym"])
@pytest.mark.parametrize("stem", GOLDEN)
def test_matches_reference_goldens(stem, tag):
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".regressor.npz"), allow_pickle=False)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    if tag == "nonsym":
        inertia = torch.tensor(g["nonsym.inertia"])
        inertia[0] = r32.inertia[0]
        r32.inertia = inertia
    r64 = r32.to(torch.float64)
    table = O.link_table(r32).float().to(DEV).contiguous()
    topo = model_of(stem)._topology
    q, qd, qdd = (torch.tensor(g[k]) for k in ("q", "qd", "qdd"))
    pre = "" if tag == "sym" else "nonsym."
    N = len(r32.names)

    def stacked(J, grav, damp):           # every stored Jacobian of one flag combination, [16, n, *] per link, concatenated
        parts = []
        for link in range(1, N):
            for pname in ("mass", "com", "inertia_mat", "joint_damping"):
                key = f"{pre}g{grav}d{damp}.{pname}.{link}"
                if key in g:
                    v = torch.as_tensor(J(key, pname, link))
                    parts.append(v.reshape(v.shape[0], v.shape[1], -1).double())
        return torch.cat(parts, dim=2)

    for grav, damp in ((1, 1), (0, 0)):
        Y = engine.dynamics_regressor_raw(topo, table, q.to(DEV), qd.to(DEV), qdd.to(DEV), flags_of(grav, damp)).cpu().double()
        got = R.urdf_parameter_jacobians(Y, r64.mass, r64.com)
        w64 = R.urdf_parameter_jacobians(R.regressor(r64, q.double(), qd.double(), qdd.double(), bool(grav), bool(damp)),
                                         r64.mass, r64.com)
        want = stacked(lambda key, p, l: g[key], grav, damp)
        # the goldens are the reference's fp32 evaluation: the bound is the fp64 oracle's distance from them
        check(f"{stem} {pre}g{grav}d{damp}", stacked(lambda key, p, l: got[p][:, :, l], grav, damp), want,
              stacked(lambda key, p, l: w64[p][:, :, l].float(), grav, damp), floor=2e-4)


# ------------------------------------------------------------------------------------------------
# identities with the shipped kernels, structure
# ------------------------------------------------------------------------------------------------
IDENTITY = ["iiwa7", "panda", "trifinger_edu", "allegro_hand_description_left", "iiwa7_allegro"]


@pytest.mark.parametrize("nonsym", [False, True], ids=["sym", "nonsym"])
@pytest.mark.parametrize("stem", IDENTITY)
def test_identities_with_inverse_dynamics_and_its_adjoint(stem, nonsym):
    r32, _, table = robots(urdf_path(stem), nonsym)
    topo = model_of(stem)._topology
    q, qd, qdd = (t.to(DEV) for t in inputs(r32, 257, seed=8))
    G = torch.randn(q.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    pi = table[:, 12:26]
    for grav, damp in FLAGS:
        flags = flags_of(grav, damp)
        Y = engine.dynamics_regressor_raw(topo, table, q, qd, qdd, flags)
        tau = engine.inverse_dynamics_raw(topo, table, q, qd, qdd, flags)
        scale = torch.einsum("bilk,lk->bi", Y.abs(), pi.abs()).amax(1, keepdim=True)     # per configuration
        err = ((torch.einsum("bilk,lk->bi", Y, pi) - tau).abs() / scale).max()
        assert float(err) < 1e-5, (stem, grav, damp, float(err))
        # sum_b g_b^T Y_b is the inertial part of the table gradient of the RNEA adjoint
        ta = table.clone().requires_grad_(True)
        out = engine.InverseDynamicsFunction.apply(ta, q, qd, qdd, topo, flags)
        gt, = torch.autograd.grad((G * out).sum(), [ta])
        vjp = torch.einsum("bi,bilk->lk", G, Y)
        vscale = torch.einsum("bi,bilk->lk", G.abs(), Y.abs()).max()
        assert float((vjp - gt[:, 12:26]).abs().max() / vscale) < 1e-5, (stem, grav, damp)
        # damping columns: qd of the link's own dof, exact zeros everywhere else
        links = r32.controlled
        dof = [r32.dof[l] for l in links]
        if damp:
            assert torch.equal(Y[:, dof, links, 13], qd[:, dof])
        zero = R.structural_zeros(r32, damp).to(DEV)
        assert bool((Y[:, zero] == 0).all())
        # fixed links with a movable ancestor have nonzero columns
        for l in range(1, len(r32.names)):
            if r32.dof[l] < 0 and any(r32.dof[k] >= 0 for k in _ancestors(r32, l)):
                assert bool((Y[:, :, l, :13] != 0).any()), (stem, r32.names[l])


def _ancestors(robot, l):
    out = []
    while robot.parent[l] > 0:
        l = robot.parent[l]
        out.append(l)
    return out


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
        r = O.load_robot(urdf_path(stem), torch.float32)
        cases.setdefault(tile_choice(r.n_dofs, len(r.names))[0], ("urdf", stem))
    for name in sorted(_FAM):
        par, mov = _FAM[name].doc()
        n = sum(mov[1:])
        if n:
            cases.setdefault(tile_choice(n, len(par))[0], ("family", name))
    cases.pop(None, None)
    return cases


TILE_CASES = _tile_cases()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_regressor"))


def _load(kind, name, model_dir):
    path = urdf_path(name) if kind == "urdf" else S.build(_FAM[name], model_dir)
    return drm.DifferentiableRobotModel(path, name, device=DEV), path


def checked_rows(T):
    return torch.unique(torch.cat([torch.arange(min(3 * T + 4, LARGE)), torch.arange(3 * T + 4, LARGE - 3, 97),
                                   torch.arange(LARGE - 3, LARGE)]))


@pytest.mark.parametrize("tile", sorted(TILE_CASES))
def test_every_tile_the_host_rule_chooses(tile, model_dir):
    kind, name = TILE_CASES[tile]
    m, path = _load(kind, name, model_dir)
    r32, r64, table = robots(path, nonsym=True)
    assert tile_choice(r32.n_dofs, len(r32.names))[0] == tile
    topo = m._topology
    q, qd, qdd = inputs(r32, LARGE, seed=21)
    x = [t.to(DEV) for t in (q, qd, qdd)]
    rows = checked_rows(tile)
    flags = flags_of(True, True)
    big = engine.dynamics_regressor_raw(topo, table, *x, flags)
    sub = [t[rows] for t in (q, qd, qdd)]
    check(f"{name} TC={tile}", big.cpu()[rows], R.regressor(r64, *(t.double() for t in sub)), R.regressor(r32, *sub))
    for B in sorted({1, max(1, tile - 1), tile, tile + 1, 3 * tile + 3}):
        assert torch.equal(engine.dynamics_regressor_raw(topo, table, *(t[:B] for t in x), flags), big[:B]), B
    Y = shifted(torch.empty_like(big))
    assert raw_call(topo, table, *(shifted(t) for t in x), LARGE, flags, Y) == 0
    assert torch.equal(Y, big)


def test_large_angles_mixed_into_ordinary_rows():
    stem = "iiwa7"
    r32, r64, table = robots(urdf_path(stem), nonsym=False)
    topo = model_of(stem)._topology
    q, qd, qdd = inputs(r32, 64, seed=23)
    q[::3, 1] = torch.tensor([2.0e5, -3.3e5, 1.1e6, 7.5e7] * 6)[: q[::3].shape[0]]
    q[1::5, 4] += 12345.678
    got = engine.dynamics_regressor_raw(topo, table, q.to(DEV), qd.to(DEV), qdd.to(DEV), flags_of(True, True))
    check("large angles", got.cpu(), R.regressor(r64, q.double(), qd.double(), qdd.double()), R.regressor(r32, q, qd, qdd))


# ------------------------------------------------------------------------------------------------
# synthetic topologies and refusals
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(_FAM))
def test_synthetic_families_match_oracle_or_are_refused(name, model_dir):
    spec = _FAM[name]
    m, path = _load("family", name, model_dir)
    r32, r64, table = robots(path, nonsym=True)
    n, N = r32.n_dofs, len(r32.names)
    topo = m._topology
    if n == 0:
        z = torch.zeros(5, 0, device=DEV)
        before = engine.launch_count()
        assert engine.dynamics_regressor_raw(topo, table, z, z, z, 3).shape == (5, 0, N, 14)
        assert engine.launch_count() == before
        return
    tile, need = tile_choice(n, N)
    q, qd, qdd = inputs(r32, SMALL, seed=17)
    if tile is None:
        before = engine.launch_count()
        with pytest.raises(RuntimeError, match=rf"needs {need} B of shared memory per CTA \(> 227 KB\) for its dynamics regressor"):
            engine.dynamics_regressor_raw(topo, table, q.to(DEV), qd.to(DEV), qdd.to(DEV), 3)
        assert engine.launch_count() == before
        return
    got = engine.dynamics_regressor_raw(topo, table, q.to(DEV), qd.to(DEV), qdd.to(DEV), 3)
    check(f"{name} TC={tile}", got.cpu(), R.regressor(r64, q.double(), qd.double(), qdd.double()), R.regressor(r32, q, qd, qdd))


def test_chain64_is_refused_with_the_documented_message(model_dir):
    m, _ = _load("family", "F_chain64", model_dir)
    tile, need = tile_choice(63, 64)
    assert tile is None
    z = torch.zeros(3, 63, device=DEV)
    with pytest.raises(RuntimeError, match=rf"code {ELIMIT}\): model needs {need} B of shared memory per CTA"):
        m.compute_dynamics_regressor(z, z, z)


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
    with pytest.raises(RuntimeError) as reg:
        m.compute_dynamics_regressor(z, z, z)
    assert engine.launch_count() == before
    assert "more than 8 live branch points" in str(reg.value)
    assert str(reg.value).split("failed ", 1)[1] == str(rnea.value).split("failed ", 1)[1]


# ------------------------------------------------------------------------------------------------
# learnable and fused link parameters, launches, capture, edge cases
# ------------------------------------------------------------------------------------------------
def test_learnable_and_fused_models_equal_a_constant_model():
    stem = "iiwa7"
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in inputs(r32, 333, seed=13))
    init = torch.tensor([[0.3, 0.01, -0.02], [0.015, 0.25, 0.005], [-0.01, 0.02, 0.2]])
    learn, fused = model_of(stem), model_of(stem)
    for m in (learn, fused):
        m.make_link_param_learnable("iiwa_link_3", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=init.clone()))
        m.make_link_param_learnable("iiwa_link_5", "trans", UnconstrainedTensor(1, 3, init_tensor=torch.tensor([[0.0, 0.02, 0.21]])))
    fused.fuse_learnable_parameters()
    table = learn._link_table().detach().clone()
    want = engine.dynamics_regressor_raw(learn._topology, table, q, qd, qdd, flags_of(True, True))
    for m in (learn, fused):
        got = m.compute_dynamics_regressor(q, qd, qdd)
        assert not got.requires_grad
        assert torch.equal(got, want)
        pi = m.inertial_parameters()
        assert pi.requires_grad and pi.shape == (len(r32.names), 14)
        tau = m.compute_inverse_dynamics(q, qd, qdd)
        scale = torch.einsum("bilk,lk->bi", got.abs(), pi.detach().abs()).amax(1, keepdim=True)
        assert float(((torch.einsum("bilk,lk->bi", got, pi.detach()) - tau.detach()).abs() / scale).max()) < 1e-5


def test_one_launch_per_call_and_cuda_graph_capture():
    m = model_of("panda")
    r32 = O.load_robot(urdf_path("panda"), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in inputs(r32, 4099, seed=15))
    want = m.compute_dynamics_regressor(q, qd, qdd)
    torch.cuda.synchronize()
    before = engine.launch_count()
    m.compute_dynamics_regressor(q, qd, qdd)
    assert engine.launch_count() == before + 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.compute_dynamics_regressor(q, qd, qdd)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = m.compute_dynamics_regressor(q, qd, qdd)
    got.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_edge_cases(model_dir):
    m = model_of("iiwa7")
    n, N = m._n_dofs, len(m.get_link_names())
    r32 = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in inputs(r32, 3, seed=16))
    topo, table = m._topology, m._link_table()
    empty = torch.zeros(0, n, device=DEV)
    assert m.compute_dynamics_regressor(empty, empty, empty).shape == (0, n, N, 14)
    one = m.compute_dynamics_regressor(q[1], qd[1], qdd[1], False, False)
    assert one.shape == (n, N, 14)
    assert torch.equal(one, m.compute_dynamics_regressor(q, qd, qdd, False, False)[1])
    Y = torch.empty(3, n, N, 14, device=DEV)
    fixed, _ = _load("family", "G_all_fixed", model_dir)
    fixed._link_table()                                # the model's table is built (one launch) before counting
    before = engine.launch_count()
    for args in ((None, q, qd, qdd), (table, None, qd, qdd), (table, q, None, qdd), (table, q, qd, None)):
        assert raw_call(topo, *args, 3, 3, Y) == EINVAL
    assert raw_call(topo, table, q, qd, qdd, 3, 3, None) == EINVAL
    assert raw_call(topo, table, q, qd, qdd, -1, 3, Y) == EINVAL
    assert raw_call(topo, table, q, qd, qdd, 0, 3, Y) == 0
    assert raw_call(topo, None, None, None, None, 0, 3, None) == 0
    assert engine.launch_count() == before
    z = torch.zeros(4, 0, device=DEV)
    assert fixed.compute_dynamics_regressor(z, z, z).shape == (4, 0, 4, 14)
    assert engine.launch_count() == before
    with pytest.raises(AssertionError):
        m.compute_dynamics_regressor(q[:, :5], qd[:, :5], qdd[:, :5])
    with pytest.raises(AssertionError):
        m.compute_dynamics_regressor(q.cpu(), qd.cpu(), qdd.cpu())
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        engine.dynamics_regressor_raw(topo, table, q.cpu(), qd.cpu(), qdd.cpu(), 0)
    with pytest.raises(RuntimeError, match="fp32-only"):
        engine.dynamics_regressor_raw(topo, table, q.double(), qd.double(), qdd.double(), 0)
