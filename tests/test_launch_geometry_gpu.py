"""GPU: how a batch is cut into tiles and staged, at the batch sizes, pointer offsets and option values that the
arithmetic tests elsewhere in the suite never reach.

  A. The persistent adjoint kernels (backward.cu, backward_rnea.cu, backward_aba.cu, and the rollout adjoint built on
     the last) at batches where every CTA walks two or more tiles, the last one ragged:
       * per-row input gradients are bit-identical to the same rows computed in a small sub-batch (one thread per row,
         and the adjoint launchers pick their tile from shared memory, not from the batch size);
       * table gradients equal the fp64 sum of the table gradients of disjoint single-pass chunks;
       * 1 024 rows from the last quarter of the batch (second or later tiles) match autograd of the fp64 oracle.
  B. The multi-end-effector tree kernel (fk_tree.cu) under every "tree_warps" x "tree_bufs" setting and a grid capped
     to one CTA per SM: bit-identical to the single-link kernel, link by link.
  C. The inverse-dynamics kernel's prefolded path under both forced tiles ("rnea_tile").
  D. Every kernel with inputs or outputs off 16-byte alignment (cooperative copies): bit-identical to aligned runs.

Options are process-global: tests set them inside fixtures or `options()` blocks that restore them in `finally`, and an
autouse check asserts after every test that each option reads its default again.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from conftest import assert_close, urdf_path
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar, UnconstrainedTensor
from oracle import drm_oracle as O
from rollout_oracle import forward_dynamics_rollout
from test_backward_gpu import _oracle_grads, learnable_model, shifted
from test_fk_multi_gpu import CASES
from test_forward_dynamics_backward_gpu import ARMS, family_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# The adjoint kernels run `for (tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)` on a grid of at most
# BWD_MAX_GRID = 132 * 8 CTAs (csrc/backward_common.cuh).  A batch of at least 2 * BWD_MAX_GRID * T_max rows plus a
# ragged remainder therefore gives every CTA two or more tiles, the last one partial, whatever the occupancy.
BWD_MAX_GRID = 132 * 8
B_FK_RNEA = 2 * BWD_MAX_GRID * 128 + 37          # FK and RNEA adjoints: tiles of at most 128 rows -> 270 373
B_ABA = 70001                                    # ABA adjoint: tiles of at most 32 rows (2 * 1056 * 32 = 67 584)
assert B_FK_RNEA >= 2 * BWD_MAX_GRID * 128 and B_FK_RNEA % 32 != 0
assert B_ABA >= 2 * BWD_MAX_GRID * 32 and B_ABA % 16 != 0
CHUNK = 16384                                    # single-pass chunks: at most 128 tiles of 128 rows, far below the cap
SUB = 4000                                       # rows of the sub-batch the big batch's input gradients are compared with
# family-relative, big-batch table gradient vs fp64 sum of the chunks; the worst measured on an H100 80GB HBM3 (400 W
# power limit) was 7.6e-7.  A lost or double-counted tile is off by orders of magnitude more.
TABLE_TOL = 1e-5

# the library's option table (csrc/c_api.cu) and its defaults; DRMB200_<NAME> in the environment overrides a default
OPTION_DEFAULTS = {"fk_variant": 1, "fk_tile": 0, "fk_unroll": 2, "fk_packed": 1, "rnea_packed": 1, "host_fused": 1,
                   "fk_reserved": 0, "fk_pdl": 0, "tree_warps": 0, "tree_grid_cap": 0, "tree_bufs": 1, "rnea_fold": 1,
                   "rnea_tile": 0, "rnea_bwd_chain": 1}


def _default(name):
    env = os.environ.get("DRMB200_" + name.upper())
    return int(env) if env is not None else OPTION_DEFAULTS[name]


@pytest.fixture(autouse=True)
def options_are_restored():
    yield
    now = {k: engine.get_option(k) for k in OPTION_DEFAULTS}
    assert now == {k: _default(k) for k in OPTION_DEFAULTS}, "a test left a library option changed"


@contextlib.contextmanager
def options(**values):
    try:
        for k, v in values.items():
            engine.set_option(k, v)
        yield
    finally:
        for k in values:
            engine.set_option(k, _default(k))


def report(what, value):
    """Measured error, printed for the record (pytest -s)."""
    print(f"[launch-geometry] {what}: {value:.3e}")


def grads_of(params):
    return {k: (torch.zeros_like(p) if p.grad is None else p.grad).detach().clone() for k, p in params.items()}


def check_table_against_chunks(name, big, chunk_sums):
    """Family-relative (one family per parameter kind over all links) comparison of the big batch's table gradient with
    the fp64 sum of the chunks' table gradients."""
    for pname in sorted({k[1] for k in big}):
        keys = [k for k in big if k[1] == pname]
        fam = max(float(chunk_sums[k].abs().max()) for k in keys)
        if fam == 0.0:
            assert all(float(big[k].abs().max()) == 0.0 for k in keys), f"{name} {pname}"
            continue
        err = max(float((big[k].double().cpu() - chunk_sums[k]).abs().max()) for k in keys)
        report(f"{name} table {pname} (family-relative)", err / fam)
        for k in keys:
            family_close(big[k].cpu().numpy(), chunk_sums[k].numpy(), fam, TABLE_TOL, f"{name} table grad {k}")


def check_inputs_against_oracle(name, got, want):
    """The tolerance of test_backward_gpu.py's oracle tests (rtol 2e-4, absolute floor 2e-5 x the gradient scale), with the
    scale taken over the input gradients alone: no parameter gradient of a 1 024-row loss loosens the floor."""
    scale = max(float(w.abs().max()) for w in want.values())
    for k in want:
        g = got[k].cpu().double()
        report(f"{name} {k}_grad vs oracle (family-relative)", float((g - want[k]).abs().max() / want[k].abs().max()))
        assert_close(g.numpy(), want[k].numpy(), rtol=2e-4, atol=2e-5 * max(scale, 1.0), what=f"{name} d{k} (later tiles)")


def run_in_chunks(batch, run_rows, params):
    """Sum (fp64) of the table gradients of run_rows over disjoint chunks of at most CHUNK rows."""
    sums = None
    for start in range(0, batch, CHUNK):
        for p in params.values():
            p.grad = None
        run_rows(slice(start, min(batch, start + CHUNK)))
        g = grads_of(params)
        sums = {k: v.double().cpu() for k, v in g.items()} if sums is None else {k: sums[k] + g[k].double().cpu() for k in g}
    return sums


def tail_rows(batch, gen, n=1024):
    """n rows from the last quarter of the batch: tiles that the persistent kernels reach on a CTA's second or later trip."""
    lo = batch - batch // 4
    return (lo + torch.randperm(batch - lo, generator=gen)[:n]).sort().values


def sub_rows(batch, gen):
    return torch.randperm(batch, generator=gen)[:SUB].sort().values


# ---------------------------------------------------------------------------------------------------------------------
# A. persistent adjoints, two or more tiles per CTA
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem,link", [("iiwa7", "iiwa_link_ee"), ("iiwa7_allegro", "link_15.0_tip")])
def test_fk_adjoint_with_several_tiles_per_cta(stem, link):
    B = B_FK_RNEA
    robot = O.load_robot(urdf_path(stem), torch.float32)
    n = robot.n_dofs
    q = O.sample_inputs(robot, B, seed=21)[0].to(DEV)
    gen = torch.Generator().manual_seed(21)
    G = [torch.randn(B, *s, generator=gen).to(DEV) for s in ((3,), (4,), (3, n), (3, n))]
    m, params = learnable_model(stem)

    def run(rows):
        qq = q[rows].clone().requires_grad_(True)
        outs = m.compute_fk_and_jacobian(qq, link)
        sum((g[rows] * o).sum() for g, o in zip(G, outs)).backward()
        return qq.grad, outs[1].detach()

    gq, quat = run(slice(None))
    big = grads_of(params)
    idx = sub_rows(B, gen)
    for p in params.values():
        p.grad = None
    gq_sub, _ = run(idx.to(DEV))
    assert torch.equal(gq[idx.to(DEV)], gq_sub), f"{stem}: q_grad rows differ between the big batch and a sub-batch"
    check_table_against_chunks(f"fk {stem}", big, run_in_chunks(B, run, params))

    # oracle: rows in later tiles; the oracle picks each row's quaternion sign, so flip G_quat per row to the same function
    rows = tail_rows(B, gen)
    qr = q[rows.to(DEV)].cpu()
    o_quat = O.forward_kinematics(O.load_robot(urdf_path(stem), torch.float64), qr.double(), link)[1]
    sign = torch.sign((quat[rows.to(DEV)].cpu().double() * o_quat).sum(1, keepdim=True))
    Gp, Gq, Gl, Ga = (g[rows.to(DEV)].cpu().double() for g in G)
    Gq = Gq * sign

    def oracle_loss(rb, qq):
        p, qu = O.forward_kinematics(rb, qq, link)
        jl, ja = O.jacobian(rb, qq, link)
        return (Gp * p).sum() + (Gq * qu).sum() + (Gl * jl).sum() + (Ga * ja).sum()

    (dq,), _, _ = _oracle_grads(stem, oracle_loss, [qr])
    check_inputs_against_oracle(f"fk {stem}", {"q": gq[rows.to(DEV)]}, {"q": dq})


@pytest.mark.parametrize("stem,kernel", [("allegro_hand_description_left", "tree"), ("trifinger_edu", "tree"),
                                         ("iiwa7_allegro", "tree"), ("iiwa7", "chain"), ("panda_no_gripper", "chain")])
def test_rnea_adjoint_with_several_tiles_per_cta(stem, kernel):
    B = B_FK_RNEA
    robot = O.load_robot(urdf_path(stem), torch.float32)
    n = robot.n_dofs
    assert all(p == i - 1 for i, p in enumerate(robot.parent) if i > 0) == (kernel == "chain")     # which adjoint kernel runs
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, B, seed=22))
    gen = torch.Generator().manual_seed(22)
    G = torch.randn(B, n, generator=gen).to(DEV)
    m, params = learnable_model(stem)

    def run(rows):
        ins = [t[rows].clone().requires_grad_(True) for t in (q, qd, qdd)]
        tau = m.compute_inverse_dynamics(*ins, include_gravity=True, use_damping=True)
        (G[rows] * tau).sum().backward()
        return [t.grad for t in ins]

    big_in = run(slice(None))
    big = grads_of(params)
    idx = sub_rows(B, gen).to(DEV)
    for p in params.values():
        p.grad = None
    for name, a, b in zip(("q", "qd", "qdd"), big_in, run(idx)):
        assert torch.equal(a[idx], b), f"{stem}: {name}_grad rows differ between the big batch and a sub-batch"
    check_table_against_chunks(f"rnea {kernel} {stem}", big, run_in_chunks(B, run, params))

    rows = tail_rows(B, gen).to(DEV)
    Gr = G[rows].cpu().double()
    want, _, _ = _oracle_grads(
        stem, lambda r, a, b, c: (Gr * O.inverse_dynamics(r, a, b, c, True, True)).sum(), [t[rows].cpu() for t in (q, qd, qdd)])
    check_inputs_against_oracle(f"rnea {kernel} {stem}", {k: g[rows] for k, g in zip(("q", "qd", "qdd"), big_in)},
                                dict(zip(("q", "qd", "qdd"), want)))


def inertial_model(stem):
    """Only mass / com / inertia_mat / damping learnable: with no input gradient the RNEA backward takes the single-sweep
    kernel (DRMB200_INERTIAL_GRADS_ONLY)."""
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    params = {}
    for i, body in enumerate(m._bodies):
        if i == 0:
            continue
        mods = {"mass": UnconstrainedScalar(init_val=body.inertia.mass().detach().clone()),
                "com": UnconstrainedTensor(1, 3, init_tensor=body.inertia.com().detach().clone().reshape(1, 3)),
                "inertia_mat": UnconstrainedTensor(3, 3, init_tensor=body.inertia.inertia_mat().detach().clone().reshape(3, 3))}
        if body.joint_idx is not None:
            mods["joint_damping"] = UnconstrainedScalar(init_val=body.joint_damping().detach().clone())
        for pname, mod in mods.items():
            m.make_link_param_learnable(body.name, pname, mod)
            params[(i, pname)] = mod.param
    assert not m._kinematic_params_learnable()
    return m, params


@pytest.mark.parametrize("stem", ["iiwa7", "iiwa7_allegro"])
def test_inertial_only_rnea_adjoint_with_several_tiles_per_cta(stem):
    """The single-sweep kernel produces table columns only, so only its table gradient is checked (no input gradients to
    compare row by row or against the oracle)."""
    B = B_FK_RNEA
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, B, seed=23))
    G = torch.randn(B, robot.n_dofs, generator=torch.Generator().manual_seed(23)).to(DEV)
    m, params = inertial_model(stem)

    def run(rows):
        (G[rows] * m.compute_inverse_dynamics(q[rows], qd[rows], qdd[rows])).sum().backward()

    run(slice(None))
    big = grads_of(params)
    check_table_against_chunks(f"rnea inertial {stem}", big, run_in_chunks(B, run, params))


@pytest.mark.parametrize("stem,nonsym", [("iiwa7", True), ("trifinger_edu", False), ("iiwa7_allegro", False)])
def test_aba_adjoint_with_several_tiles_per_cta(stem, nonsym):
    B = B_ABA
    robot = O.load_robot(urdf_path(stem), torch.float64)
    n = robot.n_dofs
    m, params = learnable_model(stem)
    if nonsym:
        gen = torch.Generator().manual_seed(17)
        scale = robot.inertia.abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-6)
        robot.inertia = (robot.inertia + 0.05 * scale * torch.randn(robot.inertia.shape, generator=gen, dtype=torch.float64)).float().double()
        with torch.no_grad():
            for (i, pname), p in params.items():
                if pname == "inertia_mat":
                    p.copy_(robot.inertia[i].float().to(DEV))
    q, qd, _ = (t.float().to(DEV) for t in O.sample_inputs(robot, B, seed=24, dtype=torch.float64))
    gen = torch.Generator().manual_seed(24)
    f = torch.randn(B, n, generator=gen).to(DEV)
    G = torch.randn(B, n, generator=gen).to(DEV)

    def run(rows):
        ins = [t[rows].clone().requires_grad_(True) for t in (q, qd, f)]
        qdd = m.compute_forward_dynamics(*ins, include_gravity=True, use_damping=True)
        (G[rows] * qdd).sum().backward()
        return [t.grad for t in ins]

    big_in = run(slice(None))
    big = grads_of(params)
    idx = sub_rows(B, gen).to(DEV)
    for p in params.values():
        p.grad = None
    for name, a, b in zip(("q", "qd", "f"), big_in, run(idx)):
        assert torch.equal(a[idx], b), f"{stem}: {name}_grad rows differ between the big batch and a sub-batch"
    check_table_against_chunks(f"aba {stem}", big, run_in_chunks(B, run, params))

    rows = tail_rows(B, gen).to(DEV)
    ins = [t[rows].cpu().double().requires_grad_(True) for t in (q, qd, f)]
    qdd_o = O.forward_dynamics(robot, *ins, True, True)
    want = torch.autograd.grad((G[rows].cpu().double() * qdd_o).sum(), ins)
    tol = 2e-3 if stem in ARMS else 2e-2
    for name, got, w in zip(("q", "qd", "f"), big_in, want):
        got = got[rows].cpu().numpy()
        report(f"aba {stem} {name}_grad vs oracle (family-relative)", float(np.abs(got - w.numpy()).max() / w.abs().max()))
        family_close(got, w.numpy(), float(w.abs().max()), tol, f"{stem} d{name} (later tiles)")


def test_rollout_adjoint_with_several_tiles_per_cta():
    """The rollout adjoint sums the ABA adjoint's per-CTA partial tables over all steps before one reduction."""
    stem, B, T, dt = "iiwa7", B_ABA, 3, 2.0 ** -10
    robot = O.load_robot(urdf_path(stem), torch.float32)
    n = robot.n_dofs
    q0, qd0, _ = O.sample_inputs(robot, B, seed=25, vel_scale=0.02)
    gen = torch.Generator().manual_seed(25)
    q0, qd0 = q0.to(DEV), qd0.clamp(-1, 1).to(DEV)
    f = (0.05 * torch.randn(T, B, n, generator=gen)).to(DEV)
    G = [torch.randn(T, B, n, generator=gen).to(DEV) for _ in range(3)]
    m, params = learnable_model(stem)

    def run(rows):
        ins = [q0[rows].clone().requires_grad_(True), qd0[rows].clone().requires_grad_(True), f[:, rows].clone().requires_grad_(True)]
        outs = m.compute_forward_dynamics_rollout(*ins, dt, include_gravity=True, use_damping=True)
        sum((g[:, rows] * o).sum() for g, o in zip(G, outs)).backward()
        return [t.grad for t in ins]

    big_in = run(slice(None))
    big = grads_of(params)
    idx = sub_rows(B, gen).to(DEV)
    for p in params.values():
        p.grad = None
    sub_in = run(idx)
    for name, a, b in zip(("q0", "qd0"), big_in[:2], sub_in[:2]):
        assert torch.equal(a[idx], b), f"{name}_grad rows differ between the big batch and a sub-batch"
    assert torch.equal(big_in[2][:, idx], sub_in[2]), "f_grad rows differ between the big batch and a sub-batch"
    check_table_against_chunks("rollout iiwa7", big, run_in_chunks(B, run, params))

    rows = tail_rows(B, gen).to(DEV)
    rb = O.load_robot(urdf_path(stem), torch.float64)
    ins = [q0[rows].cpu().double().requires_grad_(True), qd0[rows].cpu().double().requires_grad_(True),
           f[:, rows].cpu().double().requires_grad_(True)]
    outs = forward_dynamics_rollout(rb, *ins, dt, True, True)
    loss = sum((g[:, rows].cpu().double() * o).sum() for g, o in zip(G, outs))
    want = torch.autograd.grad(loss, ins)
    got = [big_in[0][rows], big_in[1][rows], big_in[2][:, rows]]
    for name, a, w in zip(("q0", "qd0", "f"), got, want):
        a = a.cpu().numpy()
        report(f"rollout {stem} {name}_grad vs oracle (family-relative)", float(np.abs(a - w.numpy()).max() / w.abs().max()))
        family_close(a, w.numpy(), float(w.abs().max()), 1e-4, f"rollout d{name} (later tiles)")


# ---------------------------------------------------------------------------------------------------------------------
# B. tree-kernel knobs
# ---------------------------------------------------------------------------------------------------------------------
TREE_CONFIGS = [(w, b, 0) for w in (1, 2, 3, 4) for b in (1, 2)] + [(1, 1, 1), (1, 2, 1)]


@pytest.fixture(params=TREE_CONFIGS, ids=[f"warps{w}_bufs{b}" + ("_cap1" if c else "") for w, b, c in TREE_CONFIGS])
def tree_config(request):
    warps, bufs, cap = request.param
    with options(tree_warps=warps, tree_bufs=bufs, tree_grid_cap=cap):
        yield request.param


_single_link_cache = {}


def single_link_outputs(stem, batch):
    """compute_fk_and_jacobian of every CASES link (default options), computed once per (robot, batch)."""
    key = (stem, batch)
    if key not in _single_link_cache:
        m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
        robot = O.load_robot(urdf_path(stem), torch.float32)
        q = O.sample_inputs(robot, batch, seed=batch + 7)[0].to(DEV)
        with torch.no_grad():
            want = {name: m.compute_fk_and_jacobian(q, name) for name in CASES[stem]}
        _single_link_cache[key] = (m, q, want)
    return _single_link_cache[key]


@pytest.mark.parametrize("stem", sorted(CASES))
def test_tree_kernel_knobs_are_bit_identical_to_the_single_link_kernel(stem, tree_config):
    warps, bufs, cap = tree_config
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    # capped grid: one CTA of one warp per SM, so at 40 000 rows every warp walks ~40 000 / (32 * SMs) tiles
    assert 40000 // (32 * sms) >= 4
    for batch in (1, 31, 4099, 40000):
        m, q, want = single_link_outputs(stem, batch)
        links = CASES[stem]
        idx = [m._name_to_idx_map[name] for name in links]
        table, topo = m._link_table(), m._topology
        full = engine.fk_jacobian_multi_raw(topo, idx, table, q)
        for e, name in enumerate(links):
            for a, b, what in zip(full, want[name], ("pos", "quat", "jlin", "jang")):
                assert torch.equal(a[e], b), f"{stem} {name} {what} differs at batch {batch}"
        if bufs == 2:
            pos, quat, jl, ja = engine.fk_jacobian_multi_raw(topo, idx, table, q, want_jac=False)
            assert jl is None and ja is None and torch.equal(pos, full[0]) and torch.equal(quat, full[1])
            pos, quat, jl, ja = engine.fk_jacobian_multi_raw(topo, idx, table, q, want_pos=False, want_quat=False)
            assert pos is None and quat is None and torch.equal(jl, full[2]) and torch.equal(ja, full[3])
            for a, b in zip(engine.fk_jacobian_multi_raw(topo, idx, table, shifted(q)), full):
                assert torch.equal(a, b), f"{stem}: unaligned q differs at batch {batch}"


# ---------------------------------------------------------------------------------------------------------------------
# C. forced inverse-dynamics tiles on the prefolded path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(params=[64, 128], ids=["tile64", "tile128"])
def rnea_tile(request):
    with options(rnea_tile=request.param):
        yield request.param


@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro"])
def test_prefolded_path_is_bit_identical_under_both_tiles(stem, rnea_tile):
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    table, topo = m._link_table(), m._topology
    folded = engine.fold_link_table(topo, table)
    assert folded is not None
    for batch in (129, 1003, 40000):
        q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=batch + 3))
        a = engine.inverse_dynamics_raw(topo, table, q, qd, qdd, 3)
        b = engine.inverse_dynamics_raw(topo, table, q, qd, qdd, 3, folded=folded)
        assert torch.equal(a, b), f"{stem} tile {rnea_tile} batch {batch}"


# ---------------------------------------------------------------------------------------------------------------------
# D. unaligned inputs and outputs
# ---------------------------------------------------------------------------------------------------------------------
UNALIGNED = pytest.mark.parametrize("stem,batch", [(s, b) for s in ("iiwa7", "iiwa7_allegro") for b in (1003, 1024)])


def shift_variants(k):
    """Which of k inputs to shift: each one in turn, then all together."""
    return [tuple(i == j for i in range(k)) for j in range(k)] + [(True,) * k]


def seeded(stem, batch):
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=batch + 11))
    f = torch.randn(batch, robot.n_dofs, generator=torch.Generator().manual_seed(batch)).to(DEV)
    return q, qd, qdd, f


@UNALIGNED
def test_unaligned_forward_kernels_are_bit_identical(stem, batch):
    q, qd, qdd, f = seeded(stem, batch)
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    table, topo = m._link_table(), m._topology
    n = q.shape[1]

    def pick(ins, mask):
        return [shifted(t) if s else t for t, s in zip(ins, mask)]

    H = engine.mass_matrix_raw(topo, table, q)
    assert torch.equal(engine.mass_matrix_raw(topo, table, shifted(q)), H)
    assert torch.equal(engine.mass_matrix_raw(topo, table, q, out=shifted(torch.empty(batch, n, n, device=DEV))), H)

    for flags in (1, 3):
        qdd_a = engine.forward_dynamics_raw(topo, table, q, qd, f, flags)
        tau = engine.inverse_dynamics_raw(topo, table, q, qd, qdd, flags)
        for mask in shift_variants(3):
            assert torch.equal(engine.forward_dynamics_raw(topo, table, *pick((q, qd, f), mask), flags), qdd_a), f"aba {mask}"
            assert torch.equal(engine.inverse_dynamics_raw(topo, table, *pick((q, qd, qdd), mask), flags), tau), f"rnea {mask}"
        assert torch.equal(engine.forward_dynamics_raw(topo, table, q, qd, f, flags, out=shifted(torch.empty_like(q))), qdd_a)
        assert torch.equal(engine.inverse_dynamics_raw(topo, table, q, qd, qdd, flags, out=shifted(torch.empty_like(q))), tau)

        state = engine.dynamic_state_raw(topo, table, q, qd, qdd, flags)
        for mask in shift_variants(3):
            for a, b in zip(engine.dynamic_state_raw(topo, table, *pick((q, qd, qdd), mask), flags), state):
                assert torch.equal(a, b), f"dynamic_state {mask}"

    kin = engine.kinematic_state_raw(topo, table, q, qd, want_quats=True)
    for mask in shift_variants(2):
        for a, b in zip(engine.kinematic_state_raw(topo, table, *pick((q, qd), mask), want_quats=True), kin):
            assert torch.equal(a, b), f"kinematic_state {mask}"
    poses = engine.kinematic_state_raw(topo, table, q)[0]
    assert torch.equal(engine.kinematic_state_raw(topo, table, shifted(q))[0], poses)


@UNALIGNED
def test_unaligned_adjoints_are_bit_identical(stem, batch):
    """Adjoints through autograd with shifted leaves: the saved inputs keep their offset, so the backward kernels stage
    them with cooperative copies (vec_ok = 0)."""
    q, qd, qdd, f = seeded(stem, batch)
    n = q.shape[1]
    gen = torch.Generator().manual_seed(batch + 1)
    Gfk = [torch.randn(batch, *s, generator=gen).to(DEV) for s in ((3,), (4,), (3, n), (3, n))]
    G = torch.randn(batch, n, generator=gen).to(DEV)
    learn, params = learnable_model(stem)
    inert, iparams = inertial_model(stem)
    link = "iiwa_link_ee" if stem == "iiwa7" else "link_15.0_tip"

    def collect(ins, ps):
        out = [t.grad.clone() for t in ins if t.requires_grad]
        out += [p.grad.clone() if p.grad is not None else torch.zeros_like(p) for p in ps.values()]
        for p in ps.values():
            p.grad = None
        return out

    def fk(mask):
        (qq,) = [(shifted(q) if mask[0] else q.clone()).requires_grad_(True)]
        sum((g * o).sum() for g, o in zip(Gfk, learn.compute_fk_and_jacobian(qq, link))).backward()
        return collect([qq], params)

    def rnea(mask):
        ins = [(shifted(t) if s else t.clone()).requires_grad_(True) for t, s in zip((q, qd, qdd), mask)]
        (G * learn.compute_inverse_dynamics(*ins)).sum().backward()
        return collect(ins, params)

    def rnea_inertial(mask):
        ins = [shifted(t) if s else t.clone() for t, s in zip((q, qd, qdd), mask)]
        (G * inert.compute_inverse_dynamics(*ins)).sum().backward()
        return collect(ins, iparams)

    def aba(mask):
        ins = [(shifted(t) if s else t.clone()).requires_grad_(True) for t, s in zip((q, qd, f), mask)]
        (G * learn.compute_forward_dynamics(*ins, use_damping=True)).sum().backward()
        return collect(ins, params)

    for name, fn, k in (("fk", fk, 1), ("rnea", rnea, 3), ("rnea inertial", rnea_inertial, 3), ("aba", aba, 3)):
        want = fn((False,) * k)
        for mask in shift_variants(k):
            for i, (a, b) in enumerate(zip(fn(mask), want)):
                assert torch.equal(a, b), f"{name} {stem} B={batch} shifted={mask}: gradient {i} differs"
