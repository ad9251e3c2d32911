"""GPU: the PD-controlled rollout (pd_rollout_kernel and rollout_adjoint_step_kernel<true>, csrc/rollout.cu) on every
synthetic topology family of tests/synthetic_robots.py and at every launch geometry it can choose:

  1. a Python mirror of the kernel's shared-memory layout (PDRolloutSmem) and tile rule -- 64 rows when 64 fit in 113 KB
     and the batch gives every SM a 64-row CTA, else 32, else 16 when the 32-row CTA exceeds 227 KB -- pinned to the
     binary by the kernels' static shared memory and by the instantiation a profiled launch runs; a case per rung;
  2. forward against the fp64 oracle (tests/pd_rollout_oracle.py) on every runnable family: both gain layouts, one to
     three input streams, with and without a binding effort limit; the 0-DoF families and the refused models;
  3. bit-identity with the stepwise loop around compute_forward_dynamics at a ragged batch, a batch that takes
     cooperative copies and misaligned views of every input;
  4. gradients against autograd of the fp64 oracle on GRAD_FAMILIES, every input and every link parameter;
  5. the adjoint at 70 001 Kuka rows, where the feedback step kernel's grid-stride loop wraps and the ABA adjoint walks
     several tiles per CTA;
  6. gradient subsets: each input requiring grad alone gets, bit for bit, its gradient of the run that requests all eight,
     under every subset of upstream gradients, and a NULL upstream of the C ABI equals a zero one.

Tolerances are those of the modules whose helpers this one imports: check() bounds the kernel's family-relative error by
max(8 x the fp32 oracle's, 2e-5) and prints it (the ERR lines, pytest -s); the large-batch checks use
test_launch_geometry_gpu.py's.
"""
import ctypes
import re

import pytest
import torch

import differentiable_robot_model_b200 as drm
import synthetic_robots as S
from conftest import urdf_path
from differentiable_robot_model_b200 import engine
from oracle import drm_oracle as O
from pd_rollout_oracle import pd_rollout
from test_backward_gpu import learnable_model, shifted
from test_launch_geometry_gpu import B_ABA, check_table_against_chunks, grads_of, report, run_in_chunks, sub_rows, tail_rows
from test_pd_rollout_gpu import pd_inputs, stepwise
from test_rollout_gpu import bits, family_close
from test_synthetic_topologies_gpu import (FAM, GRAD_FAMILIES, REFUSALS, RUNNABLE, check, check_grads, get,
                                           learnable_model_at, oracle_mass_matrix)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = 2.0 ** -10
FLAGS = engine.GRAVITY | engine.DAMPING
KEYS = ("q", "qd", "qdd", "tau")


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_pd_rollout"))


def n_dofs(name):
    return sum(FAM[name].doc()[1][1:])


MOVING = [name for name in RUNNABLE if n_dofs(name) > 0]
ZERO_DOF = [name for name in RUNNABLE if n_dofs(name) == 0]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the launch choice
# ---------------------------------------------------------------------------------------------------------------------
TWO_CTAS = 113 * 1024          # SMEM_TWO_CTAS
SMEM_CAP = 227 * 1024          # SMEM_CTA_MAX
STATIC_SMEM = 128              # the PD kernel's static shared memory at every tile, what -Xptxas -v reports
TABLE_STRIDE, ABA_LINK, ABA_SLOT = 28, 14, 42


def up4(x):
    return (x + 3) & ~3


def program(M):
    """(n, n_links, n_slots) of the tree program the rollouts run: the folded tree when the model is foldable."""
    return (M.n, 1 + M.n, M.red_slots) if M.foldable else (M.n, M.N, M.slots)


def pd_floats(T, n, n_links, n_slots, n_in, per_row):
    """PDRolloutSmem(T, n, n_links, n_slots, n_in, per_row).total_floats."""
    gain = up4((T if per_row else 1) * n)
    return (2 * T * n + 2 * n_in * T * n + 4 * T * n + 2 * gain + up4(n) + n_links * TABLE_STRIDE + n_links * ABA_LINK * T
            + n_slots * ABA_SLOT * T)


def open_loop_floats(T, n, n_links, n_slots):
    """RolloutSmem(T, n, n_links, n_slots).total_floats."""
    return 6 * T * n + n_links * TABLE_STRIDE + n_links * ABA_LINK * T + n_slots * ABA_SLOT * T


def pd_tile(prog, batch, n_in, per_row, sms):
    """launch_rollout's choice for pd_rollout_device: (tile, dynamic + static bytes); tile None = ELIMIT."""
    def need(T):
        return 4 * pd_floats(T, *prog, n_in, per_row)
    T = 64 if -(-batch // 64) >= sms and need(64) <= TWO_CTAS else 32
    if need(T) + STATIC_SMEM > SMEM_CAP:
        T = 16
    return (T if need(T) + STATIC_SMEM <= SMEM_CAP else None), need(T) + STATIC_SMEM


def sm_count():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def n_in_of(x):
    return 1 + (x["qd_ref"] is not None) + (x["f"] is not None)


def test_static_shared_memory_is_what_the_mirror_adds():
    lib = engine.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    for t in (64, 32, 16):
        sym = f"_ZN3drm17pd_rollout_kernelILi{t}EEEvNS_11TreeProgramENS_11FoldProgramENS_13PDRolloutArgsE"
        attr = (ctypes.c_size_t * 64)()
        assert cudart.cudaFuncGetAttributes(attr, ctypes.cast(getattr(lib, sym), ctypes.c_void_p)) == 0, sym
        assert attr[0] == STATIC_SMEM, (sym, attr[0])


def test_the_mirror_reaches_every_rung_and_refuses_nothing(model_dir):
    sms = sm_count()
    small = {}
    for name in MOVING:
        M = get(name, model_dir)
        prog = program(M)
        # the open-loop rollout never needs a third rung: its 32-row CTA fits every family
        assert 4 * open_loop_floats(32, *prog) + STATIC_SMEM <= SMEM_CAP, name
        for per_row in (False, True):
            for n_in in (1, 2, 3):
                tile, need = pd_tile(prog, 67, n_in, per_row, sms)
                assert tile is not None, (name, per_row, n_in, need)
                small[(name, per_row, n_in)] = tile
    print("16-row rung:", sorted(k for k, t in small.items() if t == 16))
    assert set(small.values()) == {32, 16}
    assert small[("F_chain64", True, 3)] == 16
    # the example of DESIGN.md: 235 008 B at 32 rows, 121 216 B at 16
    assert 4 * pd_floats(32, 63, 64, 0, 3, True) == 235008 and 4 * pd_floats(16, 63, 64, 0, 3, True) == 121216
    assert pd_tile(program(get("D_fixed", model_dir)), 64 * sms, 1, False, sms)[0] == 64
    assert pd_tile(program(get("D_fixed", model_dir)), 64 * sms - 64, 1, False, sms)[0] == 32


def launched_tiles(fn):
    """The template tiles of the pd_rollout_kernel instantiations fn launches (torch.profiler kernel names)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tiles = set()
    for e in prof.events():
        m = re.search(r"pd_rollout_kernel<(\d+)>|pd_rollout_kernelILi(\d+)E", e.name)
        if m:
            tiles.add(int(m.group(1) or m.group(2)))
    return tiles


# rung -> (family, gains per row, qd_ref and f given, batch; None: 64 rows for every SM plus a ragged row)
RUNGS = {64: ("D_fixed", False, False, None), 32: ("D_fixed", True, True, 67), 16: ("F_chain64", True, True, 67)}


@pytest.mark.parametrize("rung", sorted(RUNGS))
def test_every_rung_runs_the_mirror_tile_and_matches_the_stepwise_loop(rung, model_dir):
    name, per_row, streams, batch = RUNGS[rung]
    M = get(name, model_dir)
    batch = batch or 64 * sm_count() + 1
    x = select(family_inputs(M, batch, 5, seed=rung), per_row, streams, streams, True)
    assert pd_tile(program(M), batch, n_in_of(x), per_row, sm_count())[0] == rung
    with torch.no_grad():
        got = []
        assert launched_tiles(lambda: got.append(model_call(M.m, x))) == {rung}
        want = model_loop(M.m, x)
    for k, a, b in zip(KEYS, got[0], want):
        assert torch.equal(bits(a), bits(b)), (name, rung, k)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
W = 20.0


def family_inputs(M, rows, T, seed):
    """fp32 values on the device: (q0, qd0) as the topology tests sample them, q_ref near q0, small qd_ref, unit f; per-row
    gains kp = W^2 m_k, kd = 2 W m_k with m_k = 1 / (H(q0)^-1)_kk the inertia joint k sees with every other joint free (the
    diagonal H_kk overstates it along a long chain, and explicit Euler then diverges within the steps); a limit at the 70th
    percentile of |u| over the rows at step 0, so that it binds for about a third of the entries, inf on joint 0."""
    q, qd, _ = O.sample_inputs(M.r64, rows, seed=seed, dtype=torch.float32)
    n = M.n
    gen = torch.Generator().manual_seed(seed)
    q_ref = q + 0.1 * torch.randn(T, rows, n, generator=gen)
    qd_ref = 0.2 * torch.randn(T, rows, n, generator=gen)
    f = torch.randn(T, rows, n, generator=gen)
    m_eff = (1.0 / torch.diagonal(torch.linalg.inv(oracle_mass_matrix(M.r64, q.double())), dim1=1, dim2=2)).float()
    kp, kd = (W * W) * m_eff, (2 * W) * m_eff
    lim = torch.quantile((f[0] + kp * (q_ref[0] - q) + kd * (qd_ref[0] - qd)).abs(), 0.7, dim=0)
    lim[0] = float("inf")
    x = dict(q0=q, qd0=qd, q_ref=q_ref, qd_ref=qd_ref, f=f, kp=kp, kd=kd, lim=lim)
    return {k: v.to(DEV) for k, v in x.items()}


def select(x, per_row, has_qdr, has_f, has_lim):
    """x with shared gains (the mean over rows) or per-row ones, and qd_ref / f / the limit present or None."""
    return dict(x, kp=x["kp"] if per_row else x["kp"].mean(0), kd=x["kd"] if per_row else x["kd"].mean(0),
                qd_ref=x["qd_ref"] if has_qdr else None, f=x["f"] if has_f else None, lim=x["lim"] if has_lim else None)


def rows_of(x, B):
    """The first B rows of every input."""
    per_row = x["kp"].ndim == 2
    out = dict(x, q0=x["q0"][:B], qd0=x["qd0"][:B], q_ref=x["q_ref"][:, :B].contiguous())
    for k in ("qd_ref", "f"):
        out[k] = None if x[k] is None else x[k][:, :B].contiguous()
    if per_row:
        out["kp"], out["kd"] = x["kp"][:B], x["kd"][:B]
    return out


def raw_call(M, x):
    return engine.pd_rollout_raw(M.topo, M.table, x["q0"], x["qd0"], x["q_ref"], x["kp"], x["kd"], DT, FLAGS, x["qd_ref"],
                                 x["f"], x["lim"])


def model_call(m, x):
    return m.compute_pd_controlled_rollout(x["q0"], x["qd0"], x["q_ref"], x["kp"], x["kd"], DT, qd_ref=x["qd_ref"], f=x["f"],
                                           effort_limit=x["lim"], include_gravity=True, use_damping=True)


def model_loop(m, x):
    return stepwise(m, x["q0"], x["qd0"], x["q_ref"], x["kp"], x["kd"], DT, x["qd_ref"], x["f"], x["lim"], True, True)


def oracle(robot, x):
    """The oracle's trajectory from x (device or host tensors) in the robot's dtype; differentiable in host inputs of that
    dtype."""
    dtype = robot.trans.dtype
    c = {k: (None if v is None else v.cpu().to(dtype)) for k, v in x.items()}
    return pd_rollout(robot, c["q0"], c["qd0"], c["q_ref"], c["kp"], c["kd"], DT, c["qd_ref"], c["f"], c["lim"], True, True)


# (gains per row, qd_ref given, f given, effort limit): both gain layouts, one to three input streams, limit on and off
CONFIGS = {"shared-1": (False, False, False, False), "row-2-qdref": (True, True, False, False),
           "shared-2-f-lim": (False, False, True, True), "row-3-lim": (True, True, True, True)}


# ---------------------------------------------------------------------------------------------------------------------
# 2. forward against the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MOVING)
def test_pd_rollout_matches_the_oracle(name, model_dir):
    M = get(name, model_dir)
    T, rows = 5, 67
    full = family_inputs(M, rows, T, seed=5)
    for tag, cfg in CONFIGS.items():
        x = select(full, *cfg)
        got = raw_call(M, x)
        o64, o32 = oracle(M.r64, x), oracle(M.r32, x)
        for k, key in enumerate(KEYS):
            check(f"{name} pd {tag} {key}", got[k], o64[k], o32[k])
        if x["lim"] is not None:
            # rows where fp32 and fp64 put u on different sides of the limit would differ by a whole clamp: there are none
            lim = x["lim"].cpu()
            clamped = got[3].cpu().abs() == lim
            if M.n > 1:                  # joint 0's limit is inf
                assert bool(clamped.any()), f"{name} {tag}: the limit should bind on some entries"
            assert torch.equal(clamped, o64[3].abs() == lim.double()), f"{name} {tag}: fp32 and fp64 clamp different entries"


@pytest.mark.parametrize("name", ZERO_DOF)
def test_zero_dof_models_return_empty_trajectories_and_zero_gradients(name, model_dir):
    M = get(name, model_dir)
    m, params = learnable_model_at(M.path, M.r32)
    T, B = 3, 5
    for per_row in (False, True):
        x = dict(q0=torch.zeros(B, 0, device=DEV), qd0=torch.zeros(B, 0, device=DEV), q_ref=torch.zeros(T, B, 0, device=DEV),
                 qd_ref=torch.zeros(T, B, 0, device=DEV), f=torch.zeros(T, B, 0, device=DEV),
                 kp=torch.zeros((B, 0) if per_row else (0,), device=DEV), kd=torch.zeros((B, 0) if per_row else (0,), device=DEV),
                 lim=torch.ones(0, device=DEV))
        for out in (raw_call(M, x), model_call(M.m, x)):
            assert all(o.shape == (T, B, 0) for o in out), [tuple(o.shape) for o in out]
        leaves = {k: (v.clone().requires_grad_(True) if k != "lim" else v) for k, v in x.items()}
        for p in params.values():
            p.grad = None
        out = model_call(m, leaves)
        sum(o.sum() for o in out).backward()
        for k, v in leaves.items():
            if k != "lim":
                assert v.grad is not None and v.grad.shape == v.shape, k
        for key, p in params.items():
            assert p.grad is None or not bool(p.grad.any()), (name, key)


def test_refused_models_are_refused_before_any_launch(model_dir):
    specs = S.refusal_families()
    path = S.build(specs["H_nine_slots"], model_dir)
    m = drm.DifferentiableRobotModel(path, "H_nine_slots", device=DEV)
    n = m._n_dofs
    z = torch.zeros(5, n, device=DEV)
    m._link_table()
    m._folded_table()
    exc, pattern = REFUSALS[("H_nine_slots", "rollout")]
    for kp in (z[0], z):
        before = engine.launch_count()
        with pytest.raises(exc, match=pattern):
            m.compute_pd_controlled_rollout(z, z, z.expand(3, 5, n).contiguous(), kp, kp, 1e-3)
        assert engine.launch_count() == before
    exc, pattern = REFUSALS[("H_65_links", "construct")]
    with pytest.raises(exc, match=pattern):
        drm.DifferentiableRobotModel(S.build(specs["H_65_links"], model_dir), "H_65_links", device=DEV)


# ---------------------------------------------------------------------------------------------------------------------
# 3. bit-identity with the stepwise loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MOVING)
def test_pd_rollout_is_bit_identical_to_the_stepwise_loop(name, model_dir):
    M = get(name, model_dir)
    sms = sm_count()
    T = 5
    full = family_inputs(M, 72, T, seed=6)
    for tag, cfg in CONFIGS.items():
        x = select(full, *cfg)
        tile = pd_tile(program(M), 64, n_in_of(x), cfg[0], sms)[0]
        batches = {"ragged": tile + 1, "aligned": 2 * tile}
        coop = next((b for b in range(tile + 2, tile + 6) if b * M.n % 4), None)     # B n % 4 != 0: cooperative copies
        if coop is not None:
            batches["coop"] = coop
        with torch.no_grad():
            for what, B in batches.items():
                xb = rows_of(x, B)
                got, want = model_call(M.m, xb), model_loop(M.m, xb)
                for k, a, b in zip(KEYS, got, want):
                    assert torch.equal(bits(a), bits(b)), (name, tag, what, B, k)
            if tag == "row-3-lim":       # every input present: each one on its own 4 bytes off 16-byte alignment
                xb = rows_of(x, 2 * tile)
                want = model_call(M.m, xb)
                for k in ("q0", "qd0", "q_ref", "qd_ref", "f", "kp", "kd", "lim"):
                    got = model_call(M.m, dict(xb, **{k: shifted(xb[k])}))
                    for key, a, b in zip(KEYS, got, want):
                        assert torch.equal(bits(a), bits(b)), (name, "shifted", k, key)


# ---------------------------------------------------------------------------------------------------------------------
# 4. gradients against autograd of the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
# per-row gains on some families, shared on others; F_chain64 per row with every stream takes the 16-row rung
GRAD_PER_ROW = {"A_bfs_fixed_palm": False, "A_bfs_movable_palm": True, "C_random": False, "D_fixed": True,
                "E_unfoldable": False, "F_chain64": True, "F_tree64": False, "G_one_joint": True}
DIFF = ("q0", "qd0", "q_ref", "qd_ref", "f", "kp", "kd")


@pytest.mark.parametrize("name", GRAD_FAMILIES)
def test_pd_rollout_gradients_match_oracle_autograd(name, model_dir):
    M = get(name, model_dir)
    T, rows = 4, 33
    per_row = GRAD_PER_ROW[name]
    x = select(family_inputs(M, rows, T, seed=10), per_row, True, True, True)
    if name == "F_chain64":
        assert pd_tile(program(M), rows, 3, True, sm_count())[0] == 16
    gen = torch.Generator().manual_seed(10)
    G = [torch.randn(T, rows, M.n, generator=gen) for _ in KEYS]
    lim = x["lim"].cpu()

    def run(m, *ins):
        a = dict(zip(DIFF, ins), lim=x["lim"])
        return sum((g.to(DEV) * o).sum() for g, o in zip(G, model_call(m, a)))

    def loss(rb, *ins):
        a = dict(zip(DIFF, ins), lim=lim.to(ins[0].dtype))
        return sum((g.to(ins[0].dtype) * o).sum() for g, o in zip(G, oracle(rb, a)))

    check_grads(f"{name} pd rollout grad ({'per-row' if per_row else 'shared'} gains)", M, run, loss,
                [x[k].cpu() for k in DIFF])


# ---------------------------------------------------------------------------------------------------------------------
# 5. the adjoint at scale
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_row", [True, False], ids=["row", "shared"])
def test_pd_adjoint_with_several_tiles_per_cta(per_row):
    """B_ABA = 70 001 rows x 7 DoF = 490 007 elements per step: more than the 8 x 132 blocks of 256 threads of the step
    kernel cover, so its grid-stride loop wraps; the ABA adjoint walks several tiles per CTA and sums its per-CTA partial
    tables over the steps before one reduction."""
    stem, B, T = "iiwa7", B_ABA, 3
    assert B * 7 > 8 * sm_count() * 256
    m, params = learnable_model(stem)
    x = pd_inputs(m, stem, B, T, seed=26)
    gen = torch.Generator().manual_seed(26)
    G = [torch.randn(T, B, 7, generator=gen).to(DEV) for _ in KEYS]
    row_keys = ("q0", "qd0") + (("kp", "kd") if per_row else ())
    step_keys = ("q_ref", "qd_ref", "f")
    gains = {} if per_row else {k: x[k].mean(0).clone().requires_grad_(True) for k in ("kp", "kd")}
    tracked = dict(params)
    tracked.update({(-1, k): v for k, v in gains.items()})                 # shared gains: summed over chunks like the table
    taus = []

    def run(rows):
        ins = {k: x[k][rows].clone().requires_grad_(True) for k in row_keys}
        ins.update({k: x[k][:, rows].clone().requires_grad_(True) for k in step_keys})
        out = model_call(m, dict(ins, lim=x["lim"], **gains))
        taus.append(out.tau.detach())
        sum((g[:, rows] * o).sum() for g, o in zip(G, out)).backward()
        return {k: v.grad for k, v in ins.items()}

    big_in = run(slice(None))
    tau = taus[0]
    big = grads_of(tracked)
    idx = sub_rows(B, gen).to(DEV)
    for p in tracked.values():
        p.grad = None
    sub_in = run(idx)
    for k in row_keys:
        assert torch.equal(big_in[k][idx], sub_in[k]), f"{k}_grad rows differ between the big batch and a sub-batch"
    for k in step_keys:
        assert torch.equal(big_in[k][:, idx], sub_in[k]), f"{k}_grad rows differ between the big batch and a sub-batch"
    check_table_against_chunks(f"pd rollout iiwa7 {'row' if per_row else 'shared'} gains", big, run_in_chunks(B, run, tracked))

    rows = tail_rows(B, gen).to(DEV)
    rb = O.load_robot(urdf_path(stem), torch.float64)
    ins = {k: x[k][rows].cpu().double().requires_grad_(True) for k in row_keys}
    ins.update({k: x[k][:, rows].cpu().double().requires_grad_(True) for k in step_keys})
    ins.update({k: v.detach().cpu().double() for k, v in gains.items()})
    lim = x["lim"].cpu().double()
    traj = pd_rollout(rb, ins["q0"], ins["qd0"], ins["q_ref"], ins["kp"], ins["kd"], DT, ins["qd_ref"], ins["f"], lim, True, True)
    assert torch.equal(tau[:, rows].cpu().abs() == x["lim"].cpu(), traj[3].abs() == lim), "fp32 and fp64 clamp different entries"
    names = row_keys + step_keys
    want = torch.autograd.grad(sum((g[:, rows].cpu().double() * o).sum() for g, o in zip(G, traj)), [ins[k] for k in names])
    for k, w in zip(names, want):
        a = (big_in[k][rows] if k in row_keys else big_in[k][:, rows]).cpu().numpy()
        err = family_close(a, w.numpy(), 1e-4, f"pd rollout d{k} (later tiles)")
        report(f"pd rollout {stem} {k}_grad vs oracle (family-relative)", err)


# ---------------------------------------------------------------------------------------------------------------------
# 6. gradient subsets
# ---------------------------------------------------------------------------------------------------------------------
INPUTS = ("table", "q0", "qd0", "q_ref", "qd_ref", "f", "kp", "kd")
SUBSET_FLAGS = engine.GRAVITY      # without damping: explicit in qd, it makes the Allegro fingers diverge at this step
UPSTREAMS = ["q", "qd", "qdd", "tau", "last_step", "all"]


def upstream(kind, shape, seed):
    gen = torch.Generator().manual_seed(seed)
    G = [torch.randn(shape, generator=gen).to(DEV) for _ in KEYS]
    if kind in KEYS:
        G = [g if k == kind else None for k, g in zip(KEYS, G)]
    elif kind == "last_step":
        for g in G:
            g[:-1] = 0
    return G


def function_grads(m, x, wanted, G):
    """Gradients of sum(G * outputs) through engine.PDRolloutFunction with only `wanted` of INPUTS requiring grad; None for
    the others.  A None upstream leaves its output out of the loss."""
    leaves = {k: (x[k].detach().clone().requires_grad_(True) if k in wanted else x[k]) for k in INPUTS}
    out = engine.PDRolloutFunction.apply(*(leaves[k] for k in INPUTS), m._topology, SUBSET_FLAGS, DT, x["lim"])
    sum((g * o).sum() for g, o in zip(G, out) if g is not None).backward()
    return {k: leaves[k].grad for k in INPUTS}


def raw_adjoint(m, x, g):
    """drmb200_pd_rollout_backward called directly, so that upstream gradients can be NULL (autograd hands the Function
    materialised zeros instead).  Every output starts as NaN: one the adjoint does not write shows."""
    topo, table = m._topology, x["table"]
    per_row = x["kp"].ndim == 2
    q, qd, _, tau = engine.pd_rollout_raw(topo, table, x["q0"], x["qd0"], x["q_ref"], x["kp"], x["kd"], DT, SUBSET_FLAGS,
                                          x["qd_ref"], x["f"], x["lim"])
    T, B, n = x["q_ref"].shape
    nan = float("nan")
    outs = [torch.full((B, n), nan, device=DEV), torch.full((B, n), nan, device=DEV)] + \
           [torch.full((T, B, n), nan, device=DEV) for _ in range(3)] + \
           [torch.full((B, n), nan, device=DEV), torch.full((B, n), nan, device=DEV), torch.zeros_like(table)]
    nbytes = int(engine.lib().drmb200_pd_rollout_backward_workspace_bytes(ctypes.byref(topo), B))
    ws = torch.empty((max(nbytes, 4) + 3) // 4, device=DEV, dtype=torch.float32)
    p = engine._ptr
    rc = engine.lib().drmb200_pd_rollout_backward(
        ctypes.byref(topo), p(table), p(x["q0"]), p(x["qd0"]), p(x["q_ref"]), p(x["qd_ref"]), p(x["f"]), p(x["kp"]), p(x["kd"]),
        1 if per_row else 0, p(x["lim"]), B, T, ctypes.c_float(DT), SUBSET_FLAGS, p(q), p(qd), p(tau), *[p(t) for t in g],
        *[p(o) for o in outs], p(ws), engine._stream())
    engine._check(rc, "drmb200_pd_rollout_backward")
    return outs


@pytest.mark.parametrize("batch", [257, 1024])
@pytest.mark.parametrize("stem", ["iiwa7", "iiwa7_allegro"])
def test_pd_rollout_gradient_subsets(stem, batch):
    m, _ = learnable_model(stem)
    T = 5
    base = pd_inputs(m, stem, batch, T, seed=batch + 3)
    base["table"] = m._link_table().detach().contiguous()
    for per_row in (True, False):
        x = dict(base) if per_row else dict(base, kp=base["kp"].mean(0), kd=base["kd"].mean(0))
        for kind in UPSTREAMS:
            G = upstream(kind, (T, batch, m._n_dofs), seed=batch + 11)
            full = function_grads(m, x, set(INPUTS), G)
            assert all(g is not None and bool(torch.isfinite(g).all()) for g in full.values()), (per_row, kind)
            for k in INPUTS:
                got = function_grads(m, x, {k}, G)
                assert torch.equal(got[k], full[k]), f"{stem} B={batch} per_row={per_row} upstream={kind}: {k} alone differs"
                assert all(got[j] is None for j in INPUTS if j != k)
        # NULL upstreams equal zero ones: each upstream alone, and none at all
        G = upstream("all", (T, batch, m._n_dofs), seed=batch + 12)
        for keep in [(0,), (1,), (2,), (3,), ()]:
            nulls = [G[i] if i in keep else None for i in range(4)]
            zeros = [G[i] if i in keep else torch.zeros_like(G[i]) for i in range(4)]
            a, b = raw_adjoint(m, x, nulls), raw_adjoint(m, x, zeros)
            for i, (u, v) in enumerate(zip(a, b)):
                assert bool(torch.isfinite(u).all()), (per_row, keep, i)
                assert torch.equal(u, v), (per_row, keep, i)
