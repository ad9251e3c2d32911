"""GPU: the contact adjoint (csrc/contact_backward.cu) where the other contact-adjoint suites do not look: the link-parameter
gradients and the impulse instantiations at every rung of both tile rules, the raw table gradient at the C ABI, and the
persistent kinematic kernel's tile loop when every CTA walks several tiles.

* Every rung (the cases of test_contact_backward_geometry_gpu.TILE_CASES, one per distinct family / link set, dynamics and
  impulse): every link parameter learnable on the non-symmetric-inertia families of test_synthetic_topologies_gpu, B =
  3T + 4 (at least 70) rows, upstream gradients only on the last 8 rows -- the last partial tile and the rows before it --
  and every input and link-parameter gradient against torch autograd of the fp64 oracle (tests/contact_grad_oracle.py).
  Rows past the batch in the last tile walk that tile's first row, which is one of the compared rows, so a padding row
  leaking into the table sum changes the compared gradients.  The walked paths of the cases reach all six axis codes, so
  every signed permutation canon_map applies in the kinematic write-back is exercised.
* The C ABI: the table gradient of B rows is the sum of those of three chunks split off the kinematic tile; two runs and a
  run with every pointer 4 bytes off 16-byte alignment give the same bits; table_grad is accumulated into; every subset of
  the outputs may be NULL (all NULL launches nothing) with the requested outputs unchanged bit for bit; rows with NaN q in
  a tile with solved rows and rows past the batch get zero gradients and leave the table gradient of the solved rows.
* The persistent loop: more than 2 x BWD_MAX_GRID kinematic tiles, so every CTA walks at least two tiles on any card --
  per-row gradients bit-identical to sub-batches', the table gradient against a sum over chunks, tail rows against the
  fp64 oracle.

Tolerances as in test_contact_backward_gpu.py: per gradient family (q, qd, f, the reference, each link-parameter kind),
relative to its largest fp64 entry, max(8 x the fp32 oracle's error, 1e-4), on rows whose fp64 scaled pivot is at least
100 x the threshold; every other row gets zero upstream gradient."""
import ctypes
import itertools
import types

import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from conftest import urdf_path
import contact_grad_oracle as CG
import contact_oracle as C
import test_contact_backward_geometry_gpu as G
import test_contact_backward_gpu as CB
import test_synthetic_topologies_gpu as SY
import tile_mirrors as TM
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BWD_MAX_GRID = 132 * 8          # csrc/backward_common.cuh: the most CTAs a persistent adjoint kernel launches
FLAGS = engine.GRAVITY | engine.DAMPING
TAIL = 8                        # rows compared with the fp64 oracle: the last ones of the batch


def _cases():
    """One case per distinct (family, links, pose) of TILE_CASES, with the rungs it stands for."""
    by = {}
    for key, (name, links, pose) in sorted(G.TILE_CASES.items()):
        by.setdefault((name, tuple(links), pose), []).append(key)
    return [(name, links, pose, keys) for (name, links, pose), keys in by.items()]


CASES = _cases()
CASE_IDS = [f"{name}-" + "-".join(f"{s[0]}{t}" for s, t in keys) for name, _, _, keys in CASES]


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("contact_backward_coverage"))


def robot(name, model_dir):
    """A synthetic family (test_synthetic_topologies_gpu.Model: non-symmetric inertias) or a shipped robot, with the
    fields the tests use: path, r32, r64, topo, table."""
    if name in SY.FAM:
        return SY.get(name, model_dir)
    path = urdf_path(name)
    r32 = O.load_robot(path, torch.float32)
    return types.SimpleNamespace(path=path, r32=r32, r64=r32.to(torch.float64),
                                 topo=drm.DifferentiableRobotModel(path, name, device=DEV)._topology,
                                 table=O.link_table(r32).float().to(DEV).contiguous())


def tree(R):
    """(parents, movable) of the model in table order."""
    t = R.topo
    return [int(t.parent[i]) for i in range(t.n_links)], [int(t.axis[i]) != 0 for i in range(t.n_links)]


def path_axes(R, links):
    """Axis codes of the movable joints on the root -> link paths."""
    codes = set()
    for l in links:
        while l > 0:
            if R.topo.axis[l]:
                codes.add(int(R.topo.axis[l]))
            l = int(R.topo.parent[l])
    return codes


def conditioned(R, impulse, x, lnames, links, pos):
    """mu as the other contact-adjoint tests choose it (1e-3 max A_kk, 0.1 max A_kk for a redundant set) from the rows x,
    and which of them the fp64 oracle solves with a scaled pivot of at least 100 x the threshold."""
    q, qd, f, ref = (t.double() for t in x)
    par, mov = tree(R)
    _, n_u, _, _ = TM.multi_program(par, mov, list(links))
    M = ref.shape[1]
    J = C.S.stacked_jacobian(R.r64, q, lnames, pos)
    Gm = C.S.force_response(R.r64, q)
    mu = (1e-3 if M <= n_u else 1e-1) * float(torch.diagonal(J @ Gm @ J.transpose(1, 2), dim1=1, dim2=2).max())
    if impulse:
        _, _, ok64, piv = C.contact_impulse(R.r64, q, qd, lnames, ref, pos, mu)
    else:
        _, _, ok64, piv = C.contact_dynamics(R.r64, q, qd, f, lnames, ref, True, True, pos, mu)
    return mu, ok64 & (piv >= 100 * C.PIVOT_MIN)


def forward(R, impulse, links, x, pos, mu):
    q, qd, f, ref = x
    if impulse:
        return engine.contact_impulse_raw(R.topo, links, R.table, q, qd, ref, pos, mu)
    return engine.contact_dynamics_raw(R.topo, links, R.table, q, qd, f, FLAGS, ref, pos, mu)


ALL = ("q", "qd", "f", "ref", "table")


def abi(R, impulse, links, pos, mu, x, fwd, g, want=ALL, table_pre=None, misaligned=False):
    """drmb200_contact_dynamics_backward / drmb200_contact_impulse_backward with caller-allocated outputs (NaN-filled, so
    an entry the kernels never write shows); an output not in `want` is NULL.  table_grad starts as zeros or table_pre.
    A generalisation of test_contact_backward_geometry_gpu.backward_call to the impulse, NULL outputs and the table."""
    q, qd, f, ref = x
    out, lam, solved = fwd
    B, n = q.shape
    M = lam.shape[1]
    shapes = {"q": (B, n), "qd": (B, n), "f": (B, n), "ref": (B, M)}
    outs = {k: torch.full(s, float("nan"), device=DEV) if k in want and not (impulse and k == "f") else None
            for k, s in shapes.items()}
    outs["table"] = None if "table" not in want else (torch.zeros_like(R.table) if table_pre is None else table_pre.clone())
    ins = [q, qd, f, ref, out, lam, solved.contiguous().view(torch.uint8), g[0], g[1]]
    if misaligned:
        ins = [G.shifted(t) for t in ins]
        outs = {k: G.shifted(t) for k, t in outs.items()}
    q, qd, f, ref, out, lam, sv, g_out, g_lam = (G.ptr(t) for t in ins)
    o = {k: G.ptr(t) for k, t in outs.items()}
    idx = (ctypes.c_int32 * len(links))(*links)
    lib = engine.lib()
    nbytes = int(lib.drmb200_contact_backward_workspace_bytes(ctypes.byref(R.topo), len(links), idx, int(pos), B))
    ws = torch.empty((nbytes + 3) // 4 + 1, device=DEV)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if impulse:
        rc = lib.drmb200_contact_impulse_backward(ctypes.byref(R.topo), len(links), idx, G.ptr(R.table), q, qd, ref, out, lam,
                                                  sv, B, int(pos), ctypes.c_float(mu), g_out, g_lam, o["q"], o["qd"],
                                                  o["ref"], o["table"], G.ptr(ws), s)
    else:
        rc = lib.drmb200_contact_dynamics_backward(ctypes.byref(R.topo), len(links), idx, G.ptr(R.table), q, qd, f, ref, out,
                                                   lam, sv, B, FLAGS, int(pos), ctypes.c_float(mu), g_out, g_lam, o["q"],
                                                   o["qd"], o["f"], o["ref"], o["table"], G.ptr(ws), s)
    assert rc == 0, lib.drmb200_last_error()
    return {k: t.clone() for k, t in outs.items() if t is not None}


def bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def rows_of(d, a, b):
    return {k: t[a:b] for k, t in d.items() if k != "table"}


def table_error(got, want):
    """max |got - want| relative to the largest entry of want (fp64)."""
    got, want = got.double().cpu(), want.double().cpu()
    return float((got - want).abs().max()) / max(float(want.abs().max()), 1e-30)


# ------------------------------------------------------------------------------------------------
# the fp64 oracle: input and link-parameter gradients
# ------------------------------------------------------------------------------------------------
def oracle(r, impulse, x, g, lnames, pos, mu, ok):
    """(input gradients [q, qd, f, ref], {robot field: gradient}) of autograd of the oracle `r` (its dtype)."""
    dt = r.trans.dtype

    def loss(rb, q, qd, f, ref):
        if impulse:
            out, lam = CG.impulse(rb, q, qd, lnames, ref, pos, mu, ok=ok)
        else:
            out, lam = CG.dynamics(rb, q, qd, f, lnames, ref, True, True, pos, mu, ok=ok)
        return (g[0].to(dt) * out).sum() + (g[1].to(dt) * lam).sum()
    return SY.oracle_grads(r, loss, [t.to(dt) for t in x])


def compare_with_oracle(what, R, impulse, got_in, params, x, g, lnames, pos, mu, ok):
    """Every input and link-parameter family against the fp64 oracle on the rows `ok` of x; returns the worst err / bound."""
    w64, by64 = oracle(R.r64, impulse, x, g, lnames, pos, mu, ok)
    w32, by32 = oracle(R.r32, impulse, x, g, lnames, pos, mu, ok)
    fams = [(nm, got_in[j][ok], w64[j][ok], w32[j][ok]) for j, nm in enumerate(("q", "qd", "f", "ref"))
            if not (impulse and nm == "f")]
    for pname, field in SY.ORACLE_PARAM.items():
        idx = sorted(i for (i, p) in params if p == pname)
        got = torch.stack([torch.zeros_like(params[(i, pname)]) if params[(i, pname)].grad is None else params[(i, pname)].grad
                           for i in idx]).reshape(len(idx), -1)
        fams.append((pname, got, by64[field][idx].reshape(len(idx), -1), by32[field][idx].reshape(len(idx), -1)))
    worst = 0.0
    for nm, got, want64, want32 in fams:
        if float(want64.abs().max()) == 0.0:         # joint damping of the impulse: no dependence at all
            assert float(got.abs().max()) == 0.0, f"{what} {nm}: non-zero gradient of a parameter the output ignores"
            continue
        e32 = CB.family_error(want32, want64)
        err = CB.family_error(got, want64)
        bound = max(8 * e32, 1e-4)
        worst = max(worst, err / bound)
        print(f"ERR {what} {nm}: {err:.2e} (bound {bound:.2e})")
        assert err <= bound, f"{what} {nm}: {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"
    return worst


def model_gradients(R, impulse, lnames, x, g, pos, mu):
    """Input and link-parameter gradients through compute_contact_dynamics / compute_contact_impulse(differentiable=True)
    with every link parameter learnable."""
    m, params = SY.learnable_model_at(R.path, R.r32)
    xs = [t.to(DEV).clone().requires_grad_(not (impulse and k == 2)) for k, t in enumerate(x)]
    if impulse:
        out, lam, solved = m.compute_contact_impulse(xs[0], xs[1], lnames, velocity_ref=xs[3], position_only=pos,
                                                     regularization=mu, differentiable=True)
    else:
        out, lam, solved = m.compute_contact_dynamics(xs[0], xs[1], xs[2], lnames, accel_ref=xs[3], include_gravity=True,
                                                      use_damping=True, position_only=pos, regularization=mu,
                                                      differentiable=True)
    torch.autograd.backward([out, lam], [g[0].to(DEV), g[1].to(DEV)])
    grads = [torch.zeros_like(t) if t.grad is None else t.grad for t in xs]
    return [t.cpu() for t in grads], params, solved.cpu()


def tail_check(what, R, impulse, links, pose, B, seed):
    """Upstream gradients on the last TAIL rows only (those the fp64 oracle solves well), every link parameter learnable:
    input gradients of those rows and every link-parameter family against the oracle, exactly zero input gradients on
    every other row."""
    pos = not pose
    lnames = [R.r32.names[l] for l in links]
    M = (3 if pos else 6) * len(links)
    q, qd, f, ref, g_out, g_lam = CB.inputs(R.r32, B, M, seed)
    x = [q, qd, f, ref]
    tail = torch.arange(B - TAIL, B)
    mu, good = conditioned(R, impulse, [t[tail] for t in x], lnames, links, pos)
    sel = torch.zeros(B, dtype=torch.bool)
    sel[tail] = good
    g = [g_out * sel[:, None], g_lam * sel[:, None]]
    got, params, solved = model_gradients(R, impulse, lnames, x, g, pos, mu)
    assert bool(solved[sel].all()), f"{what}: the kernel leaves well-conditioned rows unsolved"
    assert int(sel.sum()) >= 2, f"{what}: only {int(sel.sum())} well-conditioned tail rows"
    for k, t in enumerate(got):
        assert bool((t[~sel] == 0).all()), f"{what}: input {k} has gradients on rows with zero upstream"
    worst = compare_with_oracle(what, R, impulse, [t[tail] for t in got], params, [t[tail] for t in x],
                                [t[tail] for t in g], lnames, pos, mu, good)
    print(f"WORST {what}: {worst:.2f} of the bound")


# ------------------------------------------------------------------------------------------------
# A. link-parameter and input gradients at every rung, dynamics and impulse
# ------------------------------------------------------------------------------------------------
def case_setup(case, model_dir):
    name, links, pose, keys = case
    R = robot(name, model_dir)
    par, mov = tree(R)
    (t1, _), (t3, _) = G.choices(par, mov, list(links), pose)
    for stage, t in keys:
        assert t == (t1 if stage == "stage1" else t3), (name, stage, t, t1, t3)
    return R, list(links), pose, t1, t3, max(3 * max(t1, t3) + 4, 70)


@pytest.mark.parametrize("impulse", [False, True], ids=["dynamics", "impulse"])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_every_rung_gradients_of_the_tail_rows_match_fp64_oracle(case, impulse, model_dir):
    R, links, pose, t1, t3, B = case_setup(case, model_dir)
    tail_check(f"{case[0]} T1={t1} T3={t3} {'impulse' if impulse else 'dynamics'}", R, impulse, links, pose, B, 23)


def test_walked_paths_reach_every_axis_code(model_dir):
    """The kinematic write-back maps each link's 12 (F, r) entries back through canon_map(parent axis, axis): the cases
    must walk joints of all six axis codes for every signed permutation to be checked."""
    codes = set()
    for case in CASES:
        codes |= path_axes(robot(case[0], model_dir), case[1])
    assert codes == {-3, -2, -1, 1, 2, 3}, sorted(codes)


# ------------------------------------------------------------------------------------------------
# B. the raw table gradient at the C ABI
# ------------------------------------------------------------------------------------------------
def abi_setup(R, impulse, links, pose, B, seed, nan_rows=()):
    pos = not pose
    lnames = [R.r32.names[l] for l in links]
    M = (3 if pos else 6) * len(links)
    q, qd, f, ref, g_out, g_lam = CB.inputs(R.r32, B, M, seed)
    tail = torch.arange(B - TAIL, B)
    mu, _ = conditioned(R, impulse, [t[tail] for t in (q, qd, f, ref)], lnames, links, pos)
    if len(nan_rows):
        q[list(nan_rows)] = float("nan")
    x = [t.to(DEV) for t in (q, qd, f, ref)]
    g = [g_out.to(DEV), g_lam.to(DEV)]
    return pos, mu, x, forward(R, impulse, links, x, pos, mu), g


def sub(x, fwd, g, a, b):
    return [t[a:b] for t in x], [t[a:b] for t in fwd], [t[a:b] for t in g]


@pytest.mark.parametrize("impulse", [False, True], ids=["dynamics", "impulse"])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_every_rung_table_gradient_at_the_c_abi(case, impulse, model_dir):
    R, links, pose, t1, t3, B = case_setup(case, model_dir)
    pos, mu, x, fwd, g = abi_setup(R, impulse, links, pose, B, 29)
    what = f"{case[0]} T1={t1} T3={t3}"
    full = abi(R, impulse, links, pos, mu, x, fwd, g)
    assert bool(torch.isfinite(full["table"]).all()) and float(full["table"].abs().max()) > 0, what
    # two runs, and every pointer 4 bytes off 16-byte alignment: the same bits
    for label, again in (("again", abi(R, impulse, links, pos, mu, x, fwd, g)),
                         ("misaligned", abi(R, impulse, links, pos, mu, x, fwd, g, misaligned=True))):
        for k in full:
            assert bits(again[k], full[k]), f"{what} {label}: {k} differs"
    # additivity over chunks cut across the kinematic tile: [0, T - 1), [T - 1, 2T + 1), [2T + 1, B)
    cuts = [0, t3 - 1, 2 * t3 + 1, B] if t3 > 1 else [0, 1, 3, B]
    parts = [abi(R, impulse, links, pos, mu, *sub(x, fwd, g, a, b)) for a, b in zip(cuts[:-1], cuts[1:])]
    err = table_error(sum(p["table"].double() for p in parts), full["table"])
    print(f"ERR {what} chunk sum: {err:.2e} (bound 1e-05)")
    assert err <= 1e-5, f"{what}: table gradient of the chunks {err:.3e} off the batch's"
    for (a, b), p in zip(zip(cuts[:-1], cuts[1:]), parts):
        for k, t in rows_of(full, a, b).items():
            assert bits(p[k], t), f"{what}: {k} rows [{a}, {b}) differ from the batch's"
    # table_grad is accumulated into: a preloaded table ends as preload + gradient (stage 2 and stage 3 each add their
    # sum, so the two roundings of preload + s2 + s3 differ by an ulp of the larger operand)
    gen = torch.Generator().manual_seed(5)
    pre = (torch.randn(R.table.shape, generator=gen) * float(full["table"].abs().max())).to(DEV)
    acc = abi(R, impulse, links, pos, mu, x, fwd, g, want=("table",), table_pre=pre)["table"]
    scale = float(pre.abs().max()) + float(full["table"].abs().max())
    assert float((acc.double() - pre.double() - full["table"].double()).abs().max()) <= 1e-6 * scale, what


def _null_cases():
    """A case whose kinematic tile is below one warp and one at a warp or more."""
    small = next(c for c in CASES if any(s == "kinematic" and t < 32 for s, t in c[3]))
    large = next(c for c in CASES if any(s == "kinematic" and t >= 32 for s, t in c[3]))
    return [small, large]


NULL_CASES = _null_cases()


@pytest.mark.parametrize("impulse", [False, True], ids=["dynamics", "impulse"])
@pytest.mark.parametrize("case", NULL_CASES, ids=[CASE_IDS[CASES.index(c)] for c in NULL_CASES])
def test_null_outputs_leave_the_requested_ones_unchanged(case, impulse, model_dir):
    R, links, pose, t1, t3, B = case_setup(case, model_dir)
    pos, mu, x, fwd, g = abi_setup(R, impulse, links, pose, B, 31)
    names = [k for k in ALL if not (impulse and k == "f")]
    full = abi(R, impulse, links, pos, mu, x, fwd, g)
    for r in range(len(names) + 1):
        for want in itertools.combinations(names, r):
            before = engine.launch_count()
            got = abi(R, impulse, links, pos, mu, x, fwd, g, want=want)
            if not want:
                assert engine.launch_count() == before, "a call with every output NULL launched kernels"
            assert set(got) == set(want), (want, sorted(got))
            for k in want:
                assert bits(got[k], full[k]), f"{case[0]} T3={t3} outputs {want}: {k} differs from the all-outputs run"


@pytest.mark.parametrize("impulse", [False, True], ids=["dynamics", "impulse"])
def test_unsolved_rows_in_a_small_tile_get_zero_gradients(impulse, model_dir):
    """NaN q on scattered rows and inside the last tile, which also holds solved rows and rows past the batch."""
    case = NULL_CASES[0]
    R, links, pose, t1, t3, _ = case_setup(case, model_dir)
    assert t3 < 32
    B = 8 * t3 + 5
    nan_rows = [3, 2 * t3 - 1, 2 * t3, B - 3, B - 2]
    pos, mu, x, fwd, g = abi_setup(R, impulse, links, pose, B, 37, nan_rows=nan_rows)
    bad = ~fwd[2].cpu()
    assert bool(bad[nan_rows].all()), "a row with NaN q is solved"
    last = torch.arange(B // t3 * t3, B)
    assert bool(bad[last].any()) and bool((~bad[last]).any()), "the last tile must mix solved and unsolved rows"
    got = abi(R, impulse, links, pos, mu, x, fwd, g)
    for k, t in got.items():
        if k == "table":
            continue
        assert bool((t.cpu()[bad] == 0).all()), f"{k}: unsolved rows get non-zero gradients"
        assert bool(torch.isfinite(t.cpu()[~bad]).all()), f"{k}: solved rows not finite"
    assert bool(torch.isfinite(got["table"]).all()), "table gradient poisoned by the unsolved rows"
    keep = (~bad).nonzero().flatten().to(DEV)
    alone = abi(R, impulse, links, pos, mu, [t[keep] for t in x], [t[keep] for t in fwd], [t[keep] for t in g])
    err = table_error(got["table"], alone["table"])
    print(f"ERR {case[0]} T3={t3} unsolved rows table: {err:.2e} (bound 1e-05)")
    assert err <= 1e-5, f"table gradient {err:.3e} off the solved rows' alone"
    for k, t in got.items():
        if k != "table":
            assert bits(t[keep], alone[k]), f"{k}: solved rows depend on the unsolved ones"


# ------------------------------------------------------------------------------------------------
# C. the persistent kinematic loop wrapping: every CTA walks at least two tiles
# ------------------------------------------------------------------------------------------------
# (family or shipped robot, contact links, pose, impulse): a small-tile synthetic family (T = 8, ~17 000 rows) and the
# Kuka end-effector pose (T = 64, ~135 000 rows)
WRAP_CASES = [("F_chain64", (63,), True, False), ("iiwa7", (8,), True, False), ("iiwa7", (8,), True, True)]


@pytest.mark.parametrize("name,links,pose,impulse", WRAP_CASES,
                         ids=["F_chain64-dynamics", "iiwa7-dynamics", "iiwa7-impulse"])
def test_persistent_loop_wraps(name, links, pose, impulse, model_dir):
    R = robot(name, model_dir)
    links = list(links)
    par, mov = tree(R)
    _, (t3, _) = G.choices(par, mov, links, pose)
    B = 2 * BWD_MAX_GRID * t3 + t3 + 3
    assert B % t3 and (B + t3 - 1) // t3 > 2 * BWD_MAX_GRID
    what = f"{name} T3={t3} B={B} {'impulse' if impulse else 'dynamics'}"
    pos, mu, x, fwd, g = abi_setup(R, impulse, links, pose, B, 41)
    full = abi(R, impulse, links, pos, mu, x, fwd, g)
    # per-row gradients: the first 3T + 4 rows, a spread in the middle and the tail, each as its own batch
    mid = (B // 2) // t3 * t3
    end = (B // t3 - 3) * t3
    for a, b in ((0, 3 * t3 + 4), (mid, mid + 3 * t3 + 4), (end, B)):
        part = abi(R, impulse, links, pos, mu, *sub(x, fwd, g, a, b), want=[k for k in ALL if k != "table"])
        for k, t in rows_of(full, a, b).items():
            assert bits(part[k], t), f"{what}: {k} rows [{a}, {b}) differ from the batch's"
    # the table gradient against the sum over chunks of at most 20 000 rows (at least three)
    step = min(20000, B // 3 + 1)
    total = torch.zeros_like(full["table"], dtype=torch.float64)
    for a in range(0, B, step):
        total += abi(R, impulse, links, pos, mu, *sub(x, fwd, g, a, min(a + step, B)), want=("table",))["table"].double()
    err = table_error(full["table"], total)
    print(f"ERR {what} chunk sum: {err:.2e} (bound 1e-05)")
    assert err <= 1e-5, f"{what}: table gradient {err:.3e} off the chunks' sum"
    del full, x, fwd, g
    # the tail rows against the fp64 oracle, every link parameter learnable
    tail_check(what, R, impulse, links, pose, B, 41)
