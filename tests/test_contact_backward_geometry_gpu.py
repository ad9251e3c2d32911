"""GPU: the contact adjoint (csrc/contact_backward.cu) at every launch geometry its host rules choose, on the synthetic
topology families, against compositions of the existing adjoints, on redundant sets, and for every subset of the inputs
that require grad.

* Launch geometry.  A mirror of contact_backward_tile and kinematic_backward_tile (the ContactBwdSmemLayout and KinBwdSmem
  byte counts through tile_ladder; neither kernel declares static shared memory), one case per reachable rung of either
  kernel, and a test that every rung the families reach has a case.  Each case compares the gradients with the fp64
  oracle, checks that input-gradient rows are bit-identical at batches tile - 1, tile, tile + 1 and 3 tile + 3 and with
  every pointer 4 bytes off 16-byte alignment (the cooperative copies).
* Synthetic families: solved against the oracle, or refused with the forward's message and no launch.
* Identities: f_grad is the forward-dynamics adjoint of g^ = g_qdd - J^T nu at f + J^T lambda; the q and table gradients
  are that adjoint's plus the per-link FK/Jacobian adjoints of g_jac = lambda_e tau^T - nu_e qdd^T at qd = 0; a fused
  model gets the per-module gradients.
Tolerances as in test_contact_backward_gpu.py: per family, relative to its largest entry, max(8 x the fp32 oracle's error,
1e-4) against the oracle; between compositions whose roundings differ 1e-4 for input gradients and 1e-3 for link-parameter
families, which carry terms that cancel exactly in the kernel but not in a sum of separately rounded adjoints."""
import ctypes
import itertools

import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar, UnconstrainedTensor
from conftest import urdf_path
import contact_oracle as C
import synthetic_robots as SR
import test_contact_backward_gpu as CB
import test_launch_geometry_solvers_gpu as LG
import tile_mirrors as TM
from test_backward_gpu import learnable_model
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FAM = SR.families()
TIPS = CB.TIPS


# ------------------------------------------------------------------------------------------------
# the mirror of the two tile rules
# ------------------------------------------------------------------------------------------------
def stage1_floats(T, n, n_links, tree_slots, n_u, M, n_jslots, n_state_slots):
    """ContactBwdSmemLayout(T, tree program, walk, M).total_floats."""
    aba = 4 * T * n + n_links * TM.TABLE_STRIDE + n_links * 14 * T + tree_slots * 42 * T
    return (TM.up4(aba) + TM.up4(M * T) + TM.up4(n * T)
            + T * (M + M * n_u + 6 * n_jslots + 24 * n_state_slots + 6 * M + M * M + 2 * n + 1))


def kinematic_floats(T, n, n_links, M, n_steps, n_state_slots):
    """KinBwdSmem(T, max(T, 32), tree program, walk, M).total_floats."""
    nt = max(T, 32)
    return (n_links * TM.TABLE_STRIDE + TM.up4(n_links * 12) + TM.up4((nt // 32) * 32 + 12 * (nt + 1))
            + 6 * TM.up4(T * n) + 2 * TM.up4(T * M) + T * (20 * n_steps + 45 * n_state_slots))


def choices(parents, movable, links, pose):
    """((stage-1 tile, bytes), (kinematic tile, bytes)); a tile is None when the rule refuses."""
    n = sum(movable[1:])
    n_steps, n_u, n_jslots, n_slots = TM.multi_program(parents, movable, links)
    M = (6 if pose else 3) * len(links)
    tree_slots = SR.live_slots(parents)
    a = TM.ladder(lambda T: stage1_floats(T, n, len(parents), tree_slots, n_u, M, n_jslots, n_slots), 0)
    b = TM.ladder(lambda T: kinematic_floats(T, n, len(parents), M, n_steps, n_slots), 0)
    return a, b


def _solvable(par, mov, links):
    def movable_path(l):
        while l > 0:
            if mov[l]:
                return True
            l = par[l]
        return False
    return all(movable_path(l) for l in links)


def _tile_cases():
    cases = {}
    for name in sorted(FAM):
        par, mov = FAM[name].doc()
        if sum(mov[1:]) == 0:
            continue
        for k in (1, 2, 4, 8):
            links = LG.deepest(par, mov, k)
            if not _solvable(par, mov, links):
                continue
            for pose in (True, False):     # pose first: a link on its only joint's axis has zero linear rows
                (t1, _), (t3, _) = choices(par, mov, links, pose)
                if t1 is None or t3 is None:
                    continue
                cases.setdefault(("stage1", t1), (name, links, pose))
                cases.setdefault(("kinematic", t3), (name, links, pose))
    return cases


TILE_CASES = _tile_cases()


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic_contact_backward"))


def shifted(t):
    if t is None:
        return None
    off = 1 if t.dtype == torch.float32 else 4
    buf = torch.empty(t.numel() + off, device=DEV, dtype=t.dtype)
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def backward_call(topo, links, table, x, out, lam, solved, g, pos, mu, flags, misaligned=False):
    """drmb200_contact_dynamics_backward with caller-allocated outputs: (q_grad, qd_grad, f_grad, ref_grad)."""
    q, qd, f, ref = x
    B, n = q.shape
    M = lam.shape[1]
    outs = [torch.empty((B, n), device=DEV) for _ in range(3)] + [torch.empty((B, M), device=DEV)]
    ins = [q, qd, f, ref, out, lam, g[0], g[1]]
    if misaligned:
        ins, outs = [shifted(t) for t in ins], [shifted(t) for t in outs]
    idx = (ctypes.c_int32 * len(links))(*links)
    lib = engine.lib()
    nbytes = int(lib.drmb200_contact_backward_workspace_bytes(ctypes.byref(topo), len(links), idx, int(pos), B))
    ws = torch.empty((nbytes + 3) // 4 + 1, device=DEV)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.drmb200_contact_dynamics_backward(
        ctypes.byref(topo), len(links), idx, ptr(table), ptr(ins[0]), ptr(ins[1]), ptr(ins[2]), ptr(ins[3]), ptr(ins[4]),
        ptr(ins[5]), ptr(solved), B, flags, int(pos), ctypes.c_float(mu), ptr(ins[6]), ptr(ins[7]), *[ptr(t) for t in outs],
        None, ptr(ws), s)
    assert rc == 0, lib.drmb200_last_error()
    return outs


def same_rows(what, small, big):
    for k, (a, b) in enumerate(zip(small, big)):
        assert torch.equal(a.view(torch.int32), b[:a.shape[0]].view(torch.int32)), f"{what}: output {k} rows differ"


@pytest.mark.parametrize("key", sorted(TILE_CASES), ids=[f"{k}-T{t}" for k, t in sorted(TILE_CASES)])
def test_backward_at_every_tile(key, model_dir):
    stage, tile = key
    name, links, pose = TILE_CASES[key]
    m, r32, r64, table = LG.family(name, model_dir)
    topo = m._topology
    pos = not pose
    M = (3 if pos else 6) * len(links)
    B = max(3 * tile + 4, 70)
    q, qd, f, ref, g_out, g_lam = CB.inputs(r32, B, M, 21)
    x = [t.to(DEV) for t in (q, qd, f, ref)]
    g = [g_out.to(DEV), g_lam.to(DEV)]
    lnames = [r32.names[l] for l in links]
    J = C.S.stacked_jacobian(r64, q.double()[:8], lnames, pos)
    G = C.S.force_response(r64, q.double()[:8])
    par, mov = FAM[name].doc()
    _, n_u, _, _ = TM.multi_program(par, mov, links)
    # a redundant set (M > n_u) is conditioned by mu alone: 0.1 max A_kk keeps every scaled pivot far above the threshold
    mu = (1e-3 if M <= n_u else 1e-1) * float(torch.diagonal(J @ G @ J.transpose(1, 2), dim1=1, dim2=2).max())
    flags = engine.GRAVITY | engine.DAMPING
    out, lam, solved = engine.contact_dynamics_raw(topo, links, table, *x[:3], flags, x[3], pos, mu)
    big = backward_call(topo, links, table, x, out, lam, solved, g, pos, mu, flags)
    for b in sorted({1, max(1, tile - 1), tile, tile + 1, 3 * tile + 3}):
        small = backward_call(topo, links, table, [t[:b] for t in x], out[:b], lam[:b], solved[:b], [t[:b] for t in g], pos,
                              mu, flags)
        same_rows(f"{name} B={b}", small, big)
    same_rows(f"{name} misaligned", backward_call(topo, links, table, x, out, lam, solved, g, pos, mu, flags, True), big)
    # the first rows against the fp64 oracle (upstream zero on the rows the oracle cannot decide)
    k = 8
    _, _, ok64, piv = C.contact_dynamics(r64, q[:k].double(), qd[:k].double(), f[:k].double(), lnames, ref[:k].double(),
                                         True, True, pos, mu)
    rows = ok64 & (piv >= 100 * C.PIVOT_MIN) & solved[:k].cpu()
    assert int(rows.sum()) >= 2, f"{name}: only {int(rows.sum())} well-conditioned rows"
    gk = [g_out[:k] * rows[:, None], g_lam[:k] * rows[:, None]]
    got = backward_call(topo, links, table, [t[:k] for t in x], out[:k], lam[:k], solved[:k], [t.to(DEV) for t in gk], pos,
                        mu, flags)
    w64 = CB.oracle_grads_robot(r64, q[:k], qd[:k], f[:k], ref[:k], *gk, lnames, pos, mu, True, True, rows)
    w32 = CB.oracle_grads_robot(r32, q[:k], qd[:k], f[:k], ref[:k], *gk, lnames, pos, mu, True, True, rows)
    for j, nm in enumerate(("q", "qd", "f", "ref")):
        e32 = CB.family_error(w32[j][rows], w64[j][rows])
        err = CB.family_error(got[j].cpu()[rows], w64[j][rows])
        bound = max(8 * e32, 1e-4)
        print(f"ERR {name} {stage} T={tile} {nm}: {err:.2e} (bound {bound:.2e})")
        assert err <= bound, f"{name} {nm}: {err:.3e} > {bound:.3e}"


def test_every_reachable_rung_has_a_case():
    reached = {}
    for name in sorted(FAM):
        par, mov = FAM[name].doc()
        if sum(mov[1:]) == 0:
            continue
        for k in range(1, 9):
            links = LG.deepest(par, mov, k)
            if not _solvable(par, mov, links):
                continue
            for pose in (False, True):
                (t1, _), (t3, _) = choices(par, mov, links, pose)
                if t1 is not None and t3 is not None:
                    reached.setdefault(("stage1", t1), name)
                    reached.setdefault(("kinematic", t3), name)
    assert set(reached) <= set(TILE_CASES), sorted(set(reached) - set(TILE_CASES))
    assert {t for s, t in TILE_CASES if s == "kinematic"} & {1, 2, 4, 8, 16}, "no case below one warp per CTA"


def test_static_shared_memory_is_zero():
    lib = engine.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    for t in TM.LADDER:
        for b in (0, 1):
            for sym in (f"_ZN3drm23contact_backward_kernelILi{t}ELb{b}EEEvNS_11TreeProgramENS_12UnionProgramENS_14ContactBwdArgsE",
                        f"_ZN3drm33contact_kinematic_backward_kernelILi{t}ELb{b}EEEvNS_11TreeProgramENS_12UnionProgramENS_10KinBwdArgsE"):
                attr = (ctypes.c_size_t * 64)()
                rc = cudart.cudaFuncGetAttributes(attr, ctypes.cast(getattr(lib, sym), ctypes.c_void_p))
                assert rc == 0 and attr[0] == 0, (sym, rc, attr[0])


# ------------------------------------------------------------------------------------------------
# synthetic topologies
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(FAM))
def test_synthetic_families_match_oracle_or_are_refused(name, model_dir):
    m, r32, r64, table = LG.family(name, model_dir)
    par, mov = FAM[name].doc()
    names = r32.names
    links = [l for l in dict.fromkeys([len(names) - 1, len(names) // 2]) if l > 0] or [0]
    B = 9
    if r32.n_dofs == 0 or not _solvable(par, mov, links):
        z = torch.zeros(B, r32.n_dofs, device=DEV)
        lam = torch.zeros(B, 3 * len(links), device=DEV)
        before = engine.launch_count()
        with pytest.raises(RuntimeError, match="no movable joint"):
            engine.contact_dynamics_backward_raw(m._topology, links, table, z, z, z, z, lam,
                                                 torch.ones(B, dtype=torch.bool, device=DEV), 0, z, lam, None, True, 0.1)
        assert engine.launch_count() == before
        return
    lnames = [names[l] for l in links]
    for pos in (False, True):
        M = (3 if pos else 6) * len(links)
        q, qd, f, ref, g_out, g_lam = CB.inputs(r32, B, M, 17)
        J = C.S.stacked_jacobian(r64, q.double(), lnames, pos)
        G = C.S.force_response(r64, q.double())
        mu = 1e-3 * float(torch.diagonal(J @ G @ J.transpose(1, 2), dim1=1, dim2=2).max())
        dev = [t.to(DEV) for t in (q, qd, f)]
        out, lam, solved = engine.contact_dynamics_raw(m._topology, links, table, *dev, engine.GRAVITY, None, pos, mu)
        _, _, ok64, piv = C.contact_dynamics(r64, q.double(), qd.double(), f.double(), lnames, None, True, False, pos, mu)
        rows = ok64 & (piv >= 100 * C.PIVOT_MIN) & solved.cpu()
        if int(rows.sum()) == 0:
            continue
        gk = [g_out * rows[:, None], g_lam * rows[:, None]]
        got = engine.contact_dynamics_backward_raw(m._topology, links, table, *dev, out, lam, solved, engine.GRAVITY,
                                                   gk[0].to(DEV), gk[1].to(DEV), None, pos, mu, want_table=False)
        zero_ref = torch.zeros(B, M)
        w64 = CB.oracle_grads_robot(r64, q, qd, f, zero_ref, *gk, lnames, pos, mu, True, False, rows)
        w32 = CB.oracle_grads_robot(r32, q, qd, f, zero_ref, *gk, lnames, pos, mu, True, False, rows)
        for j, nm in enumerate(("q", "qd", "f", "ref")):
            e32 = CB.family_error(w32[j][rows], w64[j][rows])
            err = CB.family_error(got[j].cpu()[rows], w64[j][rows])
            bound = max(8 * e32, 1e-4)
            print(f"ERR {name} pos={pos} {nm}: {err:.2e} (bound {bound:.2e})")
            assert err <= bound, f"{name} pos={pos} {nm}: {err:.3e} > {bound:.3e}"


@pytest.mark.parametrize("name", ["H_nine_slots"])
def test_too_many_branch_points_give_the_forward_dynamics_message_without_a_launch(name, model_dir):
    spec = SR.refusal_families()[name]
    path = SR.build(spec, model_dir)
    m = drm.DifferentiableRobotModel(path, name, device=DEV)
    r32 = O.load_robot(path, torch.float32)
    table = O.link_table(r32).float().to(DEV).contiguous()
    q = torch.zeros(4, r32.n_dofs, device=DEV)
    with pytest.raises(RuntimeError) as fd:
        engine.forward_dynamics_raw(m._topology, table, q, q, q, 0)
    msg = str(fd.value).split("): ", 1)[1]
    par, mov = spec.doc()
    links = LG.deepest(par, mov, 1)
    lam = torch.zeros(4, 6, device=DEV)
    ok = torch.ones(4, dtype=torch.bool, device=DEV)
    before = engine.launch_count()
    with pytest.raises(RuntimeError, match=r"code -3\): ") as got:
        engine.contact_dynamics_backward_raw(m._topology, links, table, q, q, q, q, lam, ok, 0, q, lam)
    assert str(got.value).split("): ", 1)[1] == msg
    with pytest.raises(RuntimeError, match=r"code -3\): ") as got:
        engine.contact_impulse_backward_raw(m._topology, links, table, q, q, q, lam, ok, q, lam)
    assert str(got.value).split("): ", 1)[1] == msg
    assert engine.launch_count() == before


# ------------------------------------------------------------------------------------------------
# identities with the existing adjoints
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem,links,pos", [("iiwa7", ["iiwa_link_ee"], False), ("allegro_hand_description_left", TIPS, True)])
def test_composition_of_the_existing_adjoints(stem, links, pos):
    """At qd = 0: f_grad = FD adjoint of g^ at f + J^T lambda; q and table gradients = that adjoint's plus the per-link
    FK/Jacobian adjoints of g_jac = lambda_e tau^T - nu_e qdd^T."""
    m, params = learnable_model(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    M = (3 if pos else 6) * len(links)
    q, _, f, ref, g_out, g_lam = (t.to(DEV) for t in CB.inputs(r32, 300, M, 8))
    qd = torch.zeros_like(q)
    x = [t.clone().requires_grad_(True) for t in (q, qd, f, ref)]
    out = m.compute_contact_dynamics(*x[:3], links, accel_ref=x[3], position_only=pos, differentiable=True)
    keep = out.solved
    go, gl = g_out * keep[:, None], g_lam * keep[:, None]
    torch.autograd.backward([out.qdd, out.force], [go, gl])
    got_q, got_f, nu = x[0].grad.clone(), x[2].grad.clone(), x[3].grad.clone()
    got_p = {k: p.grad.clone() for k, p in params.items() if p.grad is not None}
    for p in params.values():
        p.grad = None
    lam, qdd = out.force.detach().nan_to_num(), out.qdd.detach().nan_to_num()
    # the forward-dynamics adjoint at (q, 0, f + J^T lambda) for g^ = g - J^T nu
    with torch.no_grad():
        fk = m.compute_fk_and_jacobian_multi(q, links)
        J = torch.cat([fk[nm][2] if pos else torch.cat([fk[nm][2], fk[nm][3]], dim=1) for nm in links], dim=1)
        tauc = f + torch.einsum("bmn,bm->bn", J, lam)
        ghat = go - torch.einsum("bmn,bm->bn", J, nu)
    y = [t.clone().requires_grad_(True) for t in (q, tauc)]
    qdd_fd = m.compute_forward_dynamics(y[0], qd, y[1], include_gravity=True, use_damping=False)
    torch.autograd.backward(qdd_fd, ghat)
    taubar = y[1].grad.detach()
    assert CB.family_error(got_f[keep], taubar[keep]) <= 1e-4
    # the per-link FK/Jacobian adjoints of g_jac = lambda_e tau^T - nu_e qdd^T
    z = q.clone().requires_grad_(True)
    fk = m.compute_fk_and_jacobian_multi(z, links)
    loss = 0
    MR = 3 if pos else 6
    for e, nm in enumerate(links):
        Je = fk[nm][2] if pos else torch.cat([fk[nm][2], fk[nm][3]], dim=1)
        gj = lam[:, MR * e:MR * e + MR, None] * taubar[:, None, :] - nu[:, MR * e:MR * e + MR, None] * qdd[:, None, :]
        loss = loss + (Je * gj * keep[:, None, None]).sum()
    loss.backward()
    want_q = y[0].grad + z.grad
    assert CB.family_error(got_q[keep], want_q[keep]) <= 1e-4
    # per parameter kind, relative to the kind's largest entry: terms that cancel exactly in the kernel (the first link's
    # offset, which moves the whole model rigidly: its gradient is exactly zero there) are sums of separately rounded
    # adjoints in the composition, whose residue is ~1e-4 of the family
    for pname in {k[1] for k in params}:
        keys = sorted(k for k in params if k[1] == pname)
        got = torch.cat([got_p.get(k, torch.zeros_like(params[k])).reshape(-1) for k in keys])
        want = torch.cat([(torch.zeros_like(params[k]) if params[k].grad is None else params[k].grad).reshape(-1)
                          for k in keys])
        err = CB.family_error(got, want)
        print(f"ERR composition {stem} {pname}: {err:.2e}")
        assert err <= 1e-3, (pname, err)


def test_fused_model_gets_the_per_module_gradients():
    stem, links = "iiwa7", ["iiwa_link_ee"]
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f, ref, g_out, g_lam = (t.to(DEV) for t in CB.inputs(r32, 200, 6, 12))
    grads = []
    for fuse in (False, True):
        m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
        mods = []
        for i in (3, 5, 7):
            body = m._bodies[i]
            mods.append(UnconstrainedScalar(init_val=body.inertia.mass().detach().clone()))
            m.make_link_param_learnable(body.name, "mass", mods[-1])
            mods.append(UnconstrainedTensor(1, 3, init_tensor=body.trans().detach().clone().reshape(1, 3)))
            m.make_link_param_learnable(body.name, "trans", mods[-1])
        if fuse:
            m.fuse_learnable_parameters()
        out = m.compute_contact_dynamics(q, qd, f, links, accel_ref=ref, differentiable=True)
        torch.autograd.backward([out.qdd, out.force], [g_out * out.solved[:, None], g_lam * out.solved[:, None]])
        import test_learning_paths_gpu as LP
        grads.append([LP.gradient_of(m, mod.param).clone() for mod in mods])
    for a, b in zip(*grads):
        assert CB.family_error(a, b) <= 1e-6, (a, b)


# ------------------------------------------------------------------------------------------------
# redundant sets and gradient subsets
# ------------------------------------------------------------------------------------------------
def test_redundant_set_unsolved_rows_get_zero_gradients():
    """4 fingertip poses on iiwa7_allegro at mu = 0 (24 rows, 23 joints): the pivot threshold leaves (almost) every row
    unsolved.  Those rows get exactly zero gradients, the table gradient is finite and equals the one of the solved rows
    alone."""
    stem = "iiwa7_allegro"
    m, params = learnable_model(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f, ref, g_out, g_lam = (t.to(DEV) for t in CB.inputs(r32, 600, 24, 31))
    x = [t.clone().requires_grad_(True) for t in (q, qd, f, ref)]
    out = m.compute_contact_dynamics(*x[:3], TIPS, accel_ref=x[3], differentiable=True)
    assert float(out.solved.float().mean()) < 0.5
    torch.autograd.backward([out.qdd, out.force], [g_out, g_lam])
    bad = ~out.solved
    for k, t in enumerate(x):
        assert bool((t.grad[bad] == 0).all()), f"input {k}: unsolved rows get gradients"
    all_p = {k: p.grad.clone() for k, p in params.items() if p.grad is not None}
    assert all(bool(torch.isfinite(g).all()) for g in all_p.values())
    for p in params.values():
        p.grad = None
    sel = out.solved
    if int(sel.sum()):
        y = [t[sel].clone().requires_grad_(True) for t in (q, qd, f, ref)]
        o2 = m.compute_contact_dynamics(*y[:3], TIPS, accel_ref=y[3], differentiable=True)
        torch.autograd.backward([o2.qdd, o2.force], [g_out[sel], g_lam[sel]])
    for k, g in all_p.items():
        want = torch.zeros_like(g) if params[k].grad is None else params[k].grad
        scale = max(float(want.abs().max()), 1e-30)
        assert float((g - want).abs().max()) <= 1e-5 * scale or float((g - want).abs().max()) == 0.0, k


@pytest.mark.parametrize("impulse", [False, True], ids=["dynamics", "impulse"])
def test_every_subset_of_inputs_requiring_grad(impulse):
    stem, links = "iiwa7", ["iiwa_link_ee"]
    m, params = learnable_model(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f, ref, g_out, g_lam = (t.to(DEV) for t in CB.inputs(r32, 257, 6, 14))
    names = ["q", "qd", "ref"] if impulse else ["q", "qd", "f", "ref"]
    base = {"q": q, "qd": qd, "f": f, "ref": ref}

    def run(wanted, table, ups):
        for p in m.parameters():
            p.requires_grad_(table)
            p.grad = None
        x = {k: base[k].clone().requires_grad_(k in wanted) for k in base}
        if impulse:
            out, lam, _ = m.compute_contact_impulse(x["q"], x["qd"], links, velocity_ref=x["ref"], differentiable=True)
        else:
            out, lam, _ = m.compute_contact_dynamics(x["q"], x["qd"], x["f"], links, accel_ref=x["ref"], differentiable=True)
        outs, gs = [], []
        if ups[0]:
            outs.append(out); gs.append(g_out)
        if ups[1]:
            outs.append(lam); gs.append(g_lam)
        if not any(t.requires_grad for t in outs):
            return None
        torch.autograd.backward(outs, gs)
        return {k: x[k].grad for k in wanted}, {k: p.grad for k, p in params.items()}

    for ups in ((True, True), (True, False), (False, True)):
        full_in, full_p = run(set(names), True, ups)
        for r in range(len(names) + 1):
            for sub in itertools.combinations(names, r):
                for table in (False, True):
                    if not sub and not table:
                        continue
                    got = run(set(sub), table, ups)
                    g_in, g_p = got
                    for k in sub:
                        assert torch.allclose(g_in[k], full_in[k], rtol=1e-5, atol=1e-6 * float(full_in[k].abs().max())), \
                            (sub, table, ups, k)
                    if table:
                        for k, g in g_p.items():
                            w = full_p[k]
                            assert (g is None) == (w is None), k
                            if g is not None:
                                assert torch.allclose(g, w, rtol=1e-5, atol=1e-6 * float(w.abs().max())), (sub, ups, k)
    for p in m.parameters():
        p.requires_grad_(True)
