"""GPU: the adjoint of the contact dynamics and contact impulses (csrc/contact_backward.cu) through
compute_contact_dynamics / compute_contact_impulse(..., differentiable=True), against torch autograd of the fp64 oracle
(tests/contact_grad_oracle.py), and the autograd contract of the two entry points.

Tolerance: gradients are compared per family (q, qd, f, the reference, and each link-parameter kind), relative to the
family's largest entry, as in test_forward_dynamics_backward_gpu.py, on the rows whose fp64 smallest scaled pivot is at
least 100x the threshold (the forward tests' rule); the upstream gradients are zero on every other row, on both sides.  The
bound is max(8 x the fp32 oracle's own error on the same rows and upstream, 1e-4): the fp32 oracle differentiates the same
definition by autograd in fp32, so its error measures how much fp32 rounding the conditioning of A and of the articulated
inertias amplifies on those rows."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from conftest import urdf_path
import contact_grad_oracle as CG
import contact_oracle as C
from test_backward_gpu import _ORACLE_PARAM, learnable_model
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
TRI = ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"]
FIELDS = ("trans", "rpy", "mass", "com", "inertia", "damping")
# (robot, links, position_only, mu)
SETS = [("iiwa7", ["iiwa_link_ee"], False, 0.0), ("panda_no_gripper", ["panda_virtual_ee_link"], False, 0.0),
        ("trifinger_edu", TRI, True, 0.0), ("allegro_hand_description_left", TIPS, True, 0.0),
        ("iiwa7_allegro", TIPS, False, 50.0), ("2link_robot", ["endEffector"], False, 0.5)]
FLAGS = [(True, True), (False, False)]


def inputs(robot, B, M, seed):
    q, qd, _ = O.sample_inputs(robot.to(torch.float64), B, seed=seed, dtype=torch.float32)
    g = torch.Generator().manual_seed(seed + 1)
    f = torch.randn(B, robot.n_dofs, generator=g)
    ref = 0.3 * torch.randn(B, M, generator=g)
    g_out = torch.randn(B, robot.n_dofs, generator=g)
    g_lam = torch.randn(B, M, generator=g)
    return q, qd, f, ref, g_out, g_lam


def oracle_robot(stem, dtype):
    r = O.load_robot(urdf_path(stem), torch.float32).to(dtype)
    for name in FIELDS:
        getattr(r, name).requires_grad_(True)
    return r


def oracle_grads(stem, dtype, impulse, q, qd, f, ref, g_out, g_lam, links, pos, mu, grav, damp, ok):
    robot = oracle_robot(stem, dtype)
    ins = [t.to(dtype).clone().requires_grad_(True) for t in (q, qd, f, ref)]
    if impulse:
        out, lam = CG.impulse(robot, ins[0], ins[1], links, ins[3], pos, mu, ok=ok)
    else:
        out, lam = CG.dynamics(robot, ins[0], ins[1], ins[2], links, ins[3], grav, damp, pos, mu, ok=ok)
    loss = (g_out.to(dtype) * out).sum() + (g_lam.to(dtype) * lam).sum()
    wrt = ins + [getattr(robot, n) for n in FIELDS]
    got = torch.autograd.grad(loss, wrt, allow_unused=True)
    return [torch.zeros_like(w) if x is None else x.detach() for w, x in zip(wrt, got)]


def oracle_grads_robot(robot, q, qd, f, ref, g_out, g_lam, links, pos, mu, grav, damp, ok, impulse=False):
    """The input gradients (q, qd, f, ref) of the oracle `robot` (its dtype) by autograd; ref may be None (zero grad)."""
    dtype = robot.trans.dtype
    ins = [t.to(dtype).clone().requires_grad_(True) for t in (q, qd, f, torch.zeros_like(g_lam) if ref is None else ref)]
    r = None if ref is None else ins[3]
    if impulse:
        out, lam = CG.impulse(robot, ins[0], ins[1], links, r, pos, mu, ok=ok)
    else:
        out, lam = CG.dynamics(robot, ins[0], ins[1], ins[2], links, r, grav, damp, pos, mu, ok=ok)
    loss = (g_out.to(dtype) * out).sum() + (g_lam.to(dtype) * lam).sum()
    got = torch.autograd.grad(loss, ins, allow_unused=True)
    return [torch.zeros_like(w) if x is None else x.detach() for w, x in zip(ins, got)]


def family_error(got, want):
    got, want = got.double().cpu().reshape(-1), want.double().cpu().reshape(-1)
    scale = float(want.abs().max()) if want.numel() else 0.0
    return float((got - want).abs().max()) / max(scale, 1e-30) if want.numel() else 0.0


def kernel_grads(stem, impulse, q, qd, f, ref, g_out, g_lam, links, pos, mu, grav, damp):
    m, params = learnable_model(stem)
    x = [t.to(DEV).clone().requires_grad_(True) for t in (q, qd, f)] + [None if ref is None else ref.to(DEV).clone().requires_grad_(True)]
    if impulse:
        out, lam, solved = m.compute_contact_impulse(x[0], x[1], links, velocity_ref=x[3], position_only=pos,
                                                     regularization=mu, differentiable=True)
    else:
        out, lam, solved = m.compute_contact_dynamics(x[0], x[1], x[2], links, accel_ref=x[3], include_gravity=grav,
                                                      use_damping=damp, position_only=pos, regularization=mu,
                                                      differentiable=True)
    torch.autograd.backward([out, lam], [g_out.to(DEV), g_lam.to(DEV)])
    grads = [torch.zeros_like(x[0][:, :1].expand(-1, g_lam.shape[1])) if t is None else
             (torch.zeros_like(t) if t.grad is None else t.grad) for t in x]
    return grads, params, solved.cpu()


@pytest.mark.parametrize("with_ref", [True, False], ids=["ref", "noref"])
@pytest.mark.parametrize("impulse", [False, True], ids=["dynamics", "impulse"])
@pytest.mark.parametrize("grav,damp", FLAGS, ids=["gd", "plain"])
@pytest.mark.parametrize("stem,links,pos,mu", SETS)
def test_gradients_match_fp64_oracle(stem, links, pos, mu, grav, damp, impulse, with_ref):
    B = 48
    M = (3 if pos else 6) * len(links)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f, ref, g_out, g_lam = inputs(r32, B, M, 3)
    if not with_ref:
        ref = torch.zeros_like(ref)       # the kernel gets None, the oracle a constant zero
    r64 = r32.to(torch.float64)
    if impulse:
        _, _, ok64, piv = C.contact_impulse(r64, q.double(), qd.double(), links, ref.double(), pos, mu)
    else:
        _, _, ok64, piv = C.contact_dynamics(r64, q.double(), qd.double(), f.double(), links, ref.double(), grav, damp, pos, mu)
    rows = ok64 & (piv >= 100 * C.PIVOT_MIN)
    assert int(rows.sum()) >= B // 4, f"only {int(rows.sum())} well-conditioned rows"
    g_out, g_lam = g_out * rows[:, None], g_lam * rows[:, None]
    got, params, solved = kernel_grads(stem, impulse, q, qd, f, ref if with_ref else None, g_out, g_lam, links, pos, mu, grav,
                                       damp)
    assert bool(solved[rows].all()), "the kernel leaves well-conditioned rows unsolved"
    w64 = oracle_grads(stem, torch.float64, impulse, q, qd, f, ref, g_out, g_lam, links, pos, mu, grav, damp, rows)
    w32 = oracle_grads(stem, torch.float32, impulse, q, qd, f, ref, g_out, g_lam, links, pos, mu, grav, damp, rows)
    names = ["q", "qd", "f", "ref"] if with_ref else ["q", "qd", "f"]
    # every solved row with a non-zero upstream gets a gradient: the backward solved it too
    assert bool((got[0].cpu()[rows] != 0).any(1).all()), "a well-conditioned row got no gradient"
    for k, name in enumerate(names):
        if impulse and name == "f":
            continue
        e32 = family_error(w32[k][rows], w64[k][rows])
        err = family_error(got[k].cpu()[rows], w64[k][rows])
        bound = max(8 * e32, 1e-4)
        print(f"ERR {stem} {name}: {err:.2e} (bound {bound:.2e})")
        assert np.isfinite(err) and err <= bound, f"{name}: {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"
    for pname, field in _ORACLE_PARAM.items():
        idx = [i for (i, p) in params if p == pname]
        want64 = w64[4 + FIELDS.index(field)]
        want32 = w32[4 + FIELDS.index(field)]
        g = torch.stack([torch.zeros_like(params[(i, pname)]) if params[(i, pname)].grad is None else params[(i, pname)].grad
                         for i in idx]).cpu().reshape(len(idx), -1)
        w = want64[idx].reshape(len(idx), -1)
        w3 = want32[idx].reshape(len(idx), -1)
        e32 = family_error(w3, w)
        err = family_error(g, w)
        bound = max(8 * e32, 1e-4)
        print(f"ERR {stem} {pname}: {err:.2e} (bound {bound:.2e})")
        assert np.isfinite(err) and err <= bound, f"{pname}: {err:.3e} > {bound:.3e} (fp32 oracle {e32:.2e})"
    # rows outside the compared set had zero upstream: exactly zero input gradients there
    for k, name in enumerate(names):
        if impulse and name == "f":
            continue
        assert bool((got[k].cpu()[~rows] == 0).all()), f"{name}: non-zero gradient on a row with zero upstream"


@pytest.mark.parametrize("impulse", [False, True], ids=["dynamics", "impulse"])
def test_unsolved_rows_get_zero_gradients_and_do_not_poison_the_table(impulse):
    stem, links = "iiwa7", ["iiwa_link_ee"]
    m, params = learnable_model(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    B = 200
    q, qd, f, ref, g_out, g_lam = (t.to(DEV) for t in inputs(r32, B, 6, 9))
    bad = torch.zeros(B, dtype=torch.bool, device=DEV)
    bad[::7] = True
    q_bad = torch.where(bad[:, None], torch.full_like(q, float("nan")), q)      # A is NaN there: unsolved

    def run(qq, sel):
        for p in m.parameters():
            p.grad = None
        x = [t[sel].clone().requires_grad_(True) for t in (qq, qd, f, ref)]
        if impulse:
            out, lam, solved = m.compute_contact_impulse(x[0], x[1], links, velocity_ref=x[3], differentiable=True)
        else:
            out, lam, solved = m.compute_contact_dynamics(x[0], x[1], x[2], links, accel_ref=x[3], differentiable=True)
        torch.autograd.backward([out, lam], [g_out[sel], g_lam[sel]])
        return [t.grad for t in x], {k: p.grad.clone() for k, p in params.items() if p.grad is not None}, solved

    all_rows = torch.ones(B, dtype=torch.bool, device=DEV)
    g_all, p_all, solved = run(q_bad, all_rows)
    assert bool((solved == ~bad).all()), "the NaN rows must be exactly the unsolved ones"
    for k, g in enumerate(g_all):
        if impulse and k == 2:
            continue
        assert bool((g[bad] == 0).all()), f"input {k}: unsolved rows get non-zero gradients"
        assert bool(torch.isfinite(g[~bad]).all()), f"input {k}: solved rows not finite"
    g_sub, p_sub, _ = run(q, ~bad)
    for k, g in enumerate(g_all):
        if impulse and k == 2:
            continue
        assert torch.equal(g[~bad], g_sub[k]), f"input {k}: solved rows depend on the unsolved ones"
    for key, g in p_all.items():
        assert bool(torch.isfinite(g).all()), f"{key}: table gradient poisoned"
        scale = float(p_sub[key].abs().max()) or 1.0
        assert float((g - p_sub[key]).abs().max()) <= 1e-5 * scale, f"{key}: differs from the batch without unsolved rows"


def test_table_gradients_are_bitwise_reproducible():
    stem, links = "allegro_hand_description_left", TIPS
    m, params = learnable_model(stem)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f, ref, g_out, g_lam = (t.to(DEV) for t in inputs(r32, 3000, 12, 4))
    runs = []
    for _ in range(2):
        for p in m.parameters():
            p.grad = None
        out, lam, _ = m.compute_contact_dynamics(q, qd, f, links, accel_ref=ref, position_only=True, differentiable=True)
        torch.autograd.backward([out, lam], [g_out, g_lam])
        runs.append([p.grad.clone() for p in params.values()])
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_forward_bits_launch_counts_and_grad_subsets():
    stem, links = "iiwa7", ["iiwa_link_ee"]
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f, ref, g_out, g_lam = (t.to(DEV) for t in inputs(r32, 300, 6, 2))
    plain = m.compute_contact_dynamics(q, qd, f, links, accel_ref=ref)
    torch.cuda.synchronize()
    n0 = engine.launch_count()
    again = m.compute_contact_dynamics(q, qd, f, links, accel_ref=ref, differentiable=True)    # nothing requires grad
    assert engine.launch_count() - n0 == 1
    with torch.no_grad():
        n0 = engine.launch_count()
        m.compute_contact_dynamics(q.requires_grad_(True), qd, f, links, accel_ref=ref, differentiable=True)
        assert engine.launch_count() - n0 == 1
    x = [t.detach().clone().requires_grad_(True) for t in (q, qd, f, ref)]
    n0 = engine.launch_count()
    diff = m.compute_contact_dynamics(*x[:3], links, accel_ref=x[3], differentiable=True)
    assert engine.launch_count() - n0 == 1
    for a, b, c in zip(plain, again, diff):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)) and torch.equal(a.view(torch.uint8),
                                                                                      c.detach().view(torch.uint8))
    assert not diff.solved.requires_grad
    # the full set of gradients, then each input alone and each upstream alone
    full = torch.autograd.grad([diff.qdd, diff.force], x, [g_out, g_lam], retain_graph=True)
    again2 = torch.autograd.grad([diff.qdd, diff.force], x, [g_out, g_lam], retain_graph=True)
    for a, b in zip(full, again2):
        assert torch.equal(a, b)
    for k in range(4):
        one = torch.autograd.grad([diff.qdd, diff.force], [x[k]], [g_out, g_lam], retain_graph=True)[0]
        assert torch.equal(one, full[k])
    only_qdd = torch.autograd.grad([diff.qdd], x, [g_out], retain_graph=True)
    only_lam = torch.autograd.grad([diff.force], x, [g_lam], retain_graph=True)
    for a, b, c in zip(full, only_qdd, only_lam):
        assert float((a - b - c).abs().max()) <= 1e-4 * float(a.abs().max())
    # second order raises
    g = torch.autograd.grad((diff.qdd * g_out).sum(), x[0], create_graph=True)[0]
    with pytest.raises(RuntimeError, match="second-order"):
        g.sum().backward()


def test_side_stream_and_empty_batch():
    stem, links = "iiwa7", ["iiwa_link_ee"]
    m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)
    r32 = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, f, ref, g_out, g_lam = (t.to(DEV) for t in inputs(r32, 500, 6, 6))
    x = [t.clone().requires_grad_(True) for t in (q, qd, f)]
    out = m.compute_contact_dynamics(*x, links, differentiable=True)
    want = torch.autograd.grad([out.qdd, out.force], x, [g_out, g_lam])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        y = [t.clone().requires_grad_(True) for t in (q, qd, f)]
        out2 = m.compute_contact_dynamics(*y, links, differentiable=True)
        got = torch.autograd.grad([out2.qdd, out2.force], y, [g_out, g_lam])
    torch.cuda.current_stream().wait_stream(s)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    e = [torch.zeros(0, r32.n_dofs, device=DEV, requires_grad=True) for _ in range(3)]
    out = m.compute_contact_dynamics(*e, links, differentiable=True)
    (out.qdd.sum() + out.force.sum()).backward()
    assert all(t.grad is not None and t.grad.shape == t.shape for t in e)
    ei = [torch.zeros(0, r32.n_dofs, device=DEV, requires_grad=True) for _ in range(2)]
    out = m.compute_contact_impulse(*ei, links, differentiable=True)
    (out.qd_plus.sum() + out.impulse.sum()).backward()


def test_identify_payload_example_recovers_the_mass(tmp_path):
    """The example recovers the last link's mass (URDF + 1.5 kg) within 2 % from the held end effector's forces."""
    script = os.path.join(REPO, "examples", "identify_payload_from_contact_forces_iiwa.py")
    out = subprocess.run([sys.executable, script], capture_output=True, text=True, cwd=str(tmp_path), timeout=600,
                         env=dict(os.environ, PYTHONPATH=os.pathsep.join([REPO, os.environ.get("PYTHONPATH", "")])))
    assert out.returncode == 0, out.stdout + out.stderr
    line = [l for l in out.stdout.splitlines() if l.startswith("recovered mass")][-1]
    got, want = (float(v) for v in line.split()[2:4])
    assert abs(got - want) <= 0.02 * want, line
