"""TEST INFRASTRUCTURE -- the multi-link Levenberg-Marquardt inverse kinematics of csrc/inverse_kinematics_multi.cu restated
in batched torch over tests/ik_oracle.py (any dtype, CPU), with the kernel's choice of the smaller system: task space
(J J^T + lambda I, M x M) when M <= n_u, joint space (J^T J + lambda I, n_u x n_u) otherwise.  The algorithm is stated in
include/drm_b200.h."""
import torch

import ik_oracle as IK
from oracle import drm_oracle as O

DAMPING_INIT, DAMPING_MIN, DAMPING_MAX = IK.DAMPING_INIT, IK.DAMPING_MIN, IK.DAMPING_MAX


def union_dofs(robot, links):
    """The movable joints on the union of the root -> link paths (the set U), ascending."""
    dofs = set()
    for link in links:
        i = robot.index(link)
        while i > 0:
            if robot.dof[i] >= 0:
                dofs.add(robot.dof[i])
            i = robot.parent[i]
    return sorted(dofs)


def evaluate(robot, q, links, target_pos, target_quat=None):
    """(J [B, M, n], e [B, M], E [B], pos_err [n_ee, B], rot_err [n_ee, B]): every link's ik_oracle.evaluate block stacked
    link by link (6 rows per link in pose mode, 3 in position mode); E summed in link order."""
    blocks = [IK.evaluate(robot, q, link, target_pos[l], None if target_quat is None else target_quat[l])
              for l, link in enumerate(links)]
    E = blocks[0][2]
    for b in blocks[1:]:
        E = E + b[2]
    return (torch.cat([b[0] for b in blocks], dim=1), torch.cat([b[1] for b in blocks], dim=1), E,
            torch.stack([b[3] for b in blocks]), torch.stack([b[4] for b in blocks]))


def step(J, e, lam, space=None):
    """One damped least-squares step over the columns of J [B, M, n_u]: (dq [B, n_u], ok [B]).  space None: the kernel's
    choice ("task" when M <= n_u, else "joint"); "task" / "joint" force one.  ok is False where the Cholesky fails."""
    M, n_u = J.shape[1], J.shape[2]
    if space is None:
        space = "task" if M <= n_u else "joint"
    if space == "task":
        return IK.step(J, e, lam)
    Jt = J.transpose(1, 2)
    A = Jt @ J + lam[:, None, None] * torch.eye(n_u, dtype=J.dtype)
    L, info = torch.linalg.cholesky_ex(A)
    ok = info == 0
    L = torch.where(ok[:, None, None], L, torch.eye(n_u, dtype=J.dtype).expand_as(L))
    dq = torch.cholesky_solve((Jt @ e.unsqueeze(2)), L).squeeze(2)
    return torch.where(ok[:, None], dq, torch.zeros_like(dq)), ok


def solve(robot, q0, links, target_pos, target_quat=None, lower=None, upper=None, damping=None, max_iters=100,
          damping_init=DAMPING_INIT, pos_tol=1e-4, rot_tol=1e-3):
    """The kernel's iteration in the dtype of q0; target_pos [n_ee, B, 3], target_quat [n_ee, B, 4] or None.  Returns a
    dict of q, pos_err / rot_err [n_ee, B], converged, damping and, for the last iteration run, `accepted` and `margin`
    (|E' - E| / E of that trial), as ik_oracle.solve."""
    dt = q0.dtype
    target_pos = target_pos.to(dt)
    target_quat = None if target_quat is None else target_quat.to(dt)
    U = torch.tensor(union_dofs(robot, links), dtype=torch.long)

    def clamp(x):
        return x if lower is None else torch.minimum(torch.maximum(x, lower.to(dt)), upper.to(dt))

    def within(perr, rerr):
        return ((perr <= pos_tol) & (rerr <= rot_tol)).all(0)

    B = q0.shape[0]
    q = clamp(q0)
    lam = damping.to(dt).clone() if damping is not None else torch.full((B,), damping_init, dtype=dt)
    J, e, E, perr, rerr = evaluate(robot, q, links, target_pos, target_quat)
    done = within(perr, rerr)
    accepted = torch.zeros(B, dtype=torch.bool)
    margin = torch.full((B,), float("inf"), dtype=dt)
    for _ in range(max_iters):
        active = ~done
        if not bool(active.any()):
            break
        dq_u, ok = step(J[:, :, U], e, lam)
        dq = torch.zeros_like(q)
        dq[:, U] = dq_u
        qt = clamp(q + dq)
        Jt, et, Et, pt, rt = evaluate(robot, qt, links, target_pos, target_quat)
        acc = active & ok & (Et < E)
        rej = active & ~acc
        margin = torch.where(active & ok, (Et - E).abs() / E, torch.full_like(E, float("inf")))
        accepted = acc
        q = torch.where(acc[:, None], qt, q)
        J = torch.where(acc[:, None, None], Jt, J)
        e = torch.where(acc[:, None], et, e)
        E = torch.where(acc, Et, E)
        perr, rerr = torch.where(acc[None], pt, perr), torch.where(acc[None], rt, rerr)
        lam = torch.where(acc, torch.clamp(lam / 2, min=DAMPING_MIN), torch.where(rej, torch.clamp(4 * lam, max=DAMPING_MAX), lam))
        done = torch.where(acc, within(perr, rerr), done)
    return dict(q=q, pos_err=perr, rot_err=rerr, converged=done, damping=lam, accepted=accepted, margin=margin)


def problem(robot, links, batch, seed=0, noise=0.3):
    """Reachable targets for every link and nearby starts, as ik_oracle.problem: goal ~ U(limits), targets = fp64 FK of the
    goal per link, q0 = goal + N(0, noise^2) clamped to the limits.  fp32 (q0 [B, n], target_pos [n_ee, B, 3],
    target_quat [n_ee, B, 4])."""
    gen = torch.Generator().manual_seed(seed)
    lo, hi = IK.joint_limits(robot, torch.float64)
    goal = lo + (hi - lo) * torch.rand(batch, robot.n_dofs, generator=gen, dtype=torch.float64)
    q0 = torch.minimum(torch.maximum(goal + noise * torch.randn(batch, robot.n_dofs, generator=gen, dtype=torch.float64), lo), hi)
    r64 = robot.to(torch.float64)
    poses = [O.forward_kinematics(r64, goal, link) for link in links]
    return q0.float(), torch.stack([p for p, _ in poses]).float(), torch.stack([qt for _, qt in poses]).float()
