"""TEST INFRASTRUCTURE -- the Levenberg-Marquardt inverse kinematics of csrc/inverse_kinematics.cu restated in batched torch
over oracle/drm_oracle.py (any dtype, CPU).  Rows are independent; the kernel's per-row control flow (skip rows that are done,
reject a step whose Cholesky factorisation fails) becomes masks.  The algorithm is stated in include/drm_b200.h."""
import torch

from oracle import drm_oracle as O

DAMPING_INIT, DAMPING_MIN, DAMPING_MAX = 1e-2, 1e-5, 1e5


def quat_mul(a, b):
    """Hamilton product of xyzw quaternions [B, 4]."""
    ax, ay, az, aw = a.unbind(1)
    bx, by, bz, bw = b.unbind(1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx,
                        aw * bz + ax * by - ay * bx + az * bw,
                        aw * bw - ax * bx - ay * by - az * bz], dim=1)


def orientation_error(target_quat, quat):
    """World-frame rotation vector of R* R^T from xyzw quaternions (target normalised here, either sign of either)."""
    t = target_quat / target_quat.norm(dim=1, keepdim=True)
    qe = quat_mul(t, torch.cat([-quat[:, :3], quat[:, 3:]], dim=1))
    qe = torch.where(qe[:, 3:] < 0, -qe, qe)
    s = qe[:, :3].norm(dim=1)
    safe = torch.where(s > 0, s, torch.ones_like(s))
    g = torch.where(s > 0, 2 * torch.atan2(s, qe[:, 3]) / safe, torch.zeros_like(s))
    return g[:, None] * qe[:, :3]


def pose_and_jacobian(robot, q, link):
    """(p [B, 3], quat [B, 4], J [B, 6, n]) of one link from one kinematic-state walk (O.forward_kinematics / O.jacobian)."""
    R, p, _, _, _ = O.kinematic_state(robot, q)
    e = robot.index(link)
    zero = torch.zeros(q.shape[0], 3, dtype=q.dtype)
    lin, ang = [zero] * robot.n_dofs, [zero] * robot.n_dofs
    i = e
    while i > 0:
        if robot.dof[i] >= 0:
            z = R[i] @ robot.axis[i]
            lin[robot.dof[i]] = torch.cross(z, p[e] - p[i], dim=-1)
            ang[robot.dof[i]] = z
        i = robot.parent[i]
    J = torch.cat([torch.stack(lin, dim=2), torch.stack(ang, dim=2)], dim=1)
    return p[e], O.quaternion(R[e]), J


def evaluate(robot, q, link, target_pos, target_quat=None):
    """(J [B, M, n], e [B, M], E, pos_err, rot_err) with M = 6 (pose) or 3 (position only)."""
    p, quat, J = pose_and_jacobian(robot, q, link)
    e = target_pos - p
    pos_err = e.norm(dim=1)
    if target_quat is None:
        return J[:, :3], e, (e * e).sum(1), pos_err, torch.zeros_like(pos_err)
    e_rot = orientation_error(target_quat, quat)
    e = torch.cat([e, e_rot], dim=1)
    return J, e, (e * e).sum(1), pos_err, e_rot.norm(dim=1)


def step(J, e, lam):
    """One damped least-squares step J^T (J J^T + lam I)^-1 e by Cholesky: (dq [B, n], ok [B]); ok is False where the
    factorisation fails (the step is then rejected)."""
    M = J.shape[1]
    A = J @ J.transpose(1, 2) + lam[:, None, None] * torch.eye(M, dtype=J.dtype)
    L, info = torch.linalg.cholesky_ex(A)
    ok = info == 0
    L = torch.where(ok[:, None, None], L, torch.eye(M, dtype=J.dtype).expand_as(L))
    y = torch.cholesky_solve(e.unsqueeze(2), L).squeeze(2)
    dq = (J.transpose(1, 2) @ y.unsqueeze(2)).squeeze(2)
    return torch.where(ok[:, None], dq, torch.zeros_like(dq)), ok


def solve(robot, q0, link, target_pos, target_quat=None, lower=None, upper=None, damping=None, max_iters=100,
          damping_init=DAMPING_INIT, pos_tol=1e-4, rot_tol=1e-3):
    """The kernel's iteration in the dtype of q0.  Returns a dict of q, pos_err, rot_err, converged, damping and, for the
    last iteration run, `accepted` (rows whose last trial was accepted) and `margin` (|E' - E| / E of that trial)."""
    dt = q0.dtype
    target_pos = target_pos.to(dt)
    target_quat = None if target_quat is None else target_quat.to(dt)

    def clamp(x):
        return x if lower is None else torch.minimum(torch.maximum(x, lower.to(dt)), upper.to(dt))

    B = q0.shape[0]
    q = clamp(q0)
    lam = damping.to(dt).clone() if damping is not None else torch.full((B,), damping_init, dtype=dt)
    J, e, E, perr, rerr = evaluate(robot, q, link, target_pos, target_quat)
    done = (perr <= pos_tol) & (rerr <= rot_tol)
    accepted = torch.zeros(B, dtype=torch.bool)
    margin = torch.full((B,), float("inf"), dtype=dt)
    for _ in range(max_iters):
        active = ~done
        if not bool(active.any()):
            break
        dq, ok = step(J, e, lam)
        qt = clamp(q + dq)
        Jt, et, Et, pt, rt = evaluate(robot, qt, link, target_pos, target_quat)
        acc = active & ok & (Et < E)
        rej = active & ~acc
        margin = torch.where(active & ok, (Et - E).abs() / E, torch.full_like(E, float("inf")))
        accepted = acc
        q = torch.where(acc[:, None], qt, q)
        J = torch.where(acc[:, None, None], Jt, J)
        e = torch.where(acc[:, None], et, e)
        E, perr, rerr = (torch.where(acc, a, b) for a, b in ((Et, E), (pt, perr), (rt, rerr)))
        lam = torch.where(acc, torch.clamp(lam / 2, min=DAMPING_MIN), torch.where(rej, torch.clamp(4 * lam, max=DAMPING_MAX), lam))
        done = torch.where(acc, (perr <= pos_tol) & (rerr <= rot_tol), done)
    return dict(q=q, pos_err=perr, rot_err=rerr, converged=done, damping=lam, accepted=accepted, margin=margin)


def joint_limits(robot, dtype=torch.float32):
    lo = torch.tensor([robot.limits[i]["lower"] for i in robot.controlled], dtype=torch.float64).to(dtype)
    hi = torch.tensor([robot.limits[i]["upper"] for i in robot.controlled], dtype=torch.float64).to(dtype)
    return lo, hi


def problem(robot, link, batch, seed=0, noise=0.3):
    """Reachable targets and nearby starts: goal ~ U(limits), (target_pos, target_quat) = fp64 FK of the goal, q0 = goal +
    N(0, noise^2) clamped to the limits.  fp32 tensors (q0, target_pos, target_quat)."""
    gen = torch.Generator().manual_seed(seed)
    lo, hi = joint_limits(robot, torch.float64)
    goal = lo + (hi - lo) * torch.rand(batch, robot.n_dofs, generator=gen, dtype=torch.float64)
    q0 = torch.minimum(torch.maximum(goal + noise * torch.randn(batch, robot.n_dofs, generator=gen, dtype=torch.float64), lo), hi)
    pos, quat = O.forward_kinematics(robot.to(torch.float64), goal, link)
    return q0.float(), pos.float(), quat.float()
