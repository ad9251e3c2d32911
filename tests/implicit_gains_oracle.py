"""Reference restatement of the PD-controlled rollout with implicit PD gains (stable PD), for the tests.

Test helper module (not a conftest).  forward_dynamics restates implicit_damping_oracle.forward_dynamics (itself
oracle/drm_oracle.py: forward_dynamics with the implicit-damping pivot) with one more term, the per-row pivot addend of
DRMB200_IMPLICIT_GAINS: every movable joint k's pivot d_k (+ h damping_k) then gets + c[:, k].  Without an addend it is
that function, and at damping_dt = 0 the oracle's, bit for bit.  pd_rollout is the definition drmb200_pd_rollout
implements with DRMB200_IMPLICIT_GAINS (include/drm_b200.h); at kp = kd = 0 it is pd_rollout_oracle.pd_rollout bit for bit.
The oracle package and the other restatements are unchanged."""
import torch

from oracle import drm_oracle as O


def forward_dynamics(robot, q, qd, f, include_gravity=True, use_damping=True, damping_dt=0.0, addend=None):
    """O.forward_dynamics with the pivot d_k + damping_dt * damping_k (+ addend[:, k]) of every movable joint.  Any dtype;
    differentiable (the damping and the addend included)."""
    B = q.shape[0]
    N = len(robot.names)
    dt = q.dtype
    if use_damping:
        f = f - torch.stack([robot.damping[i] for i in robot.controlled]).unsqueeze(0) * qd
    R, p, w, v, joints = O.kinematic_state(robot, q, qd)
    zeros = torch.zeros(B, 3, dtype=dt)
    g = torch.stack([zeros[:, 0], zeros[:, 0], (9.81 if include_gravity else 0.0) * torch.ones(B, dtype=dt)], dim=1)
    c, pA, IA = [None] * N, [None] * N, [None] * N
    for i in range(1, N):
        jw = qd[:, robot.dof[i]:robot.dof[i] + 1] @ robot.axis[i:i + 1] if robot.dof[i] >= 0 else zeros
        c[i] = torch.cat([O._cross(w[i], jw), O._cross(v[i], jw)], dim=1)
        h_lin, h_ang = O._inertia_times(robot, i, w[i], v[i])
        pA[i] = torch.cat([O._cross(w[i], h_ang) + O._cross(v[i], h_lin), O._cross(w[i], h_lin)], dim=1)
        IA[i] = O._spatial_inertia(robot, i).unsqueeze(0).repeat(B, 1, 1)
    U, d, u = [None] * N, [None] * N, [None] * N
    for i in range(N - 1, 0, -1):
        S_ = torch.cat([robot.axis[i:i + 1].expand(B, 3), zeros], dim=1)
        U[i] = (IA[i] @ S_.unsqueeze(2)).squeeze(2)
        d[i] = (S_ * U[i]).sum(-1)
        u[i] = -(pA[i] * S_).sum(-1)
        if robot.dof[i] >= 0:
            u[i] = f[:, robot.dof[i]] + u[i]
            if damping_dt != 0:
                d[i] = d[i] + damping_dt * robot.damping[i]                     # the implicit-damping pivot
            if addend is not None:
                d[i] = d[i] + addend[:, robot.dof[i]]                           # the implicit gains' pivot addend
        par = robot.parent[i]
        if par > 0:
            Ud = U[i] / (d[i].unsqueeze(1) + 1e-37)
            IAi = IA[i] - U[i].unsqueeze(2) @ Ud.unsqueeze(1)
            pa = pA[i] + (IAi @ c[i].unsqueeze(2)).squeeze(2) + U[i] * (u[i] / (d[i] + 1e-37)).unsqueeze(1)
            Rj, tj = joints[i]
            X = O._motion_matrix(Rj, tj)
            IA[par] = IA[par] + X.transpose(-2, -1) @ IAi @ X
            pl = (Rj @ pa[:, 3:].unsqueeze(2)).squeeze(2)
            pg = ((O._skew(tj.expand(B, 3)) @ Rj) @ pa[:, 3:].unsqueeze(2)).squeeze(2) + (Rj @ pa[:, :3].unsqueeze(2)).squeeze(2)
            pA[par] = pA[par] + torch.cat([pg, pl], dim=1)
    acc = [torch.cat([zeros, g], dim=1)] + [None] * (N - 1)
    cols = [None] * robot.n_dofs
    for i in range(1, N):
        Rj, tj = joints[i]
        X = O._motion_matrix(Rj, tj)
        a = (X @ acc[robot.parent[i]].unsqueeze(2)).squeeze(2) + c[i]
        if robot.dof[i] >= 0:
            qdd_i = (1.0 / d[i]) * (u[i] - (U[i] * a).sum(-1))
            cols[robot.dof[i]] = qdd_i
            a = a + torch.cat([robot.axis[i:i + 1].expand(B, 3), zeros], dim=1) * qdd_i.unsqueeze(1)
        acc[i] = a
    return torch.stack(cols, dim=1)


def gains_step(q, qd, q_ref, kp, kd, dt, qd_ref=None, f=None, effort_limit=None):
    """One step's command of DRMB200_IMPLICIT_GAINS: (u, c, sat) from the state (q, qd) and the step's inputs (each
    [B, n]; qd_ref / f / effort_limit may be None)."""
    qp = q + dt * qd
    u = kp * (q_ref - qp)
    if f is not None:
        u = f + u
    u = u + kd * ((0.0 if qd_ref is None else qd_ref) - qd)
    if effort_limit is None:
        sat = torch.zeros_like(u, dtype=torch.bool)
    else:
        sat = ~((u >= -effort_limit) & (u <= effort_limit))
        u = torch.where(sat, torch.clamp(u, -effort_limit, effort_limit), u)
    c = torch.where(sat, torch.zeros_like(u), dt * (kd + dt * kp) * torch.ones_like(u))
    return u, c, sat


def pd_rollout(robot, q0, qd0, q_ref, kp, kd, dt, qd_ref=None, f=None, effort_limit=None, include_gravity=True,
               use_damping=False, implicit_damping=False):
    """For t = 0 .. T-1: (u, c, sat) = gains_step(q_t, qd_t, ...); qdd_t = FD'(q_t, qd_t, u) with the pivot addends c
    (and the implicit-damping pivot at h = dt with implicit_damping); tau_t = sat ? u : u - c qdd_t; then the integrate.
    Returns time-major (q, qd, qdd, tau) [T, B, n].  Any dtype; differentiable."""
    q, qd = q0, qd0
    outs = ([], [], [], [])
    for t in range(q_ref.shape[0]):
        u, c, sat = gains_step(q, qd, q_ref[t], kp, kd, dt, None if qd_ref is None else qd_ref[t],
                               None if f is None else f[t], effort_limit)
        qdd = forward_dynamics(robot, q, qd, u, include_gravity, use_damping, dt if implicit_damping else 0.0, c)
        tau = torch.where(sat, u, u - c * qdd)
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, x in zip(outs, (q, qd, qdd, tau)):
            lst.append(x)
    return tuple(torch.stack(lst) for lst in outs)


def step_maps(inertia, h, kp, kd):
    """The one-joint step maps (q, qd) -> (q', qd') of semi-implicit Euler under a PD law towards 0, [..., 2, 2]: explicit
    (the law at the start of the step) and implicit (at the end).  Inputs broadcast."""
    inertia, h, kp, kd = (torch.as_tensor(x, dtype=torch.float64) for x in (inertia, h, kp, kd))
    inertia, h, kp, kd = torch.broadcast_tensors(inertia, h, kp, kd)
    a, b = h * h * kp / inertia, h * kd / inertia
    # explicit: qd' = qd + h (-kp q - kd qd) / I;  q' = q + h qd'
    ex = torch.stack([torch.stack([1 - a, h * (1 - b)], -1), torch.stack([-a / h, 1 - b], -1)], -2)
    # implicit: (I + h kd + h^2 kp) qdd = -kp (q + h qd) - kd qd, i.e. qd' = m_q q + m_qd qd with
    m_q = -(a / h) / (1 + a + b)
    m_qd = 1 - (a + b) / (1 + a + b)
    im = torch.stack([torch.stack([1 + h * m_q, h * m_qd], -1), torch.stack([m_q, m_qd], -1)], -2)
    return ex, im
