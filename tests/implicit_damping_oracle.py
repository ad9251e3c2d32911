"""Reference restatement of the forward dynamics and the rollouts with implicit joint damping, for the tests.

Test helper module (not a conftest).  forward_dynamics restates oracle/drm_oracle.py: forward_dynamics with one change, the
definition of drmb200_forward_dynamics_implicit_damping (include/drm_b200.h): every movable joint's pivot d_i = S^T IA_i S
becomes d_i + h damping_i wherever it is used.  With damping_dt = 0 it is the oracle's function bit for bit (the term is not
formed).  The rollouts are the loops of rollout_oracle.py, pd_rollout_oracle.py and contact_rollout_oracle.py with that
forward dynamics at h = dt; the oracle package and those modules are unchanged."""
import torch

import contact_oracle as C
import contact_rollout_oracle as CR
import osd_oracle as S
from oracle import drm_oracle as O


def forward_dynamics(robot, q, qd, f, include_gravity=True, use_damping=True, damping_dt=0.0):
    """O.forward_dynamics with the pivot d_i + damping_dt * damping_i of every movable joint.  Any dtype; differentiable
    (the damping included, through robot.damping)."""
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


def damping_vector(robot):
    """[n]: the damping of every controlled joint, in dof order."""
    return torch.stack([robot.damping[i] for i in robot.controlled])


def forward_dynamics_rollout(robot, q0, qd0, f, dt, include_gravity=True):
    """rollout_oracle.forward_dynamics_rollout with damping, taken implicitly at h = dt."""
    q, qd = q0, qd0
    outs = ([], [], [])
    for t in range(f.shape[0]):
        qdd = forward_dynamics(robot, q, qd, f[t], include_gravity, True, dt)
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, x in zip(outs, (q, qd, qdd)):
            lst.append(x)
    return tuple(torch.stack(lst) for lst in outs)


def pd_rollout(robot, q0, qd0, q_ref, kp, kd, dt, qd_ref=None, f=None, effort_limit=None, include_gravity=True):
    """pd_rollout_oracle.pd_rollout with damping, taken implicitly at h = dt: (q, qd, qdd, tau) [T, B, n]."""
    q, qd = q0, qd0
    outs = ([], [], [], [])
    for t in range(q_ref.shape[0]):
        u = kp * (q_ref[t] - q) + kd * ((0.0 if qd_ref is None else qd_ref[t]) - qd)
        if f is not None:
            u = f[t] + u
        if effort_limit is not None:
            u = torch.maximum(torch.minimum(u, effort_limit), -effort_limit)
        qdd = forward_dynamics(robot, q, qd, u, include_gravity, True, dt)
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, x in zip(outs, (q, qd, qdd, u)):
            lst.append(x)
    return tuple(torch.stack(lst) for lst in outs)


def force_response(robot, q, damping_dt):
    """G' [B, n, n] = (H + h diag(damping))^-1 for symmetric inertias: forward_dynamics at (q, 0, e_j) without gravity or
    damping torque, with the implicit pivot (the unit-response sweeps of the contact rollout)."""
    B, n = q.shape
    eye = torch.eye(n, dtype=q.dtype)
    cols = [forward_dynamics(robot, q, torch.zeros_like(q), eye[j].expand(B, n), False, False, damping_dt) for j in range(n)]
    return torch.stack(cols, dim=2)


def contact_rollout(robot, q0, qd0, f, links, dt, omega=0.0, target_pos=None, target_quat=None, include_gravity=True,
                    position_only=False, mu=0.0):
    """contact_rollout_oracle.contact_rollout with damping, taken implicitly at h = dt: qdd_free and G are those of
    forward_dynamics(..., damping_dt=dt).  Returns (q, qd, qdd [T, B, n], force [T, B, M], solved [B])."""
    if target_pos is None:
        target_pos, target_quat = CR.poses(robot, q0, links)
    q, qd = q0, qd0
    outs = ([], [], [], [])
    ok_all = torch.ones(q0.shape[0], dtype=torch.bool)
    for t in range(f.shape[0]):
        a_ref = CR.baumgarte(robot, q, qd, links, position_only, omega, target_pos, target_quat)
        J = S.stacked_jacobian(robot, q, links, position_only).detach()
        G = force_response(robot, q, dt).detach()
        qdd_free = forward_dynamics(robot, q, qd, f[t], include_gravity, True, dt).detach()
        bias = S.bias_acceleration(robot, q, qd, links, position_only).detach()
        qdd, force, ok, _ = C.respond(J, G, qdd_free, a_ref - torch.einsum("bmn,bn->bm", J, qdd_free) - bias, mu)
        ok_all &= ok
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, x in zip(outs, (q, qd, qdd, force)):
            lst.append(x.detach())
    return (*(torch.stack(lst) for lst in outs), ok_all)
