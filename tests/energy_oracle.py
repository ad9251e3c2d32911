"""Energy, generalized momentum and centre of mass of the oracle's robots (oracle/drm_oracle.py), for the energy tests.

Test helper module (not a conftest): imported by test_oracle_energy.py and test_energy_momentum_gpu.py.
It restates the definitions of include/drm_b200.h (drmb200_energy_momentum) literally on O.kinematic_state and
O._inertia_times: every subtree sum is formed link by link, about the joint's own origin."""
import torch

from oracle import drm_oracle as O

GRAVITY = 9.81


def _mv(R, x):
    return (R @ x.unsqueeze(-1)).squeeze(-1)


def subtrees(robot):
    """sub[j]: link j and its descendants (parent[i] < i)."""
    N = len(robot.names)
    sub = [[i] for i in range(N)]
    for i in range(N - 1, 0, -1):
        sub[robot.parent[i]].extend(sub[i])
    return sub


def energy_momentum(robot, q, qd=None):
    """(kinetic [B], potential [B], momentum [B, n], com [B, 3], com_velocity [B, 3], com_jacobian [B, 3, n]) in the dtype of
    q; the velocity-dependent entries are None without qd."""
    B, n, N = q.shape[0], robot.n_dofs, len(robot.names)
    dt = q.dtype
    R, p, w, v, _ = O.kinematic_state(robot, q, qd)
    R = [r.expand(B, 3, 3) for r in R]
    m = robot.mass.to(dt)
    mc = robot.com.to(dt) * m[:, None]
    M = m.sum()
    h = [m[i] * p[i] + _mv(R[i], mc[i].expand(B, 3)) for i in range(N)]           # first moments, world frame
    lin, ang, kin = [], [], torch.zeros(B, dtype=dt)
    for i in range(N):
        f_lin, f_ang = O._inertia_times(robot, i, w[i], v[i])
        kin = kin + 0.5 * ((v[i] * f_lin).sum(-1) + (w[i] * f_ang).sum(-1))
        lin.append(_mv(R[i], f_lin))
        ang.append(_mv(R[i], f_ang))
    massive = bool(M != 0)
    inv_M = 1.0 / M if massive else torch.zeros((), dtype=dt)
    h_sum = torch.stack(h).sum(0)
    potential = GRAVITY * h_sum[:, 2]
    com = h_sum * inv_M
    sub = subtrees(robot)
    mom = torch.zeros(B, n, dtype=dt)
    jcom = torch.zeros(B, 3, n, dtype=dt)
    for j in robot.controlled:
        z = _mv(R[j], robot.axis[j].to(dt).expand(B, 3))
        pj = p[j]
        moment = sum(ang[i] + torch.cross(p[i] - pj, lin[i], dim=-1) for i in sub[j])
        mom[:, robot.dof[j]] = (z * moment).sum(-1)
        first = sum(h[i] for i in sub[j]) - sum(m[i] for i in sub[j]) * pj
        jcom[:, :, robot.dof[j]] = torch.cross(z, first, dim=-1) * inv_M
    if qd is None:
        return None, potential, None, com, None, jcom
    return kin, potential, mom, com, torch.stack(lin).sum(0) * inv_M, jcom


def total_mass(robot):
    return float(robot.mass.sum())
