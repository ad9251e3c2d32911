"""The joint-torque regressor of the oracle's inverse dynamics (oracle/drm_oracle.py), for the regressor tests.

Test helper module (not a conftest): imported by test_oracle_regressor.py and test_dynamics_regressor_gpu.py.
The oracle's RNEA re-parametrised by the link table's inertial columns pi [N, 14] = (I_o 9 | mc 3 | m | damping): the
motion state comes from O.dynamic_state (it does not depend on pi), the force pass is restated with pi per row, and
Y[b, i, l, k] = d tau[b, i] / d pi[b, l, k] by autograd (tau is linear in pi, so this is exact)."""
import torch

from oracle import drm_oracle as O


def table_params(robot):
    """pi [N, 14]: the link table's columns 12:26 of the oracle robot."""
    return O.link_table(robot)[:, 12:26]


def _cross(a, b):
    return torch.cross(a, b, dim=-1)


def inverse_dynamics_of(robot, pi, q, qd, qdd, include_gravity=True, use_damping=True):
    """tau [B, n] of the oracle's RNEA with the inertial parameters pi [B, N, 14] (one set per row)."""
    B, N = q.shape[0], len(robot.names)
    s = O.dynamic_state(robot, q, qd, qdd, include_gravity, use_damping)
    _, _, _, _, joints = O.kinematic_state(robot, q, qd)
    w, v, al, a = s["vel_ang"], s["vel_lin"], s["acc_ang"], s["acc_lin"]

    def inertia_times(i, ang, lin):                    # _inertia_times with (I_o, mc, m) taken from pi
        Io, mc, m = pi[:, i, :9].reshape(B, 3, 3), pi[:, i, 9:12], pi[:, i, 12:13]
        return m * lin - _cross(mc, ang), (Io @ ang.unsqueeze(2)).squeeze(2) + _cross(mc, lin)

    zeros = torch.zeros(B, 3, dtype=q.dtype)
    f_lin = [zeros for _ in range(N)]
    f_ang = [zeros for _ in range(N)]
    for i in range(N - 1, 0, -1):
        Rj, tj = joints[i]
        ia_lin, ia_ang = inertia_times(i, al[i], a[i])
        iv_lin, iv_ang = inertia_times(i, w[i], v[i])
        f_lin[i] = f_lin[i] + ia_lin + _cross(w[i], iv_lin)
        f_ang[i] = f_ang[i] + ia_ang + _cross(w[i], iv_ang) + _cross(v[i], iv_lin)
        par = robot.parent[i]
        new_lin = (Rj @ f_lin[i].unsqueeze(2)).squeeze(2)
        new_ang = _cross(tj.expand(B, 3), new_lin) + (Rj @ f_ang[i].unsqueeze(2)).squeeze(2)
        f_lin[par] = f_lin[par] + new_lin
        f_ang[par] = f_ang[par] + new_ang
    cols = []
    for i in robot.controlled:
        ax = robot.axis[i]
        k = int(torch.where(ax != 0)[0])
        cols.append(torch.sign(ax[k]) * f_ang[i][:, k])
    tau = torch.stack(cols, dim=1) if cols else q.new_zeros(B, 0)
    if use_damping and cols:
        tau = tau + torch.stack([pi[:, i, 13] for i in robot.controlled], dim=1) * qd
    return tau


def regressor(robot, q, qd, qdd, include_gravity=True, use_damping=True):
    """Y [B, n, N, 14] with Y[b, i, l, k] = d tau_i / d table[l, 12 + k] of O.inverse_dynamics."""
    B, n, N = q.shape[0], robot.n_dofs, len(robot.names)
    pi = table_params(robot).to(q.dtype).detach().expand(B, N, 14).clone().requires_grad_(True)
    tau = inverse_dynamics_of(robot, pi, q, qd, qdd, include_gravity, use_damping)
    Y = torch.zeros(B, n, N, 14, dtype=q.dtype)
    for i in range(n):
        g, = torch.autograd.grad(tau[:, i].sum(), [pi], retain_graph=i + 1 < n, allow_unused=True)
        if g is not None:
            Y[:, i] = g
    return Y


def urdf_parameter_jacobians(Y, mass, com):
    """The regressor mapped to the URDF parameters of every link by the chain rule, for I_o = I_c + m S(c) S(c)^T, mc = m c:
      d tau / d I_c = Y_Io,   d tau / d m = Y_m + c . Y_mc + (S S^T) : Y_Io,
      d tau / d c   = m Y_mc + m (2 c tr(Y_Io) - Y_Io c - Y_Io^T c),    d tau / d damping = Y_d.
    Y [B, n, N, 14], mass [N], com [N, 3] -> dict of [B, n, N] (mass, damping), [B, n, N, 3] (com), [B, n, N, 3, 3]."""
    YI, Ymc, Ym, Yd = Y[..., :9].unflatten(-1, (3, 3)), Y[..., 9:12], Y[..., 12], Y[..., 13]
    m, c = mass.to(Y.dtype), com.to(Y.dtype)
    SSt = (c * c).sum(-1)[:, None, None] * torch.eye(3, dtype=Y.dtype) - c[:, :, None] * c[:, None, :]      # [N, 3, 3]
    d_m = Ym + (Ymc * c).sum(-1) + (YI * SSt).sum((-1, -2))
    tr = YI.diagonal(dim1=-2, dim2=-1).sum(-1)
    d_c = m[:, None] * Ymc + m[:, None] * (2 * c * tr[..., None] - (YI @ c[..., None]).squeeze(-1)
                                           - (YI.transpose(-1, -2) @ c[..., None]).squeeze(-1))
    return {"inertia_mat": YI, "mass": d_m, "com": d_c, "joint_damping": Yd}


def structural_zeros(robot, use_damping):
    """Boolean mask [n, N, 14] of the entries that are zero for every configuration: the root's columns, links outside
    the subtree of dof i's link, fixed links' damping and, without damping, every damping column."""
    n, N = robot.n_dofs, len(robot.names)
    mask = torch.ones(n, N, 14, dtype=torch.bool)
    for l in range(1, N):
        k = l
        while k > 0:                                   # dofs of l's movable ancestors-or-self
            if robot.dof[k] >= 0:
                mask[robot.dof[k], l, :13] = False
            k = robot.parent[k]
        if use_damping and robot.dof[l] >= 0:
            mask[robot.dof[l], l, 13] = False
    return mask
