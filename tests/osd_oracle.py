"""Operational-space dynamics of the oracle (oracle/drm_oracle.py), for the operational-space tests.

Test helper module (not a conftest): imported by test_oracle_osd.py and test_operational_space_gpu.py.  Built only from
the existing oracle, in any dtype:
  J            O.jacobian of every link, stacked link by link (linear rows over angular rows; linear only for position_only)
  G            dqdd_df, the Jacobian of O.forward_dynamics w.r.t. f (derivatives_oracle.jacobians)
  qdd          O.forward_dynamics
  Jdot qd      torch.func.jvp of q -> J(q) qd in the direction qd
and returns (inv_inertia = J G J^T [B, M, M], acceleration = J qdd + Jdot qd, velocity = J qd, bias = Jdot qd [B, M])."""
import torch

import derivatives_oracle as D
from oracle import drm_oracle as O


def stacked_jacobian(robot, q, links, position_only=False):
    """[B, M, n]: the links' Jacobians stacked in list order."""
    blocks = []
    for name in links:
        lin, ang = O.jacobian(robot, q, name)
        blocks.append(lin if position_only else torch.cat([lin, ang], dim=1))
    return torch.cat(blocks, dim=1)


def force_response(robot, q):
    """G [B, n, n]: G[:, :, j] = O.forward_dynamics(q, 0, e_j) without gravity or damping (dqdd_df)."""
    z = torch.zeros_like(q)
    return D.jacobians(lambda a, b, c: O.forward_dynamics(robot, a, b, c, False, False), (q, z, z), (2,))[2]


def bias_acceleration(robot, q, qd, links, position_only=False):
    """Jdot qd [B, M] = d/dt (J(q) qd) at qdd = 0, by forward-mode differentiation in the direction qd."""
    def jqd(x):
        return torch.einsum("bmn,bn->bm", stacked_jacobian(robot, x, links, position_only), qd)
    return torch.func.jvp(jqd, (q,), (qd,))[1]


def operational_space_dynamics(robot, q, qd, f, links, include_gravity=True, use_damping=False, position_only=False):
    J = stacked_jacobian(robot, q, links, position_only)
    G = force_response(robot, q)
    qdd = O.forward_dynamics(robot, q, qd, f, include_gravity, use_damping)
    bias = bias_acceleration(robot, q, qd, links, position_only)
    inv = J @ G @ J.transpose(1, 2)
    acc = torch.einsum("bmn,bn->bm", J, qdd) + bias
    vel = torch.einsum("bmn,bn->bm", J, qd)
    return tuple(t.detach() for t in (inv, acc, vel, bias))
