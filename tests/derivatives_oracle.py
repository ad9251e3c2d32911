"""Jacobians of the oracle's dynamics (oracle/drm_oracle.py) through torch.autograd, for the derivative tests.

Test helper module (not a conftest): imported by test_oracle_derivatives.py and test_dynamics_derivatives_gpu.py.
Rows of the oracle are independent configurations, so row i of every configuration's Jacobian is one reverse pass of
sum_b y[b, i]: n passes per function instead of one per (configuration, row)."""
import torch

from oracle import drm_oracle as O


def jacobians(fn, inputs, wrt):
    """fn(*inputs) -> [B, n]; returns {k: [B, n, n_k]} with out[k][b, i, j] = d y[b, i] / d inputs[k][b, j]."""
    xs = [x.detach().clone().requires_grad_(k in wrt) for k, x in enumerate(inputs)]
    y = fn(*xs)
    B, n = y.shape
    out = {k: torch.zeros(B, n, inputs[k].shape[1], dtype=y.dtype) for k in wrt}
    for i in range(n):
        grads = torch.autograd.grad(y[:, i].sum(), [xs[k] for k in wrt], retain_graph=i + 1 < n, allow_unused=True)
        for k, g in zip(wrt, grads):
            if g is not None:
                out[k][:, i, :] = g
    return out


def inverse_dynamics_derivatives(robot, q, qd, qdd, include_gravity=True, use_damping=True):
    """(dtau_dq, dtau_dqd) [B, n, n] of O.inverse_dynamics."""
    J = jacobians(lambda a, b, c: O.inverse_dynamics(robot, a, b, c, include_gravity, use_damping), (q, qd, qdd), (0, 1))
    return J[0], J[1]


def forward_dynamics_derivatives(robot, q, qd, f, include_gravity=True, use_damping=False):
    """(dqdd_dq, dqdd_dqd, dqdd_df) [B, n, n] of O.forward_dynamics."""
    J = jacobians(lambda a, b, c: O.forward_dynamics(robot, a, b, c, include_gravity, use_damping), (q, qd, f), (0, 1, 2))
    return J[0], J[1], J[2]


def mass_matrix(robot, q):
    """H(q): column j = ID(q, 0, e_j) without gravity or damping."""
    B, n = q.shape
    z = torch.zeros_like(q)
    return torch.stack([O.inverse_dynamics(robot, q, z, torch.eye(n, dtype=q.dtype)[j].expand(B, n), False, False)
                        for j in range(n)], dim=2)


def shortcut_forward_dynamics_derivatives(robot, q, qd, f, include_gravity=True, use_damping=False):
    """The textbook shortcut dqdd/dx = -H^-1 dtau/dx at qdd = FD(q, qd, f), dqdd/df = H^-1.  Exact only when the
    articulated-body algorithm inverts the RNEA, i.e. for symmetric inertia matrices."""
    qdd = O.forward_dynamics(robot, q, qd, f, include_gravity, use_damping).detach()
    dq, dqd = inverse_dynamics_derivatives(robot, q, qd, qdd, include_gravity, use_damping)
    Hinv = torch.linalg.inv(mass_matrix(robot, q))
    return -Hinv @ dq, -Hinv @ dqd, Hinv


def perturbed(robot, seed=99):
    """A copy of `robot` whose inertia matrices are perturbed to non-symmetric ones (5 % of each link's largest entry)."""
    import copy
    r = copy.copy(robot)
    gen = torch.Generator().manual_seed(seed)
    scale = robot.inertia.abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-6)
    noise = torch.randn(robot.inertia.shape, generator=gen, dtype=torch.float64).to(robot.inertia.dtype)
    r.inertia = robot.inertia + 0.05 * scale * noise
    return r
