"""Reference restatement of a forward-dynamics rollout for the tests: semi-implicit Euler over the oracle's
articulated-body algorithm (oracle/drm_oracle.py: forward_dynamics), the definition drmb200_forward_dynamics_rollout
implements.  Kept beside the tests that use it; the oracle package itself is unchanged."""
import torch

from oracle import drm_oracle as O


def forward_dynamics_rollout(robot, q0, qd0, f, dt, include_gravity=True, use_damping=False):
    """For t = 0 .. T-1: qdd_t = FD(q_t, qd_t, f[t]); qd_{t+1} = qd_t + dt qdd_t; q_{t+1} = q_t + dt qd_{t+1}.  Returns
    time-major (q, qd, qdd) [T, B, n] with q[t] = q_{t+1}, qd[t] = qd_{t+1}, qdd[t] = qdd_t.  Any dtype; differentiable."""
    q, qd = q0, qd0
    qs, qds, qdds = [], [], []
    for t in range(f.shape[0]):
        qdd = O.forward_dynamics(robot, q, qd, f[t], include_gravity, use_damping)
        qd = qd + dt * qdd
        q = q + dt * qd
        qs.append(q)
        qds.append(qd)
        qdds.append(qdd)
    if not qs:
        empty = q0.new_zeros((0,) + tuple(q0.shape))
        return empty, empty.clone(), empty.clone()
    return torch.stack(qs), torch.stack(qds), torch.stack(qdds)
