"""Reference restatement of a PD-controlled rollout for the tests: semi-implicit Euler over the oracle's articulated-body
algorithm (oracle/drm_oracle.py: forward_dynamics) driven by a diagonal joint-space PD law, the definition
drmb200_pd_rollout implements.  Kept beside the tests that use it; the oracle package itself is unchanged."""
import torch

from oracle import drm_oracle as O


def pd_rollout(robot, q0, qd0, q_ref, kp, kd, dt, qd_ref=None, f=None, effort_limit=None, include_gravity=True,
               use_damping=False):
    """For t = 0 .. T-1: u = f[t] + kp (q_ref[t] - q_t) + kd (qd_ref[t] - qd_t); tau_t = clamp(u, -lim, lim);
    qdd_t = FD(q_t, qd_t, tau_t); qd_{t+1} = qd_t + dt qdd_t; q_{t+1} = q_t + dt qd_{t+1}.  kp / kd [n] or [B, n]; qd_ref,
    f, effort_limit may be None (zero, zero, no limit).  Returns time-major (q, qd, qdd, tau) [T, B, n] with q[t] = q_{t+1},
    qd[t] = qd_{t+1}, qdd[t] = qdd_t, tau[t] = tau_t.  Any dtype; differentiable."""
    q, qd = q0, qd0
    outs = ([], [], [], [])
    for t in range(q_ref.shape[0]):
        u = kp * (q_ref[t] - q)
        if f is not None:
            u = f[t] + u
        u = u + kd * ((0.0 if qd_ref is None else qd_ref[t]) - qd)
        if effort_limit is not None:
            u = torch.clamp(u, -effort_limit, effort_limit)
        qdd = O.forward_dynamics(robot, q, qd, u, include_gravity, use_damping)
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, v in zip(outs, (q, qd, qdd, u)):
            lst.append(v)
    if not outs[0]:
        empty = q0.new_zeros((0,) + tuple(q0.shape))
        return empty, empty.clone(), empty.clone(), empty.clone()
    return tuple(torch.stack(lst) for lst in outs)
