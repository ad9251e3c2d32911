"""Contact-constrained rollouts of the oracle, for the contact-rollout tests.

Test helper module (not a conftest): imported by test_oracle_contact_rollout.py and test_contact_rollout_gpu.py.  It restates
the loop of include/drm_b200.h (drmb200_contact_rollout) on the contact oracle (tests/contact_oracle.py), in any dtype:
  e        per link p - p* and, in pose mode, the world-frame rotation vector of R R*^T, the shorter way round
  a_ref    -(2 w) J qd - (w^2) e   (w = 0: a_ref = 0)
  step     (qdd, force, ok) = contact_dynamics(q, qd, f[t], a_ref);  qd = qd + dt qdd;  q = q + dt qd
Targets default to the links' poses at q0."""
import torch

import contact_oracle as C
import osd_oracle as S
from oracle import drm_oracle as O


def quat_mul(a, b):
    """Hamilton product of xyzw quaternions [..., 4]."""
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                        aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)


def rotvec_error(quat, target):
    """The world-frame rotation vector of R R*^T, the shorter way round, from xyzw quaternions [B, 4] (target normalised)."""
    target = target / target.norm(dim=-1, keepdim=True)
    conj = target * torch.tensor([-1, -1, -1, 1], dtype=target.dtype)
    qe = quat_mul(quat, conj)
    qe = torch.where(qe[:, 3:] < 0, -qe, qe)
    s = qe[:, :3].norm(dim=-1, keepdim=True)
    g = torch.where(s > 0, 2 * torch.atan2(s, qe[:, 3:]) / s.clamp_min(1e-300), torch.zeros_like(s))
    return g * qe[:, :3]


def poses(robot, q, links):
    """(positions [E, B, 3], quaternions [E, B, 4] xyzw) of the links."""
    out = [O.forward_kinematics(robot, q, name) for name in links]
    return torch.stack([p for p, _ in out]), torch.stack([r for _, r in out])


def baumgarte(robot, q, qd, links, position_only, omega, target_pos, target_quat):
    """a_ref [B, M] = -(2 omega) J qd - (omega^2) e at (q, qd)."""
    J = S.stacked_jacobian(robot, q, links, position_only).detach()
    v = torch.einsum("bmn,bn->bm", J, qd)
    if omega == 0:
        return torch.zeros_like(v)
    pos, quat = poses(robot, q, links)
    blocks = []
    for l in range(len(links)):
        blocks.append(pos[l] - target_pos[l])
        if not position_only:
            blocks.append(rotvec_error(quat[l], target_quat[l]))
    e = torch.cat(blocks, dim=1)
    return -(2 * omega) * v - (omega * omega) * e


def contact_rollout(robot, q0, qd0, f, links, dt, omega=0.0, target_pos=None, target_quat=None, include_gravity=True,
                    use_damping=False, position_only=False, mu=0.0, teacher=None):
    """(q, qd, qdd [T, B, n], force, accel_ref [T, B, M], solved [B], min_pivot [B]: the smallest scaled pivot over the
    steps).  teacher = (q_t, qd_t) [T, B, n] evaluates every step at the given states instead of the oracle's own (teacher
    forcing); q / qd then hold the integrated single steps."""
    if target_pos is None:
        target_pos, target_quat = poses(robot, q0, links)
    q, qd = q0, qd0
    outs = ([], [], [], [], [])
    ok_all = torch.ones(q0.shape[0], dtype=torch.bool)
    min_piv = torch.full((q0.shape[0],), float("inf"), dtype=q0.dtype)
    for t in range(f.shape[0]):
        if teacher is not None:
            q, qd = teacher[0][t], teacher[1][t]
        a_ref = baumgarte(robot, q, qd, links, position_only, omega, target_pos, target_quat)
        qdd, force, ok, piv = C.contact_dynamics(robot, q, qd, f[t], links, a_ref, include_gravity, use_damping, position_only,
                                                 mu)
        ok_all &= ok
        min_piv = torch.minimum(min_piv, torch.nan_to_num(piv.to(min_piv.dtype), nan=0.0))
        qd = qd + dt * qdd
        q = q + dt * qd
        for lst, v in zip(outs, (q, qd, qdd, force, a_ref)):
            lst.append(v.detach())
    return (*(torch.stack(lst) for lst in outs), ok_all, min_piv)
