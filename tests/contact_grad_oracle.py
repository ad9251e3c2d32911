"""Differentiable contact dynamics and contact impulses of the fp64 oracle, and the adjoint formula in torch.

Test helper module (not a conftest): imported by test_oracle_contact_grad.py and test_contact_backward_gpu.py.

* ``dynamics`` / ``impulse`` restate the definitions of include/drm_b200.h so that torch autograd differentiates them
  w.r.t. q, qd, f, the reference and every Robot field: J from ``O.jacobian``, G from the columns
  ``O.forward_dynamics(q, 0, e_j, False, False)``, ``Jdot qd`` by ``torch.func.jvp`` and the solve by ``torch.linalg.solve``
  (rows the caller marks unsolved get an identity system and zero outputs, so they never poison a batch sum).
* ``adjoint_dynamics`` / ``adjoint_impulse`` are the three-stage formula of include/drm_b200.h written in torch: the
  transposed solve for nu, the forward-dynamics adjoint (autograd of O.forward_dynamics with lambda held) for g^, and the
  kinematic term phi = lambda^T J tau^ - nu^T (J qdd + Jdot qd) with lambda, nu, tau^, qdd held constant."""
import torch

import osd_oracle as S
from oracle import drm_oracle as O


def force_response(robot, q):
    """G [B, n, n] with G[:, :, j] = O.forward_dynamics(q, 0, e_j) without gravity or damping; differentiable."""
    B, n = q.shape
    eye = torch.eye(n, dtype=q.dtype).repeat(B, 1)
    qr = q.repeat_interleave(n, 0)
    cols = O.forward_dynamics(robot, qr, torch.zeros_like(qr), eye, False, False)
    return cols.reshape(B, n, n).transpose(1, 2)


def bias_acceleration(robot, q, qd, links, position_only):
    def jqd(x):
        return torch.einsum("bmn,bn->bm", S.stacked_jacobian(robot, x, links, position_only), qd)
    return torch.func.jvp(jqd, (q,), (qd,))[1]


def _solve(A, rhs, ok):
    eye = torch.eye(A.shape[1], dtype=A.dtype).expand_as(A)
    A = torch.where(ok[:, None, None], A, eye)
    x = torch.linalg.solve(A, rhs.unsqueeze(-1)).squeeze(-1)
    return torch.where(ok[:, None], x, torch.zeros_like(x))


def dynamics(robot, q, qd, f, links, accel_ref=None, include_gravity=True, use_damping=False, position_only=False, mu=0.0,
             ok=None):
    """(qdd [B, n], force [B, M]); rows with ok False get zeros."""
    J = S.stacked_jacobian(robot, q, links, position_only)
    G = force_response(robot, q)
    free = O.forward_dynamics(robot, q, qd, f, include_gravity, use_damping)
    bias = bias_acceleration(robot, q, qd, links, position_only)
    ref = torch.zeros_like(bias) if accel_ref is None else accel_ref
    A = J @ G @ J.transpose(1, 2) + mu * torch.eye(J.shape[1], dtype=q.dtype)
    ok = torch.ones(q.shape[0], dtype=torch.bool) if ok is None else ok
    lam = _solve(A, ref - torch.einsum("bmn,bn->bm", J, free) - bias, ok)
    qdd = free + torch.einsum("bij,bmj,bm->bi", G, J, lam)
    return torch.where(ok[:, None], qdd, torch.zeros_like(qdd)), lam


def impulse(robot, q, qd, links, velocity_ref=None, position_only=False, mu=0.0, ok=None):
    """(qd_plus [B, n], impulse [B, M]); rows with ok False get zeros."""
    J = S.stacked_jacobian(robot, q, links, position_only)
    G = force_response(robot, q)
    vel = torch.einsum("bmn,bn->bm", J, qd)
    ref = torch.zeros_like(vel) if velocity_ref is None else velocity_ref
    A = J @ G @ J.transpose(1, 2) + mu * torch.eye(J.shape[1], dtype=q.dtype)
    ok = torch.ones(q.shape[0], dtype=torch.bool) if ok is None else ok
    lam = _solve(A, ref - vel, ok)
    qdp = qd + torch.einsum("bij,bmj,bm->bi", G, J, lam)
    return torch.where(ok[:, None], qdp, torch.zeros_like(qdp)), lam


def _grads(out, wrt, g):
    got = torch.autograd.grad(out, wrt, g, allow_unused=True)
    return [torch.zeros_like(w) if x is None else x for w, x in zip(wrt, got)]


def adjoint_dynamics(robot, q, qd, f, links, g_qdd, g_force, accel_ref=None, include_gravity=True, use_damping=False,
                     position_only=False, mu=0.0, params=()):
    """The three-stage formula: (q_grad, qd_grad, f_grad, accel_ref_grad, [grad of each tensor in params])."""
    q, qd, f = (t.detach().requires_grad_(True) for t in (q, qd, f))
    with torch.no_grad():
        J = S.stacked_jacobian(robot, q, links, position_only)
        G = force_response(robot, q)
        qdd, lam = dynamics(robot, q, qd, f, links, accel_ref, include_gravity, use_damping, position_only, mu)
        A = J @ G @ J.transpose(1, 2) + mu * torch.eye(J.shape[1], dtype=q.dtype)
        s = g_force + torch.einsum("bmn,bkn,bk->bm", J, G, g_qdd)                 # J G^T g
        nu = torch.linalg.solve(A.transpose(1, 2), s.unsqueeze(-1)).squeeze(-1)
        ghat = g_qdd - torch.einsum("bmn,bm->bn", J, nu)
        tauc = f + torch.einsum("bmn,bm->bn", J, lam)
    tauc = tauc.requires_grad_(True)
    wrt = [q, qd, tauc] + list(params)
    fd = _grads(O.forward_dynamics(robot, q, qd, tauc, include_gravity, use_damping), wrt, ghat)
    taubar = fd[2]
    Jq = S.stacked_jacobian(robot, q, links, position_only)
    phi = (torch.einsum("bm,bmn,bn->", lam, Jq, taubar)
           - torch.einsum("bm,bmn,bn->", nu, Jq, qdd) - (nu * bias_acceleration(robot, q, qd, links, position_only)).sum())
    kin = torch.autograd.grad(phi, [q, qd] + list(params), allow_unused=True)
    kin = [torch.zeros_like(w) if x is None else x for w, x in zip([q, qd] + list(params), kin)]
    return (fd[0] + kin[0], fd[1] + kin[1], taubar, nu, [a + b for a, b in zip(fd[3:], kin[2:])])


def adjoint_impulse(robot, q, qd, links, g_qdp, g_imp, velocity_ref=None, position_only=False, mu=0.0, params=()):
    """The impulse's formula: (q_grad, qd_grad, velocity_ref_grad, [grad of each tensor in params])."""
    q = q.detach().requires_grad_(True)
    with torch.no_grad():
        J = S.stacked_jacobian(robot, q, links, position_only)
        G = force_response(robot, q)
        qdp, lam = impulse(robot, q, qd, links, velocity_ref, position_only, mu)
        A = J @ G @ J.transpose(1, 2) + mu * torch.eye(J.shape[1], dtype=q.dtype)
        s = g_imp + torch.einsum("bmn,bkn,bk->bm", J, G, g_qdp)
        nu = torch.linalg.solve(A.transpose(1, 2), s.unsqueeze(-1)).squeeze(-1)
        ghat = g_qdp - torch.einsum("bmn,bm->bn", J, nu)
        tauc = torch.einsum("bmn,bm->bn", J, lam)
    tauc = tauc.requires_grad_(True)
    wrt = [q, tauc] + list(params)
    fd = _grads(O.forward_dynamics(robot, q, torch.zeros_like(qd), tauc, False, False), wrt, ghat)
    taubar = fd[1]
    Jq = S.stacked_jacobian(robot, q, links, position_only)
    phi = torch.einsum("bm,bmn,bn->", lam, Jq, taubar) - torch.einsum("bm,bmn,bn->", nu, Jq, qdp)
    kin = torch.autograd.grad(phi, [q] + list(params), allow_unused=True)
    kin = [torch.zeros_like(w) if x is None else x for w, x in zip([q] + list(params), kin)]
    return fd[0] + kin[0], ghat, nu, [a + b for a, b in zip(fd[2:], kin[1:])]
