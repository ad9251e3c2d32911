"""Contact dynamics and contact impulses of the oracle, for the contact tests.

Test helper module (not a conftest): imported by test_oracle_contact.py and test_contact_dynamics_gpu.py.  It restates the
definitions of include/drm_b200.h on the operational-space oracle's pieces (tests/osd_oracle.py), in any dtype:
  J, G, Jdot qd        osd_oracle.stacked_jacobian / force_response / bias_acceleration
  qdd_free             O.forward_dynamics with the call's gravity / damping
  A                    J G J^T + mu I
  dynamics             A lambda = a_ref - (J qdd_free + Jdot qd),  qdd = qdd_free + G J^T lambda,  force = lambda
  impulse              A Lambda = v_ref - J qd,                    qd_plus = qd + G J^T Lambda,   impulse = Lambda
and the kernel's solve: Jacobi equilibration s_k = |A_kk|^-1/2, Gaussian elimination with partial pivoting on S A S (ties
to the lower row), unsolved when an A_kk is zero or not finite or a pivot is not finite or has magnitude <= PIVOT_MIN.
Every function also returns the row's smallest pivot magnitude of S A S (0 when a diagonal entry is unusable)."""
import torch

import osd_oracle as S
from oracle import drm_oracle as O

PIVOT_MIN = 1e-5             # CONTACT_PIVOT_MIN of csrc/contact_dynamics.cu


def equilibrated_solve(A, rhs):
    """x [B, M], solved [B] bool, min_pivot [B] for A [B, M, M] x = rhs [B, M]; x is NaN on unsolved rows."""
    A, b = A.clone(), rhs.clone()
    B, M, _ = A.shape
    rows = torch.arange(B)
    d = torch.diagonal(A, dim1=1, dim2=2).abs()
    ok = ((d > 0) & torch.isfinite(d)).all(1)
    s = torch.where((d > 0) & torch.isfinite(d), d, torch.ones_like(d)).rsqrt()
    A = s[:, :, None] * A * s[:, None, :]
    b = s * b
    min_piv = torch.where(ok, torch.full((B,), float("inf"), dtype=A.dtype), torch.zeros(B, dtype=A.dtype))
    for k in range(M):
        p = k + torch.argmax(A[:, k:, k].abs(), dim=1)          # the first maximum: ties go to the lower row
        piv = A[rows, p, k]
        good = torch.isfinite(piv) & (piv.abs() > PIVOT_MIN)
        ok &= good
        min_piv = torch.minimum(min_piv, torch.where(torch.isfinite(piv), piv.abs(), torch.zeros_like(piv)))
        rk, rp = A[rows, k].clone(), A[rows, p].clone()
        A[rows, k], A[rows, p] = rp, rk
        bk, bp = b[rows, k].clone(), b[rows, p].clone()
        b[rows, k], b[rows, p] = bp, bk
        piv = torch.where(good, piv, torch.ones_like(piv))
        lk = A[:, k + 1:, k] / piv[:, None]
        A[:, k + 1:, k:] -= lk[:, :, None] * A[:, k:k + 1, k:]
        b[:, k + 1:] -= lk * b[:, k:k + 1]
    U = torch.triu(A)
    diag = torch.diagonal(U, dim1=1, dim2=2)
    U = U + torch.diag_embed(torch.where(ok[:, None], torch.zeros_like(diag), 1 - diag))     # unsolved rows: any solvable U
    y = torch.linalg.solve_triangular(U, b.unsqueeze(-1), upper=True).squeeze(-1)
    x = torch.where(ok[:, None], s * y, torch.full_like(y, float("nan")))
    return x, ok, min_piv


def _regularised(J, G, mu):
    A = J @ G @ J.transpose(1, 2)
    mu = torch.as_tensor(mu, dtype=A.dtype).reshape(-1, 1, 1)
    return A + mu * torch.eye(A.shape[1], dtype=A.dtype)


def respond(J, G, base, rhs, mu):
    """(base + G J^T x, x, solved, min_pivot) with x solving (J G J^T + mu I) x = rhs; NaN on unsolved rows."""
    x, ok, min_piv = equilibrated_solve(_regularised(J, G, mu), rhs)
    out = base + torch.einsum("bij,bmj,bm->bi", G, J, torch.where(ok[:, None], x, torch.zeros_like(x)))
    out = torch.where(ok[:, None], out, torch.full_like(out, float("nan")))
    return out, x, ok, min_piv


def contact_dynamics(robot, q, qd, f, links, accel_ref=None, include_gravity=True, use_damping=False, position_only=False,
                     mu=0.0):
    """(qdd [B, n], force [B, M], solved [B], min_pivot [B])."""
    J = S.stacked_jacobian(robot, q, links, position_only).detach()
    G = S.force_response(robot, q)
    qdd_free = O.forward_dynamics(robot, q, qd, f, include_gravity, use_damping).detach()
    bias = S.bias_acceleration(robot, q, qd, links, position_only).detach()
    ref = torch.zeros_like(bias) if accel_ref is None else accel_ref
    return respond(J, G, qdd_free, ref - torch.einsum("bmn,bn->bm", J, qdd_free) - bias, mu)


def contact_impulse(robot, q, qd, links, velocity_ref=None, position_only=False, mu=0.0):
    """(qd_plus [B, n], impulse [B, M], solved [B], min_pivot [B])."""
    J = S.stacked_jacobian(robot, q, links, position_only).detach()
    G = S.force_response(robot, q)
    vel = torch.einsum("bmn,bn->bm", J, qd)
    ref = torch.zeros_like(vel) if velocity_ref is None else velocity_ref
    return respond(J, G, qd, ref - vel, mu)
