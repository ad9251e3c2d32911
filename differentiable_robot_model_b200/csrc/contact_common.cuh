// contact_common.cuh -- the per-row body of the contact dynamics and contact impulse, shared by contact_dynamics.cu and
// contact_rollout.cu so that one contact step of a rollout is the contact kernel's arithmetic in the same order:
//   contact_solve   the equilibrated Gaussian elimination with partial pivoting of A x = b
//   contact_row     steps 1-5 of contact_dynamics.cu's header: walk, ABA, J G J^T + mu I, solve, + G J^T lambda
// The definitions are stated in include/drm_b200.h.
#pragma once
#include "osd_common.cuh"

namespace drm {

constexpr float CONTACT_PIVOT_MIN = 1e-5f;  // smallest pivot magnitude of the equilibrated system that counts as solved

// Solves A x = b for one row (slot-major A [M][M] and b [M], both overwritten; x returned in b; s: M scale slots), as stated
// in include/drm_b200.h: x = S y with (S A S) y = S b, S = diag(|A_kk|^-1/2), by Gaussian elimination with partial pivoting.
// Returns false (b then undefined) when the row is unsolved.
template <int T>
__device__ __forceinline__ bool contact_solve(float* A, float* b, float* s, int M) {
    const int rs = M * T;
    for (int k = 0; k < M; ++k) {
        const float d = fabsf(A[k * rs + k * T]);
        if (!(d > 0.f) || !isfinite(d)) return false;
        s[k * T] = 1.0f / sqrtf(d);
    }
    for (int i = 0; i < M; ++i) {
        const float si = s[i * T];
        for (int j = 0; j < M; ++j) A[i * rs + j * T] = si * A[i * rs + j * T] * s[j * T];
        b[i * T] *= si;
    }
    for (int k = 0; k < M; ++k) {
        int p = k;
        float best = fabsf(A[k * rs + k * T]);
        for (int i = k + 1; i < M; ++i) {               // strictly larger: ties go to the lower row
            const float v = fabsf(A[i * rs + k * T]);
            if (v > best) { best = v; p = i; }
        }
        const float piv = A[p * rs + k * T];
        if (!(fabsf(piv) > CONTACT_PIVOT_MIN) || !isfinite(piv)) return false;
        if (p != k) {
            for (int j = k; j < M; ++j) {
                const float t = A[k * rs + j * T]; A[k * rs + j * T] = A[p * rs + j * T]; A[p * rs + j * T] = t;
            }
            const float t = b[k * T]; b[k * T] = b[p * T]; b[p * T] = t;
        }
        const float inv = 1.0f / piv;
        for (int i = k + 1; i < M; ++i) {
            const float l = A[i * rs + k * T] * inv;
            for (int j = k + 1; j < M; ++j) A[i * rs + j * T] = fmaf(-l, A[k * rs + j * T], A[i * rs + j * T]);
            b[i * T] = fmaf(-l, b[k * T], b[i * T]);
        }
    }
    for (int i = M - 1; i >= 0; --i) {
        float x = b[i * T];
        for (int j = i + 1; j < M; ++j) x = fmaf(-A[i * rs + j * T], b[j * T], x);
        b[i * T] = x / A[i * rs + i * T];
    }
    for (int i = 0; i < M; ++i) b[i * T] *= s[i * T];
    return true;
}

// The factorisation of contact_solve, kept for a solve with the transpose (contact_backward.cu): the same float operations
// on A in the same order, so the pivot sequence and the solved decision are contact_solve's bit for bit.  On return
// (true) s holds the scales, A the LU factors of P S A S (U on and above the diagonal, the multipliers of the unit lower L
// below it, rows swapped in full) and piv[k T] the row swapped with row k at step k, as a float.
template <int T>
__device__ __forceinline__ bool contact_factor(float* A, float* s, float* piv, int M) {
    const int rs = M * T;
    for (int k = 0; k < M; ++k) {
        const float d = fabsf(A[k * rs + k * T]);
        if (!(d > 0.f) || !isfinite(d)) return false;
        s[k * T] = 1.0f / sqrtf(d);
    }
    for (int i = 0; i < M; ++i) {
        const float si = s[i * T];
        for (int j = 0; j < M; ++j) A[i * rs + j * T] = si * A[i * rs + j * T] * s[j * T];
    }
    for (int k = 0; k < M; ++k) {
        int p = k;
        float best = fabsf(A[k * rs + k * T]);
        for (int i = k + 1; i < M; ++i) {               // strictly larger: ties go to the lower row
            const float v = fabsf(A[i * rs + k * T]);
            if (v > best) { best = v; p = i; }
        }
        const float pv = A[p * rs + k * T];
        if (!(fabsf(pv) > CONTACT_PIVOT_MIN) || !isfinite(pv)) return false;
        piv[k * T] = (float)p;
        if (p != k) {
            for (int j = 0; j < M; ++j) {               // the multipliers (j < k) move with their rows
                const float t = A[k * rs + j * T]; A[k * rs + j * T] = A[p * rs + j * T]; A[p * rs + j * T] = t;
            }
        }
        const float inv = 1.0f / pv;
        for (int i = k + 1; i < M; ++i) {
            const float l = A[i * rs + k * T] * inv;
            for (int j = k + 1; j < M; ++j) A[i * rs + j * T] = fmaf(-l, A[k * rs + j * T], A[i * rs + j * T]);
            A[i * rs + k * T] = l;
        }
    }
    return true;
}

// Solves A^T x = b (b overwritten with x) on the factors contact_factor left: with A~ = S A S and P A~ = L U,
// A~^T y = S b is U^T L^T P y = S b (forward substitution with U^T, back substitution with the unit L^T, then the swaps in
// reverse order), and x = S y.
template <int T>
__device__ __forceinline__ void contact_solve_transposed(const float* A, float* b, const float* s, const float* piv, int M) {
    const int rs = M * T;
    for (int i = 0; i < M; ++i) b[i * T] *= s[i * T];
    for (int i = 0; i < M; ++i) {                       // U^T z = S b
        float x = b[i * T];
        for (int j = 0; j < i; ++j) x = fmaf(-A[j * rs + i * T], b[j * T], x);
        b[i * T] = x / A[i * rs + i * T];
    }
    for (int i = M - 1; i >= 0; --i) {                  // L^T w = z
        float x = b[i * T];
        for (int j = i + 1; j < M; ++j) x = fmaf(-A[j * rs + i * T], b[j * T], x);
        b[i * T] = x;
    }
    for (int k = M - 1; k >= 0; --k) {                  // y = P^T w
        const int p = (int)piv[k * T];
        if (p != k) { const float t = b[k * T]; b[k * T] = b[p * T]; b[p * T] = t; }
    }
    for (int i = 0; i < M; ++i) b[i * T] *= s[i * T];
}

// One row of the contact dynamics (IMPULSE: the contact impulse), thread tid of a CTA of T rows:
//   1. osd_walk: J, J qd and Jdot qd (and, with POSES, every link's pose);   then the statements AFTER_WALK, which may
//      write the row's reference slots;
//   2. aba_body: qdd_free (the impulse: at zero velocity and force, without gravity, for U, d, cos, sin only);
//   3. osd_inverse_inertia: A = J G J^T, then MU on the diagonal;
//   4. contact_solve: lambda, or unsolved;
//   5. + G J^T lambda (one more aba_unit_response); unsolved rows get NaN in out and lam.
// OK (a bool lvalue) receives whether the row was solved.  IMPLICIT (a constant) and H: aba_body's implicit damping of step H
// (dynamics only), which the unit-response sweeps then follow through the stored pivots.  The slots come from the enclosing scope's layout L: the ABA rows
// s_q / s_qd / s_f / s_qdd (row-major n floats; the f row is overwritten by the unit-response sweeps, the qdd row is
// scratch), the reference rows (L.ref, row-major M), and slot-major the ABA link and branch state (L.aba.link,
// L.aba.slots), J [M][n_u] (L.jac), the walk's joint scratch and spilled state (L.jscr, L.state), J qd and Jdot qd (L.vel,
// L.bias), lambda (L.lam), the scales (L.scale), A [M][M] (L.a), the joint output [n] (L.out) and, with POSES, the link
// poses (POSE: this row's first pose slot, see osd_walk; nullptr without POSES).  It also reads prog, P, smem, s_tab, tid,
// n, n_u, M and MR from that scope.
//
// A macro rather than a __forceinline__ function: a function is simplified on its own before it is inlined, which changes
// the contact kernel's code generation (its SASS, not its results); the macro expands to the kernel's own statements.
#define DRM_CONTACT_ROW(T, IMPULSE, POSES, POSE, FLAGS, MU, OK, IMPLICIT, H, AFTER_WALK)                                    \
    do {                                                                                                                   \
        const float* qrow = s_q + tid * n;                                                                                 \
        const float* qdrow = s_qd + tid * n;                                                                               \
        float* frow = s_f + tid * n;                                                                                       \
        float* xrow = s_qdd + tid * n;                                                                                     \
        const float* ref = smem + L.ref + tid * M;                                                                         \
        float* lk0 = smem + L.aba.link + tid;                                                                              \
        float* sl0 = smem + L.aba.slots + tid;                                                                             \
        float* J = smem + L.jac + tid;                                                                                     \
        float* vel = smem + L.vel + tid;                                                                                   \
        float* bias = smem + L.bias + tid;                                                                                 \
        float* lam = smem + L.lam + tid;                                                                                   \
        float* A = smem + L.a + tid;                                                                                       \
        float* out = smem + L.out + tid;                                                                                   \
        const int rs = n_u * T;                                                                                            \
        osd_walk<T, POSES>(P, s_tab, qrow, qdrow, MR, J, vel, bias, smem + L.jscr + tid, smem + L.state + tid, POSE);      \
        AFTER_WALK                                                                                                         \
        if (!IMPULSE) {                                                                                                    \
            aba_body<T, IMPLICIT>(prog, s_tab, qrow, qdrow, frow, xrow, lk0, sl0, FLAGS, H);                               \
            for (int m = 0; m < M; ++m) { /* a_ref - (J qdd_free + Jdot qd) */                                             \
                float s = bias[m * T];                                                                                     \
                for (int u = 0; u < n_u; ++u) s = fmaf(J[m * rs + u * T], xrow[P.u_dof[u]], s);                            \
                lam[m * T] = ref[m] - s;                                                                                   \
            }                                                                                                              \
            for (int c = 0; c < n; ++c) out[c * T] = xrow[c];                                                              \
        } else {                                                                                                           \
            aba_body<T>(prog, s_tab, qrow, frow, frow, xrow, lk0, sl0, 0u);                                                \
            for (int m = 0; m < M; ++m) lam[m * T] = ref[m] - vel[m * T]; /* v_ref - J qd */                               \
            for (int c = 0; c < n; ++c) out[c * T] = qdrow[c];                                                             \
        }                                                                                                                  \
        osd_inverse_inertia<T>(prog, P, s_tab, M, J, A, frow, xrow, lk0, sl0);                                             \
        for (int k = 0; k < M; ++k) A[(k * M + k) * T] += MU;                                                              \
        OK = contact_solve<T>(A, lam, smem + L.scale + tid, M);                                                            \
        if (OK) { /* + G J^T lambda */                                                                                     \
            for (int c = 0; c < n; ++c) frow[c] = 0.f;                                                                     \
            for (int u = 0; u < n_u; ++u) {                                                                                \
                float s = 0.f;                                                                                             \
                for (int m = 0; m < M; ++m) s = fmaf(J[m * rs + u * T], lam[m * T], s);                                    \
                frow[P.u_dof[u]] = s;                                                                                      \
            }                                                                                                              \
            aba_unit_response<T>(prog, s_tab, frow, xrow, lk0, sl0);                                                       \
            for (int c = 0; c < n; ++c) out[c * T] += xrow[c];                                                             \
        } else {                                                                                                           \
            for (int c = 0; c < n; ++c) out[c * T] = __int_as_float(0x7fc00000);                                           \
            for (int m = 0; m < M; ++m) lam[m * T] = __int_as_float(0x7fc00000);                                           \
        }                                                                                                                  \
    } while (0)

}  // namespace drm
