// osd_common.cuh -- the per-row pieces of the operational-space dynamics, shared by operational_space.cu,
// contact_dynamics.cu and contact_rollout.cu so that they compute J, Jdot qd and J G J^T with the same arithmetic:
//   osd_walk              the kinematic walk of the union of the root -> link paths: J, J qd and Jdot qd
//   aba_unit_response     x = G tau, on the articulated inertias aba_body left behind (two O(n) sweeps)
//   osd_inverse_inertia   J G J^T, formed in the smaller of the two spaces
// The mathematics is stated at the top of operational_space.cu.
#pragma once
#include "aba_body.cuh"
#include "multi_program.cuh"

namespace drm {

constexpr int OSD_STATE = 24;          // floats of a spilled branch state: R (9), p, omega, v, alpha, a

// The kinematic walk of one row: J [M][n_u], velocity and bias [M] (this row's slot-major slots; entries of links that are
// not walked -- the root -- and of joints off a link's path are left as staged: zero).  qrow / qdrow: the row's q, qd.
// POSES: also every link's world pose, p (3) then R (9, row-major, canonical +z frame) at pose + 12 l T.
template <int T, bool POSES = false>
__device__ __forceinline__ void osd_walk(const UnionProgram& P, const float* s_tab, const float* qrow, const float* qdrow, int MR,
                                         float* J, float* vel, float* bias, float* jscr, float* st, float* pose = nullptr) {
    const MultiProgram& W = P.walk;
    const V3 zero = v3(0.f, 0.f, 0.f);
    M3 R = identity3();
    V3 p = zero, w = zero, v = zero, A = zero, a = zero;
    for (int k = 0; k < W.n_steps; ++k) {
        M3 F; V3 r;
        load_Fr(s_tab + (int)W.link[k] * DRMB200_TABLE_STRIDE, F, r);
        const int src = W.psrc[k];
        if (src < 0) {
            R = identity3(); p = w = v = A = a = zero;
        } else if (src > 0) {
            const float* s = st + (src - 1) * OSD_STATE * T;
            R = ldm(s, T); p = ldv(s + 9 * T, T); w = ldv(s + 12 * T, T); v = ldv(s + 15 * T, T);
            A = ldv(s + 18 * T, T); a = ldv(s + 21 * T, T);
        }
        const V3 d = mul(R, r);              // parent origin -> this origin, world frame, on the parent body
        p = p + d;
        v = cross_add(w, d, v);              // v_i = v_p + w_p x d
        a = a + cross_add(A, d, cross(w, cross(w, d)));     // a_i = a_p + A_p x d + w_p x (w_p x d)
        R = mul(R, F);
        const int c = W.dof[k];
        if (c >= 0) {
            float sn, cs;
            sincos_pi2(qrow[c], sn, cs);
            const V3 z = col2(R);            // joint axis in the world frame (unchanged by Rz)
            float* js = jscr + W.jslot[k] * 6 * T;
            stv(js, T, z);
            stv(js + 3 * T, T, cross(z, p));
            const float qd = qdrow[c];
            A = A + qd * cross(w, z);        // + qd dz/dt
            w = w + qd * z;
            rotate_z(R, cs, sn);
        }
        const int sv = W.save[k];
        if (sv >= 0) {
            float* s = st + sv * OSD_STATE * T;
            stm(s, T, R); stv(s + 9 * T, T, p); stv(s + 12 * T, T, w); stv(s + 15 * T, T, v);
            stv(s + 18 * T, T, A); stv(s + 21 * T, T, a);
        }
        const int l = W.ee[k];
        if (l < 0) continue;
        // link l: its rows of J, of J qd and of Jdot qd
        link_jacobian(P, l, MR, p, jscr, J, T);
        stv(vel + MR * l * T, T, v);
        stv(bias + MR * l * T, T, a);
        if (MR == 6) { stv(vel + (MR * l + 3) * T, T, w); stv(bias + (MR * l + 3) * T, T, A); }
        if (POSES) { float* ps = pose + 12 * l * T; stv(ps, T, p); stm(ps + 3 * T, T, R); }
    }
}

// x = G tau for one row: passes 2 and 3 of aba_body at zero velocity and gravity, on the U, d, cos, sin that aba_body left
// in the row's link slots (lk0).  tau / x: the row's n floats (row-major, like the ABA's f / qdd rows); sl0: its branch slots.
// Each link's u is kept in the slot aba_body used for its own u (dead once aba_body returned).
template <int T>
__device__ __forceinline__ void aba_unit_response(const TreeProgram& prog, const float* s_tab, const float* tau, float* x,
                                                  float* lk0, float* sl0) {
    const int N = prog.n_links;
    const V3 zero = v3(0.f, 0.f, 0.f);
    {   // leaves -> root
        V3 c_ang = zero, c_lin = zero;
        for (int i = N - 1; i >= 1; --i) {
            float* lk = lk0 + i * ABA_LINK * T;
            V3 p_ang = zero, p_lin = zero;
            if (i + 1 < N && prog.psrc[i + 1] == 0) { p_ang = c_ang; p_lin = c_lin; }
            const int sv = prog.save[i];
            if (sv >= 0) {
                const float* sl = sl0 + sv * ABA_SLOT * T;
                p_ang = p_ang + ldv(sl + 36 * T, T); p_lin = p_lin + ldv(sl + 39 * T, T);
            }
            const int c = prog.dof[i];
            float u = 0.f;
            if (c >= 0) u = tau[c] - p_ang.z;
            const int Pi = prog.parent[i];
            if (Pi > 0) {
                V3 pa_ang = p_ang, pa_lin = p_lin;
                M3 M; V3 r;
                load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
                if (c >= 0) {
                    const float ud = u * (1.f / (lk[13 * T] + ABA_EPS));
                    pa_ang = pa_ang + ud * ldv(lk + 6 * T, T);
                    pa_lin = pa_lin + ud * ldv(lk + 9 * T, T);
                    rotate_z(M, lk[0], lk[T]);
                }
                const V3 q_lin = mul(M, pa_lin);                       // force transform X^T
                const V3 q_ang = cross_add(r, q_lin, mul(M, pa_ang));
                if (Pi == i - 1) { c_ang = q_ang; c_lin = q_lin; }
                else {
                    float* sl = sl0 + (int)prog.save[Pi] * ABA_SLOT * T;
                    if (prog.accw[i] != 2) {
                        stv(sl + 36 * T, T, ldv(sl + 36 * T, T) + q_ang); stv(sl + 39 * T, T, ldv(sl + 39 * T, T) + q_lin);
                    } else {
                        stv(sl + 36 * T, T, q_ang); stv(sl + 39 * T, T, q_lin);
                    }
                }
            }
            lk[12 * T] = u;
        }
    }
    {   // root -> leaves
        V3 al = zero, a = zero;
        for (int i = 1; i < N; ++i) {
            M3 M; V3 r;
            load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
            const float* lk = lk0 + i * ABA_LINK * T;
            const int src = prog.psrc[i];
            V3 alp, ap;
            if (src == 0) { alp = al; ap = a; }
            else if (src < 0) { alp = zero; ap = zero; }
            else { const float* sl = sl0 + (src - 1) * ABA_SLOT * T; alp = ldv(sl, T); ap = ldv(sl + 3 * T, T); }
            const int c = prog.dof[i];
            if (c >= 0) rotate_z(M, lk[0], lk[T]);
            al = mulT(M, alp);
            a = mulT(M, cross_add(alp, r, ap));
            if (c >= 0) {
                const V3 Ua = ldv(lk + 6 * T, T), Ul = ldv(lk + 9 * T, T);
                const float u = lk[12 * T], d = lk[13 * T];
                const float xc = (1.0f / d) * (u - (dot(Ua, al) + dot(Ul, a)));
                x[c] = xc;
                al.z += xc;
            }
            const int sv = prog.save[i];
            if (sv >= 0) { float* sl = sl0 + sv * ABA_SLOT * T; stv(sl, T, al); stv(sl + 3 * T, T, a); }
        }
    }
}

// inv [M][M] (this row's slot-major slots) = J G J^T, after aba_body left U, d, cos, sin in lk0.  frow / xrow: n floats of
// the row used as the right-hand side and the response of each sweep (both overwritten).  The product is formed in the
// smaller space:  M <= n_u: M sweeps with tau = J^T e_k give the columns of G J^T;  M > n_u: n_u sweeps with tau = e_j,
// then inv += (J G e_j) J[:, j]^T.
//
// GDOT (contact_backward.cu): also sdot [M] (slot-major) = J G^T g for the row's n floats g, from the same sweeps -- entry k
// is g . (G J^T e_k) when M <= n_u; when M > n_u each sweep gives (G^T g)_j = g . (G e_j) and sdot += J[:, j] (G^T g)_j.
// The false instantiation is the code without these dot products.
template <int T, bool GDOT = false>
__device__ __forceinline__ void osd_inverse_inertia(const TreeProgram& prog, const UnionProgram& P, const float* s_tab, int M,
                                                    const float* J, float* inv, float* frow, float* xrow, float* lk0, float* sl0,
                                                    const float* g = nullptr, float* sdot = nullptr) {
    const int n = prog.n_dofs;
    const int n_u = P.n_u;
    const int rs = n_u * T;
    if (M <= n_u) {
        for (int k = 0; k < M; ++k) {       // column k: J G J^T e_k
            for (int c = 0; c < n; ++c) frow[c] = 0.f;
            for (int u = 0; u < n_u; ++u) frow[P.u_dof[u]] = J[k * rs + u * T];
            aba_unit_response<T>(prog, s_tab, frow, xrow, lk0, sl0);
            for (int m = 0; m < M; ++m) {
                float s = 0.f;
                for (int u = 0; u < n_u; ++u) s = fmaf(J[m * rs + u * T], xrow[P.u_dof[u]], s);
                inv[(m * M + k) * T] = s;
            }
            if constexpr (GDOT) {
                float s = 0.f;
                for (int c = 0; c < n; ++c) s = fmaf(g[c], xrow[c], s);
                sdot[k * T] = s;
            }
        }
    } else {
        for (int i = 0; i < M * M; ++i) inv[i * T] = 0.f;
        if constexpr (GDOT) for (int m = 0; m < M; ++m) sdot[m * T] = 0.f;
        for (int j = 0; j < n_u; ++j) {     // += (J G e_j) J[:, j]^T
            for (int c = 0; c < n; ++c) frow[c] = 0.f;
            frow[P.u_dof[j]] = 1.f;
            aba_unit_response<T>(prog, s_tab, frow, xrow, lk0, sl0);
            for (int m = 0; m < M; ++m) {
                float y = 0.f;
                for (int u = 0; u < n_u; ++u) y = fmaf(J[m * rs + u * T], xrow[P.u_dof[u]], y);
                for (int k = 0; k < M; ++k) inv[(m * M + k) * T] = fmaf(y, J[k * rs + j * T], inv[(m * M + k) * T]);
            }
            if constexpr (GDOT) {
                float t = 0.f;
                for (int c = 0; c < n; ++c) t = fmaf(g[c], xrow[c], t);
                for (int m = 0; m < M; ++m) sdot[m * T] = fmaf(J[m * rs + j * T], t, sdot[m * T]);
            }
        }
    }
}

}  // namespace drm
