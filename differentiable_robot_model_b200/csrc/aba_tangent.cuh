// aba_tangent.cuh -- forward-mode (tangent) articulated-body algorithm for one (configuration, column j): the primal of
// aba_body.cuh plus three tangent lanes, carried through every pass of the reference's arithmetic:
//   lane 0   dq  = e_j    ->  column j of d qdd / d q
//   lane 1   dqd = e_j    ->  column j of d qdd / d qd
//   lane f   df  = e_j    ->  column j of d qdd / d f  (= ABA(q, 0, e_j) without gravity or damping: ABA is affine in f)
// Only lane 0 moves the articulated inertias (they depend on q alone); lane 1 and lane f only move velocities, biases and
// accelerations.  The primal repeats aba_body()'s operations (general 6x6 inertias, U = IA S as a column in both places,
// the 1e-37 regularisers), so the tangents are the exact derivatives of what the forward-dynamics kernel evaluates, for
// non-symmetric inertia matrices too.  aba_body.cuh itself is left untouched: the forward and rollout kernels keep their code.
//
// Rotation derivatives in the canonical joint frames (M = F~ Rz(q), joint axis e_z, K = skew(e_z)):
//   d(M^T x)/dq = (M^T x) x e_z          d(M x)/dq = M (e_z x x)          d(M Z M^T)/dq = M (K Z - Z K) M^T
// so a joint's own angle enters its link step through three cheap corrections, and only in the thread whose column is
// that joint.
#pragma once
#include "aba_body.cuh"

namespace drm {

constexpr int FDD_LINK = 32;     // floats per link and thread (see the layout in aba_tangent_body)
constexpr int FDD_SLOT = 96;     // floats per branch slot and thread (pass 2: IA, pA, dIA, dpA x 2, dpA_f)

__device__ __forceinline__ V3 zc1(V3 a) { return v3(a.y, -a.x, 0.f); }         // a x e_z
__device__ __forceinline__ V3 ezx(V3 a) { return v3(-a.y, a.x, 0.f); }         // e_z x a
__device__ __forceinline__ M3 kcomm(const M3& Z) {                            // K Z - Z K, K = skew(e_z)
    // K Z: row0 = -row1(Z), row1 = row0(Z), row2 = 0;  Z K: col0 = col1(Z), col1 = -col0(Z), col2 = 0
    M3 r;
    r.a00 = -Z.a10 - Z.a01; r.a01 = -Z.a11 + Z.a00; r.a02 = -Z.a12;
    r.a10 = Z.a00 - Z.a11;  r.a11 = Z.a01 + Z.a10;  r.a12 = Z.a02;
    r.a20 = -Z.a21;         r.a21 = Z.a20;          r.a22 = 0.f;
    return r;
}
// X^T IA X for the motion transform of a link (the blocks of aba_body's pass 2, scalar form)
__device__ __forceinline__ void xform6(const M3& M, V3 r, const M3& A, const M3& B, const M3& C, const M3& D,
                                       M3& Ya, M3& Yb, M3& Yc, M3& Yd) {
    Ya = conj_by(M, A); Yb = conj_by(M, B); Yc = conj_by(M, C); Yd = conj_by(M, D);
    Ya = Ya + left_cross(r, Yc);
    Yb = Yb + left_cross(r, Yd);
    Ya = Ya - right_cross(Yb, r);
    Yc = Yc - right_cross(Yd, r);
}
__device__ __forceinline__ V3 mul2v(const M3& A, V3 x, const M3& B, V3 y) { return mul_add(A, x, mul(B, y)); }   // A x + B y

// One thread: configuration rows qrow / qdrow / frow, column j.  Outputs (may be null): column j of the three matrices,
// element (c, j) at o[c * n].  lk0 / sl0: this thread's column of the per-link / branch-slot regions, stride S.
__device__ __forceinline__ void aba_tangent_body(const TreeProgram& prog, const float* s_tab, const float* qrow,
                                                 const float* qdrow, const float* frow, int j, int n, float* o_q,
                                                 float* o_qd, float* o_f, float* lk0, float* sl0, int S, uint32_t flags) {
    const int N = prog.n_links;
    const float g = (flags & DRMB200_GRAVITY) ? ABA_GRAVITY : 0.f;
    const bool damp = (flags & DRMB200_DAMPING) != 0;
    const V3 zero = v3(0.f, 0.f, 0.f);
    // per-link layout (x S):  0 cs, 1 sn, 2..5 c = (ca.x, ca.y, cl.x, cl.y), 6..11 pA -> U, 12..15 dc lane 0,
    //   16..19 dc lane 1, 20..25 dpA lane 0 -> dU, 26..31 dpA lane 1 -> (u, d, du0, du1, dd, u_f)

    // ---- pass 1: root -> leaves, velocities, c and pA, and their tangents -----------------------------------------
    {
        V3 w = zero, v = zero, tw0 = zero, tv0 = zero, tw1 = zero, tv1 = zero;
        for (int i = 1; i < N; ++i) {
            const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
            const int src = prog.psrc[i];
            V3 wp, vp, twp0, tvp0, twp1, tvp1;
            if (src == 0) { wp = w; vp = v; twp0 = tw0; tvp0 = tv0; twp1 = tw1; tvp1 = tv1; }
            else if (src < 0) { wp = vp = twp0 = tvp0 = twp1 = tvp1 = zero; }
            else {
                const float* sl = sl0 + (src - 1) * FDD_SLOT * S;
                wp = ldv(sl, S); vp = ldv(sl + 3 * S, S); twp0 = ldv(sl + 6 * S, S); tvp0 = ldv(sl + 9 * S, S);
                twp1 = ldv(sl + 12 * S, S); tvp1 = ldv(sl + 15 * S, S);
            }
            M3 M = C.F;
            const int c = prog.dof[i];
            float cs = 1.f, sn = 0.f, qd_k = 0.f;
            if (c >= 0) {
                qd_k = qdrow[c];
                sincos_pi2(qrow[c], sn, cs);
                rotate_z(M, cs, sn);
            }
            const bool own = (c == j);
            const V3 Ew = mulT(M, wp), Ev = mulT(M, cross_add(wp, C.r, vp));
            w = Ew; w.z += qd_k;
            v = Ev;
            const V3 ca = cross_z(w, qd_k), cl = cross_z(v, qd_k);
            const V3 hl = C.m * v - cross(C.mc, w);
            const V3 ha = mul_add(C.Io, w, cross(C.mc, v));
            const V3 pa_ang = cross_add(w, ha, cross(v, hl));
            const V3 pa_lin = cross(w, hl);
            // lane 0 (dq_j): the joint's own rotation;  lane 1 (dqd_j): the joint rate
            tw0 = mulT(M, twp0); tv0 = mulT(M, cross_add(twp0, C.r, tvp0));
            tw1 = mulT(M, twp1); tv1 = mulT(M, cross_add(twp1, C.r, tvp1));
            if (own) { tw0 = tw0 + zc1(Ew); tv0 = tv0 + zc1(Ev); tw1.z += 1.f; }
            const float dqd1 = own ? 1.f : 0.f;
            const V3 dca0 = cross_z(tw0, qd_k), dcl0 = cross_z(tv0, qd_k);
            const V3 dca1 = cross_z(tw1, qd_k) + cross_z(w, dqd1), dcl1 = cross_z(tv1, qd_k) + cross_z(v, dqd1);
            auto dpa = [&](V3 tw, V3 tv, V3& dang, V3& dlin) {
                const V3 dhl = C.m * tv - cross(C.mc, tw);
                const V3 dha = mul_add(C.Io, tw, cross(C.mc, tv));
                dang = cross(tw, ha) + cross(w, dha) + cross(tv, hl) + cross(v, dhl);
                dlin = cross(tw, hl) + cross(w, dhl);
            };
            V3 da0, dl0, da1, dl1;
            dpa(tw0, tv0, da0, dl0);
            dpa(tw1, tv1, da1, dl1);
            float* lk = lk0 + i * FDD_LINK * S;
            lk[0] = cs; lk[S] = sn; lk[2 * S] = ca.x; lk[3 * S] = ca.y; lk[4 * S] = cl.x; lk[5 * S] = cl.y;
            stv(lk + 6 * S, S, pa_ang); stv(lk + 9 * S, S, pa_lin);
            lk[12 * S] = dca0.x; lk[13 * S] = dca0.y; lk[14 * S] = dcl0.x; lk[15 * S] = dcl0.y;
            lk[16 * S] = dca1.x; lk[17 * S] = dca1.y; lk[18 * S] = dcl1.x; lk[19 * S] = dcl1.y;
            stv(lk + 20 * S, S, da0); stv(lk + 23 * S, S, dl0); stv(lk + 26 * S, S, da1); stv(lk + 29 * S, S, dl1);
            const int sv = prog.save[i];
            if (sv >= 0) {
                float* sl = sl0 + sv * FDD_SLOT * S;
                stv(sl, S, w); stv(sl + 3 * S, S, v); stv(sl + 6 * S, S, tw0); stv(sl + 9 * S, S, tv0);
                stv(sl + 12 * S, S, tw1); stv(sl + 15 * S, S, tv1);
            }
        }
    }

    // ---- pass 2: leaves -> root, articulated inertias, biases and their tangents --------------------------------------
    // slot layout (x S): 0 A, 9 B, 18 C, 27 D, 36 pA_ang, 39 pA_lin, 42 dA, 51 dB, 60 dC, 69 dD, 78 dpA lane 0 (ang, lin),
    //   84 dpA lane 1, 90 pA lane f
    {
        M3 cA = zero3(), cB = zero3(), cC = zero3(), cD = zero3(), cdA = zero3(), cdB = zero3(), cdC = zero3(), cdD = zero3();
        V3 cpa = zero, cpl = zero, cda0 = zero, cdl0 = zero, cda1 = zero, cdl1 = zero, cfa = zero, cfl = zero;
        for (int i = N - 1; i >= 1; --i) {
            const LinkRow L = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
            float* lk = lk0 + i * FDD_LINK * S;
            M3 A = L.Io, B = skew(L.mc), C = transpose(B), D = zero3();
            D.a00 = D.a11 = D.a22 = L.m;
            M3 dA = zero3(), dB = zero3(), dC = zero3(), dD = zero3();
            V3 pa = ldv(lk + 6 * S, S), pl = ldv(lk + 9 * S, S);
            V3 da0 = ldv(lk + 20 * S, S), dl0 = ldv(lk + 23 * S, S), da1 = ldv(lk + 26 * S, S), dl1 = ldv(lk + 29 * S, S);
            V3 fa = zero, fl = zero;
            if (i + 1 < N && prog.psrc[i + 1] == 0) {
                A = A + cA; B = B + cB; C = C + cC; D = D + cD;
                dA = dA + cdA; dB = dB + cdB; dC = dC + cdC; dD = dD + cdD;
                pa = pa + cpa; pl = pl + cpl; da0 = da0 + cda0; dl0 = dl0 + cdl0; da1 = da1 + cda1; dl1 = dl1 + cdl1;
                fa = fa + cfa; fl = fl + cfl;
            }
            const int sv = prog.save[i];
            if (sv >= 0) {
                const float* sl = sl0 + sv * FDD_SLOT * S;
                A = A + ldm(sl, S); B = B + ldm(sl + 9 * S, S); C = C + ldm(sl + 18 * S, S); D = D + ldm(sl + 27 * S, S);
                pa = pa + ldv(sl + 36 * S, S); pl = pl + ldv(sl + 39 * S, S);
                dA = dA + ldm(sl + 42 * S, S); dB = dB + ldm(sl + 51 * S, S); dC = dC + ldm(sl + 60 * S, S); dD = dD + ldm(sl + 69 * S, S);
                da0 = da0 + ldv(sl + 78 * S, S); dl0 = dl0 + ldv(sl + 81 * S, S);
                da1 = da1 + ldv(sl + 84 * S, S); dl1 = dl1 + ldv(sl + 87 * S, S);
                fa = fa + ldv(sl + 90 * S, S); fl = fl + ldv(sl + 93 * S, S);
            }
            const int c = prog.dof[i];
            const bool own = (c == j);
            V3 Ua = zero, Ul = zero, dUa = zero, dUl = zero;
            float d = 0.f, u = 0.f, dd = 0.f, du0 = 0.f, du1 = 0.f, uf = 0.f;
            if (c >= 0) {
                Ua = col2(A); Ul = col2(C); d = Ua.z;                          // U = IA S, d = S . U
                dUa = col2(dA); dUl = col2(dC); dd = dUa.z;
                float fk = frow[c];
                if (damp) fk = fmaf(-L.d, qdrow[c], fk);
                u = fk - pa.z;
                du0 = -da0.z;
                du1 = -da1.z - ((damp && own) ? L.d : 0.f);
                uf = (own ? 1.f : 0.f) - fa.z;
            }
            const int P = prog.parent[i];
            if (P > 0) {
                const float cs = lk[0], sn = lk[S];
                if (c >= 0) {
                    const float inv = 1.f / (d + ABA_EPS);
                    const float dinv = -inv * inv * dd;
                    const V3 Uda = inv * Ua, Udl = inv * Ul;
                    const V3 dUda = dinv * Ua + inv * dUa, dUdl = dinv * Ul + inv * dUl;
                    // IA' = IA - U Ud^T;  dIA' = dIA - dU Ud^T - U dUd^T
                    sub_outer(dA, dUa, Uda); sub_outer(dA, Ua, dUda);
                    sub_outer(dB, dUa, Udl); sub_outer(dB, Ua, dUdl);
                    sub_outer(dC, dUl, Uda); sub_outer(dC, Ul, dUda);
                    sub_outer(dD, dUl, Udl); sub_outer(dD, Ul, dUdl);
                    sub_outer(A, Ua, Uda); sub_outer(B, Ua, Udl); sub_outer(C, Ul, Uda); sub_outer(D, Ul, Udl);
                    const V3 ca = v3(lk[2 * S], lk[3 * S], 0.f), cl = v3(lk[4 * S], lk[5 * S], 0.f);
                    const V3 dca0 = v3(lk[12 * S], lk[13 * S], 0.f), dcl0 = v3(lk[14 * S], lk[15 * S], 0.f);
                    const V3 dca1 = v3(lk[16 * S], lk[17 * S], 0.f), dcl1 = v3(lk[18 * S], lk[19 * S], 0.f);
                    const float ud = u * inv, dud0 = du0 * inv + u * dinv, dud1 = du1 * inv, udf = uf * inv;
                    // pa = pA + IA' c + U ud, and its tangents
                    da0 = da0 + mul2v(dA, ca, dB, cl) + mul2v(A, dca0, B, dcl0) + ud * dUa + dud0 * Ua;
                    dl0 = dl0 + mul2v(dC, ca, dD, cl) + mul2v(C, dca0, D, dcl0) + ud * dUl + dud0 * Ul;
                    da1 = da1 + mul2v(A, dca1, B, dcl1) + dud1 * Ua;
                    dl1 = dl1 + mul2v(C, dca1, D, dcl1) + dud1 * Ul;
                    fa = fa + udf * Ua; fl = fl + udf * Ul;
                    pa = pa + mul2v(A, ca, B, cl) + ud * Ua;
                    pl = pl + mul2v(C, ca, D, cl) + ud * Ul;
                }
                M3 M = L.F;
                if (c >= 0) rotate_z(M, cs, sn);
                if (own) {                                                     // the joint's own rotation moves X
                    dA = dA + kcomm(A); dB = dB + kcomm(B); dC = dC + kcomm(C); dD = dD + kcomm(D);
                    da0 = da0 + ezx(pa); dl0 = dl0 + ezx(pl);
                }
                M3 Ya, Yb, Yc, Yd, dYa, dYb, dYc, dYd;
                xform6(M, L.r, A, B, C, D, Ya, Yb, Yc, Yd);
                xform6(M, L.r, dA, dB, dC, dD, dYa, dYb, dYc, dYd);
                auto force = [&](V3 ang, V3 lin, V3& oa, V3& ol) { ol = mul(M, lin); oa = cross_add(L.r, ol, mul(M, ang)); };
                V3 qa, ql, qa0, ql0, qa1, ql1, qfa, qfl;
                force(pa, pl, qa, ql); force(da0, dl0, qa0, ql0); force(da1, dl1, qa1, ql1); force(fa, fl, qfa, qfl);
                if (P == i - 1) {
                    cA = Ya; cB = Yb; cC = Yc; cD = Yd; cdA = dYa; cdB = dYb; cdC = dYc; cdD = dYd;
                    cpa = qa; cpl = ql; cda0 = qa0; cdl0 = ql0; cda1 = qa1; cdl1 = ql1; cfa = qfa; cfl = qfl;
                } else {
                    float* sl = sl0 + (int)prog.save[P] * FDD_SLOT * S;
                    if (prog.accw[i] != 2) {
                        Ya = Ya + ldm(sl, S); Yb = Yb + ldm(sl + 9 * S, S); Yc = Yc + ldm(sl + 18 * S, S); Yd = Yd + ldm(sl + 27 * S, S);
                        qa = qa + ldv(sl + 36 * S, S); ql = ql + ldv(sl + 39 * S, S);
                        dYa = dYa + ldm(sl + 42 * S, S); dYb = dYb + ldm(sl + 51 * S, S);
                        dYc = dYc + ldm(sl + 60 * S, S); dYd = dYd + ldm(sl + 69 * S, S);
                        qa0 = qa0 + ldv(sl + 78 * S, S); ql0 = ql0 + ldv(sl + 81 * S, S);
                        qa1 = qa1 + ldv(sl + 84 * S, S); ql1 = ql1 + ldv(sl + 87 * S, S);
                        qfa = qfa + ldv(sl + 90 * S, S); qfl = qfl + ldv(sl + 93 * S, S);
                    }
                    stm(sl, S, Ya); stm(sl + 9 * S, S, Yb); stm(sl + 18 * S, S, Yc); stm(sl + 27 * S, S, Yd);
                    stv(sl + 36 * S, S, qa); stv(sl + 39 * S, S, ql);
                    stm(sl + 42 * S, S, dYa); stm(sl + 51 * S, S, dYb); stm(sl + 60 * S, S, dYc); stm(sl + 69 * S, S, dYd);
                    stv(sl + 78 * S, S, qa0); stv(sl + 81 * S, S, ql0); stv(sl + 84 * S, S, qa1); stv(sl + 87 * S, S, ql1);
                    stv(sl + 90 * S, S, qfa); stv(sl + 93 * S, S, qfl);
                }
            }
            stv(lk + 6 * S, S, Ua); stv(lk + 9 * S, S, Ul); stv(lk + 20 * S, S, dUa); stv(lk + 23 * S, S, dUl);
            lk[26 * S] = u; lk[27 * S] = d; lk[28 * S] = du0; lk[29 * S] = du1; lk[30 * S] = dd; lk[31 * S] = uf;
        }
    }

    // ---- pass 3: root -> leaves, accelerations and their tangents ----------------------------------------------------
    {
        V3 al = zero, a = zero, dal0 = zero, da0 = zero, dal1 = zero, da1 = zero, dalf = zero, daf = zero;
        for (int i = 1; i < N; ++i) {
            const float* row = s_tab + i * DRMB200_TABLE_STRIDE;
            M3 M; V3 r;
            load_Fr(row, M, r);
            const float* lk = lk0 + i * FDD_LINK * S;
            const int src = prog.psrc[i];
            V3 alp, ap, dalp0, dap0, dalp1, dap1, dalpf, dapf;
            if (src == 0) { alp = al; ap = a; dalp0 = dal0; dap0 = da0; dalp1 = dal1; dap1 = da1; dalpf = dalf; dapf = daf; }
            else if (src < 0) { alp = dalp0 = dap0 = dalp1 = dap1 = dalpf = dapf = zero; ap = v3(0.f, 0.f, g); }
            else {
                const float* sl = sl0 + (src - 1) * FDD_SLOT * S;
                alp = ldv(sl, S); ap = ldv(sl + 3 * S, S); dalp0 = ldv(sl + 6 * S, S); dap0 = ldv(sl + 9 * S, S);
                dalp1 = ldv(sl + 12 * S, S); dap1 = ldv(sl + 15 * S, S); dalpf = ldv(sl + 18 * S, S); dapf = ldv(sl + 21 * S, S);
            }
            const int c = prog.dof[i];
            if (c >= 0) rotate_z(M, lk[0], lk[S]);
            const V3 Eal = mulT(M, alp), Ea = mulT(M, cross_add(alp, r, ap));
            al = Eal; a = Ea;
            dal0 = mulT(M, dalp0); da0 = mulT(M, cross_add(dalp0, r, dap0));
            dal1 = mulT(M, dalp1); da1 = mulT(M, cross_add(dalp1, r, dap1));
            dalf = mulT(M, dalpf); daf = mulT(M, cross_add(dalpf, r, dapf));
            if (c >= 0) {
                if (c == j) { dal0 = dal0 + zc1(Eal); da0 = da0 + zc1(Ea); }
                al.x += lk[2 * S]; al.y += lk[3 * S]; a.x += lk[4 * S]; a.y += lk[5 * S];
                dal0.x += lk[12 * S]; dal0.y += lk[13 * S]; da0.x += lk[14 * S]; da0.y += lk[15 * S];
                dal1.x += lk[16 * S]; dal1.y += lk[17 * S]; da1.x += lk[18 * S]; da1.y += lk[19 * S];
                const V3 Ua = ldv(lk + 6 * S, S), Ul = ldv(lk + 9 * S, S), dUa = ldv(lk + 20 * S, S), dUl = ldv(lk + 23 * S, S);
                const float u = lk[26 * S], d = lk[27 * S], du0 = lk[28 * S], du1 = lk[29 * S], dd = lk[30 * S], uf = lk[31 * S];
                const float inv = 1.0f / d;
                const float qdd = inv * (u - (dot(Ua, al) + dot(Ul, a)));
                const float g0 = inv * (du0 - (dot(dUa, al) + dot(Ua, dal0) + dot(dUl, a) + dot(Ul, da0)) - qdd * dd);
                const float g1 = inv * (du1 - (dot(Ua, dal1) + dot(Ul, da1)));
                const float gf = inv * (uf - (dot(Ua, dalf) + dot(Ul, daf)));
                if (o_q) o_q[c * n] = g0;
                if (o_qd) o_qd[c * n] = g1;
                if (o_f) o_f[c * n] = gf;
                al.z += qdd; dal0.z += g0; dal1.z += g1; dalf.z += gf;
            }
            const int sv = prog.save[i];
            if (sv >= 0) {
                float* sl = sl0 + sv * FDD_SLOT * S;
                stv(sl, S, al); stv(sl + 3 * S, S, a); stv(sl + 6 * S, S, dal0); stv(sl + 9 * S, S, da0);
                stv(sl + 12 * S, S, dal1); stv(sl + 15 * S, S, da1); stv(sl + 18 * S, S, dalf); stv(sl + 21 * S, S, daf);
            }
        }
    }
}

}  // namespace drm
