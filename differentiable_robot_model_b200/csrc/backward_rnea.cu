// backward_rnea.cu -- analytic reverse-mode kernels for RNEA inverse dynamics (sm_90a).
//
// See backward.cu for the common design (recompute instead of save, deterministic table-gradient reduction,
// canonical joint frames) and oracle/adjoint_proto.py for the recursions in executable form.
//
// Two kernels:
//   rnea_backward_kernel            the full adjoint: gradients w.r.t. q, qd, qdd and every table column;
//   rnea_backward_inertial_kernel   a single root->leaves sweep for the case that only the inertial columns
//                                   (I_o, mc, m) and the damping are wanted (DRMB200_INERTIAL_GRADS_ONLY).
//
// Shared-memory diet of the full adjoint.  Shared memory is what limits its occupancy.  The leaves->root sweep
// needs the motion state (w, v, al, a) of every link and of its parent, but the forward recursion is invertible
// (E = M^T is orthogonal):
//     w_p  = M (w_i - (0,0,qd))                    v_p = M v_i - w_p x r
//     al_p = M (al_i - (0,0,qdd) - w_i x (0,0,qd))  a_p = M (a_i - v_i x (0,0,qd)) - al_p x r
// so the sweep carries the state DOWN the tree in registers and only the "tips" (links whose successor in
// document order is not their child: the end of every chain) keep their 12 floats in shared memory.  Per link
// that leaves 8 floats (accumulated wrench -> wrench adjoints, cos, sin) instead of 20: 3x the resident warps
// for a 7-DoF arm.  The re-derived states differ from the forward ones by rounding only (~1e-7 relative).
#include "backward_common.cuh"

namespace drm {

struct RneaBwdArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ qdd;
    const float* __restrict__ g_tau;
    float* __restrict__ q_grad;
    float* __restrict__ qd_grad;
    float* __restrict__ qdd_grad;
    float* __restrict__ partials;
    int64_t batch;
    uint32_t flags;
    int32_t vec_ok;
};

// per-link per-thread state, slot-major: f n -> mu lambda (6) | cos sin (2)
constexpr int LSTATE = 8;

struct RneaBwdSmem {
    int q, qd, qdd, g, qg, qdg, qddg, table, link, slots, tips, scratch, acc, total_floats;
    __host__ __device__ RneaBwdSmem(int tile, int n, int n_links, int n_slots, int n_tips) {
        int o = 0;
        q = o; o += tile * n;
        qd = o; o += tile * n;
        qdd = o; o += tile * n;
        g = o; o += tile * n;
        qg = o; o += tile * n;
        qdg = o; o += tile * n;
        qddg = o; o += tile * n;
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o; o += n_links * LSTATE * tile;
        slots = o; o += n_slots * 12 * tile;      // forward: branch-point motion states; backward: adjoint accumulators
        tips = o; o += n_tips * 12 * tile;        // motion state of every chain end
        scratch = o; o += block_accumulate_floats(25, tile);
        acc = o; o += n_links * DRMB200_TABLE_STRIDE;
        total_floats = o;
    }
};

template <bool NEED_TABLE, int T>
__global__ void __launch_bounds__(T)
rnea_backward_kernel(const __grid_constant__ TreeProgram prog, const RneaBwdArgs args) {
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs, N = prog.n_links;
    const RneaBwdSmem L(T, n, N, prog.n_slots, prog.n_tips);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_qdd = smem + L.qdd;
    float* s_g = smem + L.g;
    float* s_qg = smem + L.qg;
    float* s_qdg = smem + L.qdg;
    float* s_qddg = smem + L.qddg;
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_slot = smem + L.slots;
    float* s_tips = smem + L.tips;
    float* s_scr = smem + L.scratch;
    float* s_acc = smem + L.acc;
    const int tid = threadIdx.x;
    const bool vec_ok = args.vec_ok;
    const float grav = (args.flags & DRMB200_GRAVITY) ? GRAVITY_B : 0.f;
    const bool damp = (args.flags & DRMB200_DAMPING) != 0;

    for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) {
        const int l = i / DRMB200_TABLE_STRIDE, e = i - l * DRMB200_TABLE_STRIDE;
        const int p = prog.parent[l];
        int src;
        const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
        s_tab[i] = sg * __ldg(args.table + l * DRMB200_TABLE_STRIDE + src);
        if (NEED_TABLE) s_acc[i] = 0.f;
    }

    const int64_t n_tiles = (args.batch + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t start = tile * T;
        const int valid = (int)min((int64_t)T, args.batch - start);
        __syncthreads();
        coop_copy(s_q, args.q + start * n, valid * n, vec_ok);
        coop_copy(s_qd, args.qd + start * n, valid * n, vec_ok);
        coop_copy(s_qdd, args.qdd + start * n, valid * n, vec_ok);
        coop_copy(s_g, args.g_tau + start * n, valid * n, vec_ok);
        __syncthreads();

        const bool active = tid < valid;
        const float* qrow = s_q + tid * n;
        const float* qdrow = s_qd + tid * n;
        const float* qddrow = s_qdd + tid * n;
        const float* grow = s_g + tid * n;
        float* qg = s_qg + tid * n;
        float* qdg = s_qdg + tid * n;
        float* qddg = s_qddg + tid * n;
        float* lk = s_link + tid;
        const V3 zero = v3(0.f, 0.f, 0.f);
        const V3 a_root = v3(0.f, 0.f, grav);

        // ---- forward recompute, pass A: motion state (registers / branch slots) + body wrench ------
        {
            V3 w = zero, v = zero, al = zero, a = zero;
            for (int i = 1; i < N; ++i) {
                const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
                const int src = prog.psrc[i];
                V3 wp, vp, alp, ap;
                if (src == 0) { wp = w; vp = v; alp = al; ap = a; }
                else if (src < 0) { wp = vp = alp = zero; ap = a_root; }
                else {
                    const float* sl = s_slot + (src - 1) * 12 * T + tid;
                    wp = ldv(sl, T); vp = ldv(sl + 3 * T, T); alp = ldv(sl + 6 * T, T); ap = ldv(sl + 9 * T, T);
                }
                M3 M = C.F;
                const int c = prog.dof[i];
                float cs = 1.f, sn = 0.f, qd_k = 0.f, qdd_k = 0.f;
                if (c >= 0) {
                    qd_k = qdrow[c]; qdd_k = qddrow[c];
                    sincos_pi2(qrow[c], sn, cs);
                    rotate_z(M, cs, sn);
                }
                w = mulT(M, wp); w.z += qd_k;
                v = mulT(M, cross_add(wp, C.r, vp));
                al = mulT(M, alp) + cross_z(w, qd_k); al.z += qdd_k;
                a = mulT(M, cross_add(alp, C.r, ap)) + cross_z(v, qd_k);
                const V3 hl_a = C.m * a - cross(C.mc, al);
                const V3 ha_a = mul_add(C.Io, al, cross(C.mc, a));
                const V3 hl_v = C.m * v - cross(C.mc, w);
                const V3 ha_v = mul_add(C.Io, w, cross(C.mc, v));
                const V3 f = cross_add(w, hl_v, hl_a);
                const V3 nn = cross_add(w, ha_v, cross_add(v, hl_v, ha_a));
                float* s = lk + i * LSTATE * T;
                stv(s, T, f); stv(s + 3 * T, T, nn);
                s[6 * T] = cs; s[7 * T] = sn;
                const int sv = prog.save[i];
                if (sv >= 0) {
                    float* sl = s_slot + sv * 12 * T + tid;
                    stv(sl, T, w); stv(sl + 3 * T, T, v); stv(sl + 6 * T, T, al); stv(sl + 9 * T, T, a);
                }
                const int tp = prog.tip[i];
                if (tp >= 0) {
                    float* st = s_tips + tp * 12 * T + tid;
                    stv(st, T, w); stv(st + 3 * T, T, v); stv(st + 6 * T, T, al); stv(st + 9 * T, T, a);
                }
            }
        }
        // ---- forward recompute, pass B: accumulate wrenches leaves -> root -----------------------
        for (int i = N - 1; i >= 1; --i) {
            const int P = prog.parent[i];
            if (P <= 0) continue;
            const float* s = lk + i * LSTATE * T;
            M3 F; V3 r;
            load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, F, r);
            const float cs = s[6 * T], sn = s[7 * T];
            const V3 fp = mul(F, rotz(ldv(s, T), cs, sn));
            const V3 np = cross_add(r, fp, mul(F, rotz(ldv(s + 3 * T, T), cs, sn)));
            float* sp = lk + P * LSTATE * T;
            stv(sp, T, ldv(sp, T) + fp);
            stv(sp + 3 * T, T, ldv(sp + 3 * T, T) + np);
        }

        // ---- adjoint pass 1, root -> leaves: lambda = n-bar, mu = f-bar ----------------------------
        for (int i = 1; i < N; ++i) {
            float* s = lk + i * LSTATE * T;
            const float* row = s_tab + i * DRMB200_TABLE_STRIDE;
            M3 M; V3 r;
            load_Fr(row, M, r);
            const int P = prog.parent[i];
            V3 lamP = zero, muP = zero;
            if (P > 0) { const float* sp = lk + P * LSTATE * T; muP = ldv(sp, T); lamP = ldv(sp + 3 * T, T); }
            const int c = prog.dof[i];
            const float cs = s[6 * T], sn = s[7 * T];
            float gk = 0.f;
            if (c >= 0) { rotate_z(M, cs, sn); gk = grow[c]; }
            const V3 f = ldv(s, T), nn = ldv(s + 3 * T, T);                 // accumulated wrenches
            const V3 u = cross_add(lamP, r, muP);
            V3 lam = mulT(M, lamP); lam.z += gk;                            // tau_k = n_i . e_z
            const V3 mu = mulT(M, u);
            stv(s, T, mu);                                                   // f slot -> mu
            stv(s + 3 * T, T, lam);                                          // n slot -> lambda
            M3 Mbar = zero3();
            add_outer(Mbar, lamP, nn);
            add_outer(Mbar, u, f);
            const V3 rbar = cross(mul(M, f), lamP);
            float dbar = 0.f;
            if (c >= 0) {
                qg[c] = theta_grad_z(Mbar, M);
                float qdv = 0.f;
                if (damp) { qdv = row[25] * gk; dbar = gk * qdrow[c]; }
                qdg[c] = qdv;
            }
            if (NEED_TABLE) {
                M3 Fbar = Mbar;
                if (c >= 0) rotate_z(Fbar, cs, -sn);
                float vals[13];
                m3_to_array(Fbar, vals);
                vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z; vals[12] = dbar;
                block_accumulate<13, T>(s_scr, s_acc + i * DRMB200_TABLE_STRIDE, vals, active,
                                        [](int j) { return j < 12 ? j : 25; });
            }
        }

        // ---- adjoint pass 2, leaves -> root: motion adjoints -------------------------------------
        V3 c_wb = zero, c_vb = zero, c_alb = zero, c_ab = zero;     // adjoints carried into link i from child i+1
        V3 s_w = zero, s_v = zero, s_al = zero, s_a = zero;         // motion state of link i re-derived from child i+1
        for (int i = N - 1; i >= 1; --i) {
            const float* s = lk + i * LSTATE * T;
            const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
            const int P = prog.parent[i];
            const int c = prog.dof[i];
            const float cs = s[6 * T], sn = s[7 * T];
            M3 M = C.F;
            float qd_k = 0.f, qdd_k = 0.f;
            if (c >= 0) { rotate_z(M, cs, sn); qd_k = qdrow[c]; qdd_k = qddrow[c]; }
            // this link's motion state: stored for chain ends, otherwise handed down by child i+1
            V3 w, v, al, a;
            const int tp = prog.tip[i];
            if (tp >= 0) {
                const float* st = s_tips + tp * 12 * T + tid;
                w = ldv(st, T); v = ldv(st + 3 * T, T); al = ldv(st + 6 * T, T); a = ldv(st + 9 * T, T);
            } else { w = s_w; v = s_v; al = s_al; a = s_a; }
            // the parent's state through the inverted recursion (root: constants)
            V3 wp = zero, vp = zero, alp = zero, ap = a_root;
            if (P > 0) {
                V3 t = w; t.z -= qd_k;
                wp = mul(M, t);
                vp = mul(M, v) - cross(wp, C.r);
                t = al - cross_z(w, qd_k); t.z -= qdd_k;
                alp = mul(M, t);
                ap = mul(M, a - cross_z(v, qd_k)) - cross(alp, C.r);
            }
            s_w = wp; s_v = vp; s_al = alp; s_a = ap;               // used by iteration i-1 iff parent(i) == i-1
            const V3 mu = ldv(s, T), lam = ldv(s + 3 * T, T);
            // incoming adjoints: child i+1 through registers, far children through the branch slot
            V3 wb = zero, vb = zero, alb = zero, ab = zero;
            if (i + 1 < N && prog.psrc[i + 1] == 0) { wb = c_wb; vb = c_vb; alb = c_alb; ab = c_ab; }
            const int sv = prog.save[i];
            if (sv >= 0) {
                const float* sl = s_slot + sv * 12 * T + tid;
                wb = wb + ldv(sl, T); vb = vb + ldv(sl + 3 * T, T); alb = alb + ldv(sl + 6 * T, T); ab = ab + ldv(sl + 9 * T, T);
            }
            // body part (momentum H, wrench adjoints lam / mu)
            const V3 Hl = C.m * v - cross(C.mc, w);
            const V3 Ha = mul_add(C.Io, w, cross(C.mc, v));
            const V3 Hlb = cross_add(mu, w, cross(lam, v));
            const V3 Hab = cross(lam, w);
            alb = alb + cross_add(C.mc, mu, mulT(C.Io, lam));
            ab = ab + cross_add(lam, C.mc, C.m * mu);
            wb = wb + cross_add(Hl, mu, cross_add(Ha, lam, cross_add(C.mc, Hlb, mulT(C.Io, Hab))));
            vb = vb + cross_add(Hl, lam, cross_add(Hab, C.mc, C.m * Hlb));
            float vals[25];
            if (NEED_TABLE) {
                M3 Iob = zero3();
                add_outer(Iob, lam, al);
                add_outer(Iob, Hab, w);
                m3_to_array(Iob, vals + 12);
                const V3 mcb = cross_add(mu, al, cross_add(a, lam, cross_add(Hlb, w, cross(v, Hab))));
                vals[21] = mcb.x; vals[22] = mcb.y; vals[23] = mcb.z;
                vals[24] = dot(mu, a) + dot(Hlb, v);
            }
            // kinematic part, in the order a, alpha, v, omega; wJ = (0, 0, qd_k)
            M3 Mbar = zero3();
            float wJb = ab.x * v.y - ab.y * v.x;            // (ab x v).z -- only the z component of wJ-bar matters
            vb = vb + z_cross(qd_k, ab);
            const V3 ua = mul(M, ab);
            const V3 abP = ua;
            V3 albP = cross(C.r, ua);
            V3 rbar = cross(ua, alp);
            add_outer(Mbar, cross_add(alp, C.r, ap), ab);

            wb = wb + z_cross(qd_k, alb);
            wJb += alb.x * w.y - alb.y * w.x;               // (alb x w).z
            albP = albP + mul(M, alb);
            add_outer(Mbar, alp, alb);

            const V3 uv = mul(M, vb);
            const V3 vbP = uv;
            V3 wbP = cross(C.r, uv);
            rbar = rbar + cross(uv, wp);
            add_outer(Mbar, cross_add(wp, C.r, vp), vb);

            wbP = wbP + mul(M, wb);
            add_outer(Mbar, wp, wb);
            wJb += wb.z;

            if (c >= 0) {
                qddg[c] = alb.z;
                qdg[c] += wJb;
                qg[c] += theta_grad_z(Mbar, M);
            }
            // route the parent contributions
            if (P == i - 1) { c_wb = wbP; c_vb = vbP; c_alb = albP; c_ab = abP; }
            else if (P > 0) {
                float* sl = s_slot + (int)prog.save[P] * 12 * T + tid;
                if (prog.accw[i] == 2) {
                    stv(sl, T, wbP); stv(sl + 3 * T, T, vbP); stv(sl + 6 * T, T, albP); stv(sl + 9 * T, T, abP);
                } else {
                    stv(sl, T, ldv(sl, T) + wbP); stv(sl + 3 * T, T, ldv(sl + 3 * T, T) + vbP);
                    stv(sl + 6 * T, T, ldv(sl + 6 * T, T) + albP); stv(sl + 9 * T, T, ldv(sl + 9 * T, T) + abP);
                }
            }
            if (NEED_TABLE) {
                M3 Fbar = Mbar;
                if (c >= 0) rotate_z(Fbar, cs, -sn);
                m3_to_array(Fbar, vals);
                vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z;
                block_accumulate<25, T>(s_scr, s_acc + i * DRMB200_TABLE_STRIDE, vals, active, [](int j) { return j; });
            }
        }
        __syncthreads();
        if (args.q_grad != nullptr) coop_copy(args.q_grad + start * n, s_qg, valid * n, vec_ok);
        if (args.qd_grad != nullptr) coop_copy(args.qd_grad + start * n, s_qdg, valid * n, vec_ok);
        if (args.qdd_grad != nullptr) coop_copy(args.qdd_grad + start * n, s_qddg, valid * n, vec_ok);
    }
    if (NEED_TABLE) {
        __syncthreads();
        float* out = args.partials + (size_t)blockIdx.x * N * DRMB200_TABLE_STRIDE;
        for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) {        // canonical -> natural (bijection per row)
            const int l = i / DRMB200_TABLE_STRIDE, e = i - l * DRMB200_TABLE_STRIDE;
            const int p = prog.parent[l];
            int src;
            const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
            out[l * DRMB200_TABLE_STRIDE + src] = sg * s_acc[i];
        }
    }
}

// =============================================================================================
// RNEA backward, inertial parameters only (DRMB200_INERTIAL_GRADS_ONLY)
// =============================================================================================
// tau is LINEAR in (m, mc, I_o) and the damping, and the wrench adjoints (lambda, mu) obey a root->leaves
// recursion just like the motion state, so when only those table columns are wanted (the classic "learn the link
// inertias" setting, BASELINE config 5: nothing kinematic is learnable and no input gradients are requested) the
// whole backward collapses into ONE root->leaves sweep with no per-link storage:
//   lam_i = E lam_p + (0,0,g_k)        mu_i = E (mu_p + lam_p x r)
//   Io-bar = lam al^T + (lam x w) w^T   mc-bar = mu x al + a x lam + Hl-bar x w + v x Ha-bar
//   m-bar  = mu . a + Hl-bar . v        d-bar  = g_k qd_k           (Hl-bar = mu x w + lam x v, Ha-bar = lam x w)
// About 230 instructions per link instead of ~1350 for the full adjoint, and shared memory only for the I/O tiles.
struct RneaInertialSmem {
    int q, qd, qdd, g, table, slots, scratch, acc, total_floats;
    __host__ __device__ RneaInertialSmem(int tile, int n, int n_links, int n_slots) {
        int o = 0;
        q = o; o += tile * n;
        qd = o; o += tile * n;
        qdd = o; o += tile * n;
        g = o; o += tile * n;
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        slots = o; o += n_slots * 18 * tile;
        scratch = o; o += block_accumulate_floats(14, tile);
        acc = o; o += n_links * DRMB200_TABLE_STRIDE;
        total_floats = o;
    }
};

template <int T>
__global__ void __launch_bounds__(T)
rnea_backward_inertial_kernel(const __grid_constant__ TreeProgram prog, const RneaBwdArgs args) {
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs, N = prog.n_links;
    const RneaInertialSmem L(T, n, N, prog.n_slots);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_qdd = smem + L.qdd;
    float* s_g = smem + L.g;
    float* s_tab = smem + L.table;
    float* s_slot = smem + L.slots;
    float* s_scr = smem + L.scratch;
    float* s_acc = smem + L.acc;
    const int tid = threadIdx.x;
    const bool vec_ok = args.vec_ok;
    const float grav = (args.flags & DRMB200_GRAVITY) ? GRAVITY_B : 0.f;
    const bool damp = (args.flags & DRMB200_DAMPING) != 0;

    for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) {
        const int l = i / DRMB200_TABLE_STRIDE, e = i - l * DRMB200_TABLE_STRIDE;
        const int p = prog.parent[l];
        int src;
        const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
        s_tab[i] = sg * __ldg(args.table + l * DRMB200_TABLE_STRIDE + src);
        s_acc[i] = 0.f;
    }
    const int64_t n_tiles = (args.batch + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t start = tile * T;
        const int valid = (int)min((int64_t)T, args.batch - start);
        __syncthreads();
        coop_copy(s_q, args.q + start * n, valid * n, vec_ok);
        coop_copy(s_qd, args.qd + start * n, valid * n, vec_ok);
        coop_copy(s_qdd, args.qdd + start * n, valid * n, vec_ok);
        coop_copy(s_g, args.g_tau + start * n, valid * n, vec_ok);
        __syncthreads();
        const bool active = tid < valid;
        const float* qrow = s_q + tid * n;
        const float* qdrow = s_qd + tid * n;
        const float* qddrow = s_qdd + tid * n;
        const float* grow = s_g + tid * n;
        const V3 zero = v3(0.f, 0.f, 0.f);
        V3 w = zero, v = zero, al = zero, a = zero, lam = zero, mu = zero;      // state of the previous link
        for (int i = 1; i < N; ++i) {
            M3 M; V3 r;
            load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
            const int src = prog.psrc[i];
            V3 wp, vp, alp, ap, lamP, muP;
            if (src == 0) { wp = w; vp = v; alp = al; ap = a; lamP = lam; muP = mu; }
            else if (src < 0) { wp = vp = alp = lamP = muP = zero; ap = v3(0.f, 0.f, grav); }
            else {
                const float* sl = s_slot + (src - 1) * 18 * T + tid;
                wp = ldv(sl, T); vp = ldv(sl + 3 * T, T); alp = ldv(sl + 6 * T, T); ap = ldv(sl + 9 * T, T);
                lamP = ldv(sl + 12 * T, T); muP = ldv(sl + 15 * T, T);
            }
            const int c = prog.dof[i];
            float qd_k = 0.f, qdd_k = 0.f, gk = 0.f;
            if (c >= 0) {
                float sn, cs;
                sincos_pi2(qrow[c], sn, cs);
                rotate_z(M, cs, sn);
                qd_k = qdrow[c]; qdd_k = qddrow[c]; gk = grow[c];
            }
            w = mulT(M, wp); w.z += qd_k;
            v = mulT(M, cross_add(wp, r, vp));
            al = mulT(M, alp) + cross_z(w, qd_k); al.z += qdd_k;
            a = mulT(M, cross_add(alp, r, ap)) + cross_z(v, qd_k);
            lam = mulT(M, lamP); lam.z += gk;
            mu = mulT(M, cross_add(lamP, r, muP));
            const V3 Hlb = cross_add(mu, w, cross(lam, v));
            const V3 Hab = cross(lam, w);
            float vals[14];
            M3 Iob = zero3();
            add_outer(Iob, lam, al);
            add_outer(Iob, Hab, w);
            m3_to_array(Iob, vals);
            const V3 mcb = cross_add(mu, al, cross_add(a, lam, cross_add(Hlb, w, cross(v, Hab))));
            vals[9] = mcb.x; vals[10] = mcb.y; vals[11] = mcb.z;
            vals[12] = dot(mu, a) + dot(Hlb, v);
            vals[13] = (damp && c >= 0) ? gk * qd_k : 0.f;
            block_accumulate<14, T>(s_scr, s_acc + i * DRMB200_TABLE_STRIDE, vals, active,
                                    [](int j) { return j < 13 ? 12 + j : 25; });
            const int sv = prog.save[i];
            if (sv >= 0) {
                float* sl = s_slot + sv * 18 * T + tid;
                stv(sl, T, w); stv(sl + 3 * T, T, v); stv(sl + 6 * T, T, al); stv(sl + 9 * T, T, a);
                stv(sl + 12 * T, T, lam); stv(sl + 15 * T, T, mu);
            }
        }
    }
    __syncthreads();
    float* out = args.partials + (size_t)blockIdx.x * N * DRMB200_TABLE_STRIDE;
    for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) {            // canonical -> natural (bijection per row)
        const int l = i / DRMB200_TABLE_STRIDE, e = i - l * DRMB200_TABLE_STRIDE;
        const int p = prog.parent[l];
        int src;
        const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
        out[l * DRMB200_TABLE_STRIDE + src] = sg * s_acc[i];
    }
}

// =============================================================================================
// RNEA backward on a serial chain: two sweeps, f32x2 pair, TMA-staged tiles
// =============================================================================================
// For robots whose links form one chain (parent of link i is link i - 1: Kuka iiwa, Franka Panda, ...) the four passes of
// rnea_backward_kernel collapse into TWO sweeps (oracle/adjoint_proto.py: inverse_dynamics_backward_chain states them
// executably and is checked against autograd of the fp64 oracle):
//   sweep 1, root -> leaves: the motion state (w, v, al, a) and the wrench adjoints lam = n-bar, mu = f-bar, which obey a
//     root -> leaves recursion of the same form -- all of it only to arrive at the LAST link's values; per link just
//     (cos, sin) go to shared memory (2 floats instead of 8 + the chain-end state);
//   sweep 2, leaves -> root: link i - 1's motion state AND wrench adjoints re-derived from link i's (both recursions are
//     invertible, E is orthogonal), the body wrench RECOMPUTED from that state and accumulated on the way down (f, n never
//     touch memory), the motion adjoints carried in registers, and every gradient: one 26-value table-gradient reduction
//     per link instead of 13 + 25.
// M = F Rz(theta) is never formed: x -> Rz^T (F^T x), x -> F (Rz x).  For y = M^T x with adjoint y-bar the joint-angle
// gradient is (y-bar x y).z and the F gradient x (Rz y-bar)^T, so no 3x3 M-bar is accumulated for theta either.
// Velocity- and acceleration-level vectors (and their adjoints) go through the same maps as f32x2 PAIRS.
// The q / qd / qdd / g_tau row tiles arrive by TMA bulk copies on an mbarrier and the three input-gradient tiles leave by
// bulk stores FROM THE SAME shared memory: each thread has read q_k, qd_k, qdd_k of its row before it writes the gradient
// there, so the tiles alias (4 instead of 7 row tiles).  Rows past the end of the batch are zero-filled: with g = 0 every
// adjoint and every table-gradient term is exactly zero, so the reduction needs no per-value select.
struct RneaChainSmem {
    int q, qd, qdd, g, table, link, scratch, acc, total_floats;
    __host__ __device__ RneaChainSmem(int tile, int n, int n_links) {
        int o = 0;
        q = o; o += tile * n;
        qd = o; o += tile * n;
        qdd = o; o += tile * n;
        g = o; o += tile * n;
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o; o += (n_links - 1) * 2 * tile;           // cos sin of links 1 .. N-1
        scratch = o; o += (tile / 32) * 32 + 26 * (tile + 4);
        acc = o; o += n_links * DRMB200_TABLE_STRIDE;
        total_floats = o;
    }
};

// block_accumulate (backward_common.cuh) with the transposed sums read as float4: leading dimension T + 4 keeps the rows
// 16-byte aligned and both the per-thread stores and the quarter-warp 128-bit loads conflict-free.  Every thread
// contributes (rows past the end of the batch hold exact zeros).
template <int NV, int T>
__device__ __forceinline__ void chain_accumulate(float* scratch, float* acc_row, const float (&vals)[NV]) {
    static_assert(NV <= 32 && T % 32 == 0, "one lane per value");
    constexpr int LD = T + 4, NW = T / 32;
    float* partial = scratch;                 // [NW][32]
    float* values = scratch + NW * 32;        // [NV][LD]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
#pragma unroll
    for (int j = 0; j < NV; ++j) values[j * LD + tid] = vals[j];
    __syncthreads();
    if (lane < NV) {
        const float4* row = reinterpret_cast<const float4*>(values + lane * LD + warp * 32);
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) { const float4 x = row[c]; s0 += x.x; s1 += x.y; s2 += x.z; s3 += x.w; }
        const float t = (s0 + s1) + (s2 + s3);
        if (NW == 1) acc_row[lane] += t;
        else partial[warp * 32 + lane] = t;
    }
    __syncthreads();
    if (NW > 1 && warp == 0 && lane < NV) {
        float t = partial[lane];
#pragma unroll
        for (int w = 1; w < NW; ++w) t += partial[w * 32 + lane];
        acc_row[lane] += t;
    }
}

template <bool NEED_TABLE, int T>
__global__ void __launch_bounds__(T, (T == 64) ? 7 : 8)
rnea_backward_chain_kernel(const __grid_constant__ TreeProgram prog, const RneaBwdArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;
    const int n = prog.n_dofs, N = prog.n_links;
    const RneaChainSmem L(T, n, N);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_qdd = smem + L.qdd;
    float* s_g = smem + L.g;
    float* s_tab = smem + L.table;
    float* s_scr = smem + L.scratch;
    float* s_acc = smem + L.acc;
    const int tid = threadIdx.x;
    const bool vec_ok = args.vec_ok;
    const float grav = (args.flags & DRMB200_GRAVITY) ? GRAVITY_B : 0.f;
    const bool damp = (args.flags & DRMB200_DAMPING) != 0;

    if (tid == 0) { mbar_init(&mbar, 1); fence_mbar_init(); }
    // the reduction kernel that follows (launch_reduce: programmatic dependent launch) may be set up while this grid runs;
    // it waits for this grid to finish before it reads the partials
    if (NEED_TABLE) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    bool table_staged = false;

    const uint32_t a_q = smem_addr_opaque(s_q + tid * n), a_qd = smem_addr_opaque(s_qd + tid * n);
    const uint32_t a_qdd = smem_addr_opaque(s_qdd + tid * n), a_g = smem_addr_opaque(s_g + tid * n);
    const uint32_t a_tab = smem_addr_opaque(s_tab);
    const uint32_t a_link = smem_addr_opaque(smem + L.link + tid);
    constexpr uint32_t E = 4u * T;                      // byte stride between the elements of a slot-major vector
    constexpr uint32_t LB = 2u * E;                     // bytes per link of the per-thread state (cos, sin)
    auto ldv_s = [](uint32_t a) { return v3(lds_f32(a), lds_f32(a + E), lds_f32(a + 2 * E)); };
    auto stv_s = [](uint32_t a, V3 x) { sts_f32(a, x.x); sts_f32(a + E, x.y); sts_f32(a + 2 * E, x.z); };
    auto neg = [](V3 x) { return v3(-x.x, -x.y, -x.z); };
    auto fma3 = [](float s, V3 x, V3 y) { return v3(fmaf(s, x.x, y.x), fmaf(s, x.y, y.y), fmaf(s, x.z, y.z)); };       // s x + y
    auto mulT_add = [](const M3& m, V3 x, V3 y) {                                                                         // M^T x + y
        return v3(fmaf(m.a00, x.x, fmaf(m.a10, x.y, fmaf(m.a20, x.z, y.x))), fmaf(m.a01, x.x, fmaf(m.a11, x.y, fmaf(m.a21, x.z, y.y))),
                  fmaf(m.a02, x.x, fmaf(m.a12, x.y, fmaf(m.a22, x.z, y.z))));
    };
    const V3 zero = v3(0.f, 0.f, 0.f);
    const V3 a_root = v3(0.f, 0.f, grav);

    uint32_t phase = 0;
    const int64_t n_tiles = (args.batch + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t start = tile * T;
        const int valid = (int)min((int64_t)T, args.batch - start);
        const bool bulk = vec_ok && ((valid * n) & 3) == 0;
        fence_proxy_async();                            // this thread's generic accesses to the tiles before the bulk copies below
        __syncthreads();
        if (bulk) {
            if (tid == 0) {
                const uint32_t bytes = (uint32_t)(valid * n) * 4u;
                mbar_arrive_expect_tx(&mbar, 4u * bytes);
                bulk_g2s(s_q, args.q + start * n, bytes, &mbar);
                bulk_g2s(s_qd, args.qd + start * n, bytes, &mbar);
                bulk_g2s(s_qdd, args.qdd + start * n, bytes, &mbar);
                bulk_g2s(s_g, args.g_tau + start * n, bytes, &mbar);
            }
        } else {
            coop_copy(s_q, args.q + start * n, valid * n, vec_ok);
            coop_copy(s_qd, args.qd + start * n, valid * n, vec_ok);
            coop_copy(s_qdd, args.qdd + start * n, valid * n, vec_ok);
            coop_copy(s_g, args.g_tau + start * n, valid * n, vec_ok);
        }
        if (valid < T)                                  // rows past the end of the batch: all-zero inputs, all-zero gradients
            for (int i = valid * n + tid; i < T * n; i += T) { s_q[i] = 0.f; s_qd[i] = 0.f; s_qdd[i] = 0.f; s_g[i] = 0.f; }
        if (!table_staged) {                            // once per CTA, while the first tile's bulk copies are in flight
            stage_canonical_table(s_tab, args.table, prog, T);
            if (NEED_TABLE) for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) s_acc[i] = 0.f;
            table_staged = true;
        }
        __syncthreads();
        if (bulk) { mbar_wait(&mbar, phase); phase ^= 1u; }

        // ---- sweep 1, root -> leaves ---------------------------------------------------------------
        V3 w, v, al, a, lam = zero, mu = zero;
        {
            V3P W = pk3(zero, zero), V = pk3(zero, a_root);         // (w | al), (v | a) of the link before
            for (int i = 1; i < N; ++i) {
                M3 F; V3 r;
                load_Fr_s(a_tab + i * (DRMB200_TABLE_STRIDE * 4), F, r);
                const int c = prog.dof[i];
                float cs = 1.f, sn = 0.f, qd_k = 0.f, qdd_k = 0.f, gk = 0.f;
                if (c >= 0) {
                    qd_k = lds_f32(a_qd + 4u * c); qdd_k = lds_f32(a_qdd + 4u * c); gk = lds_f32(a_g + 4u * c);
                    sincos_pi2(lds_f32(a_q + 4u * c), sn, cs);
                }
                const V3P Wn = rotzT_p(mulT_p(F, W), cs, sn);
                const V3P Vn = rotzT_p(mulT_p(F, cross_add_p(W, r, V)), cs, sn);
                const V3 u = cross_add(lam, r, mu);
                const V3P Y = rotzT_p(mulT_p(F, pk3(lam, u)), cs, sn);
                upk3(Y, lam, mu);
                lam.z += gk;                                        // tau_k = n_i . e_z
                upk3(Wn, w, al); upk3(Vn, v, a);
                w.z += qd_k;
                al.x = fmaf(w.y, qd_k, al.x); al.y = fmaf(-w.x, qd_k, al.y); al.z += qdd_k;
                a.x = fmaf(v.y, qd_k, a.x); a.y = fmaf(-v.x, qd_k, a.y);
                W = pk3(w, al); V = pk3(v, a);
                const uint32_t lk = a_link + (uint32_t)(i - 1) * LB;
                sts_f32(lk, cs); sts_f32(lk + E, sn);
            }
        }

        // ---- sweep 2, leaves -> root ---------------------------------------------------------------
        V3 c_wb = zero, c_vb = zero, c_alb = zero, c_ab = zero;     // motion adjoints handed down by link i + 1
        V3 carry_f = zero, carry_n = zero;                          // wrench handed down by link i + 1
        for (int i = N - 1; i >= 1; --i) {
            const uint32_t row = a_tab + i * (DRMB200_TABLE_STRIDE * 4);
            LinkRow C;
            load_Fr_s(row, C.F, C.r);
            {
                const float4 d = lds_f32x4(row + 48), e = lds_f32x4(row + 64), f4 = lds_f32x4(row + 80), gg = lds_f32x4(row + 96);
                C.Io.a00 = d.x; C.Io.a01 = d.y; C.Io.a02 = d.z; C.Io.a10 = d.w; C.Io.a11 = e.x; C.Io.a12 = e.y;
                C.Io.a20 = e.z; C.Io.a21 = e.w; C.Io.a22 = f4.x;
                C.mc = v3(f4.y, f4.z, f4.w);
                C.m = gg.x; C.d = gg.y;
            }
            const uint32_t lk = a_link + (uint32_t)(i - 1) * LB;
            const float cs = lds_f32(lk), sn = lds_f32(lk + E);
            const int c = prog.dof[i];
            float qd_k = 0.f, qdd_k = 0.f, gk = 0.f;
            if (c >= 0) { qd_k = lds_f32(a_qd + 4u * c); qdd_k = lds_f32(a_qdd + 4u * c); gk = lds_f32(a_g + 4u * c); }

            // the joint's own contribution taken off again: y = M^T x for x = w_p, al_p, ...
            V3 tw = w; tw.z -= qd_k;
            const V3 tal = v3(fmaf(-w.y, qd_k, al.x), fmaf(w.x, qd_k, al.y), al.z - qdd_k);
            const V3 apre = v3(fmaf(-v.y, qd_k, a.x), fmaf(v.x, qd_k, a.y), a.z);
            // the parent's state and wrench adjoints through the inverted recursions (the root's are constants);
            // MV = (w_p x r + v_p | al_p x r + a_p),  u = lam_p x r + mu_p
            V3P Wp, MV, Vp;
            V3 lamP = zero, u = zero, muP = zero;
            if (i > 1) {
                Wp = mul_pv(C.F, rotz_p(pk3(tw, tal), cs, sn));
                MV = mul_pv(C.F, rotz_p(pk3(v, apre), cs, sn));
                Vp = cross_add_p(Wp, neg(C.r), MV);
                V3 tl = lam; tl.z -= gk;
                upk3(mul_pv(C.F, rotz_p(pk3(tl, mu), cs, sn)), lamP, u);
                muP = cross_add(C.r, lamP, u);
            } else {
                Wp = pk3(zero, zero); MV = pk3(zero, a_root); Vp = MV;
            }
            // body wrench from the state (robot_model.py:289-293) + what link i + 1 handed down
            V3 Hl, hl_a, Ha, ha_a;
            {
                const V3P Wc = pk3(w, al), Vc = pk3(v, a);
                upk3(inertia_lin_p(C.m, C.mc, Wc, Vc), Hl, hl_a);
                upk3(inertia_ang_p(C.Io, C.mc, Wc, Vc), Ha, ha_a);
            }
            const V3 f = cross_add(w, Hl, hl_a) + carry_f;
            const V3 nn = cross_add(w, Ha, cross_add(v, Hl, ha_a)) + carry_n;
            const V3P Rfn = rotz_p(pk3(f, nn), cs, sn);             // (Rz f | Rz n)
            V3 fp, np;
            upk3(mul_pv(C.F, Rfn), fp, np);
            np = cross_add(C.r, fp, np);
            carry_f = fp; carry_n = np;
            // wrench adjoints: theta
            float th = (nn.x * lam.y - nn.y * lam.x) + (f.x * mu.y - f.y * mu.x);
            // body part of the motion adjoints
            V3 wb = c_wb, vb = c_vb, alb = c_alb, ab = c_ab;
            const V3 Hlb = cross_add(mu, w, cross(lam, v));
            const V3 Hab = cross(lam, w);
            alb = cross_add(C.mc, mu, mulT_add(C.Io, lam, alb));
            ab = cross_add(lam, C.mc, fma3(C.m, mu, ab));
            wb = cross_add(Hl, mu, cross_add(Ha, lam, cross_add(C.mc, Hlb, mulT_add(C.Io, Hab, wb))));
            vb = cross_add(Hl, lam, cross_add(Hab, C.mc, fma3(C.m, Hlb, vb)));
            float vals[26];
            if (NEED_TABLE) {
                M3 Iob = zero3();
                add_outer(Iob, lam, al);
                add_outer(Iob, Hab, w);
                m3_to_array(Iob, vals + 12);
                const V3 mcb = cross_add(mu, al, cross_add(a, lam, cross_add(Hlb, w, cross(v, Hab))));
                vals[21] = mcb.x; vals[22] = mcb.y; vals[23] = mcb.z;
                vals[24] = dot(mu, a) + dot(Hlb, v);
                vals[25] = damp ? gk * qd_k : 0.f;
            }
            // kinematic part, in the order a, alpha, v, omega; wJ = (0, 0, qd_k)
            float wJb = ab.x * v.y - ab.y * v.x;                    // (ab x v).z
            vb.x = fmaf(-qd_k, ab.y, vb.x); vb.y = fmaf(qd_k, ab.x, vb.y);           // + (0, 0, qd) x ab
            wb.x = fmaf(-qd_k, alb.y, wb.x); wb.y = fmaf(qd_k, alb.x, wb.y);         // + (0, 0, qd) x alb
            wJb += alb.x * w.y - alb.y * w.x;                       // (alb x w).z
            wJb += wb.z;
            th += (ab.x * apre.y - ab.y * apre.x) + (alb.x * tal.y - alb.y * tal.x);
            th += (vb.x * v.y - vb.y * v.x) + (wb.x * w.y - wb.y * w.x);
            const V3P RW = rotz_p(pk3(wb, alb), cs, sn), RV = rotz_p(pk3(vb, ab), cs, sn);
            const V3P UW = mul_pv(C.F, RW), UV = mul_pv(C.F, RV);
            V3 uv, ua;
            upk3(UV, uv, ua);
            c_vb = uv; c_ab = ua;
            upk3(cross_add_p(UV, neg(C.r), UW), c_wb, c_alb);       // M wb + r x (M vb) | M alb + r x (M ab)
            if (c >= 0) {
                sts_f32(a_q + 4u * c, th);
                sts_f32(a_qd + 4u * c, damp ? fmaf(C.d, gk, wJb) : wJb);
                sts_f32(a_qdd + 4u * c, alb.z);
            }
            V3 wp, alp;
            upk3(Wp, wp, alp);
            if (NEED_TABLE) {
                // F-bar = sum x (Rz y-bar)^T over the six products through M, two per packed accumulator
                const V3P P1 = pk3(u, lamP);                        // pairs with (Rz f | Rz n)
                f32x2 b;
                float lo, hi;
#define DRM_FBAR(K, XI, RJ)                                                                      \
                b = fma2(Wp.XI, RW.RJ, fma2(MV.XI, RV.RJ, mul2(P1.XI, Rfn.RJ)));                 \
                upk2(b, lo, hi); vals[K] = lo + hi;
                DRM_FBAR(0, x, x) DRM_FBAR(1, x, y) DRM_FBAR(2, x, z)
                DRM_FBAR(3, y, x) DRM_FBAR(4, y, y) DRM_FBAR(5, y, z)
                DRM_FBAR(6, z, x) DRM_FBAR(7, z, y) DRM_FBAR(8, z, z)
#undef DRM_FBAR
                const V3 rbar = cross_add(ua, alp, cross_add(uv, wp, cross(fp, lamP)));
                vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z;
                chain_accumulate<26, T>(s_scr, s_acc + i * DRMB200_TABLE_STRIDE, vals);
            }
            w = wp; al = alp;
            upk3(Vp, v, a);
            lam = lamP; mu = muP;
        }

        if (bulk) {
            fence_proxy_async();
            __syncthreads();
            if (tid == 0) {
                const uint32_t bytes = (uint32_t)(valid * n) * 4u;
                if (args.q_grad != nullptr) bulk_s2g(args.q_grad + start * n, s_q, bytes);
                if (args.qd_grad != nullptr) bulk_s2g(args.qd_grad + start * n, s_qd, bytes);
                if (args.qdd_grad != nullptr) bulk_s2g(args.qdd_grad + start * n, s_qdd, bytes);
                bulk_commit();
                bulk_wait_read<0>();
            }
        } else {
            __syncthreads();
            if (args.q_grad != nullptr) coop_copy(args.q_grad + start * n, s_q, valid * n, vec_ok);
            if (args.qd_grad != nullptr) coop_copy(args.qd_grad + start * n, s_qd, valid * n, vec_ok);
            if (args.qdd_grad != nullptr) coop_copy(args.qdd_grad + start * n, s_qdd, valid * n, vec_ok);
        }
    }
    if (NEED_TABLE) {
        __syncthreads();
        float* out = args.partials + (size_t)blockIdx.x * N * DRMB200_TABLE_STRIDE;
        for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) {        // canonical -> natural (bijection per row)
            const int l = i / DRMB200_TABLE_STRIDE, e = i - l * DRMB200_TABLE_STRIDE;
            const int p = prog.parent[l];
            int src;
            const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
            out[l * DRMB200_TABLE_STRIDE + src] = sg * s_acc[i];
        }
    }
}

int inverse_dynamics_backward_device(const drmb200_topology_t* topo, const float* table, const float* q,
                                     const float* qd, const float* qdd, int64_t batch, uint32_t flags,
                                     const float* g_tau, float* q_grad, float* qd_grad, float* qdd_grad,
                                     float* table_grad, void* workspace, cudaStream_t stream) {
    TreeProgram prog;
    int rc = build_tree_program(topo, &prog);
    if (rc != DRMB200_OK) return rc;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (q_grad == nullptr && qd_grad == nullptr && qdd_grad == nullptr && table_grad == nullptr) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || qdd == nullptr || g_tau == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    if (table_grad != nullptr && workspace == nullptr) { set_error("table_grad requested without workspace"); return DRMB200_EINVAL; }

    RneaBwdArgs args;
    args.table = table; args.q = q; args.qd = qd; args.qdd = qdd; args.g_tau = g_tau;
    args.q_grad = q_grad; args.qd_grad = qd_grad; args.qdd_grad = qdd_grad;
    args.partials = static_cast<float*>(workspace); args.batch = batch; args.flags = flags;
    args.vec_ok = aligned16(q, qd, qdd, g_tau, q_grad, qd_grad, qdd_grad);

    if ((flags & DRMB200_INERTIAL_GRADS_ONLY) && table_grad != nullptr) {
        if (q_grad != nullptr || qd_grad != nullptr || qdd_grad != nullptr) {
            set_error("DRMB200_INERTIAL_GRADS_ONLY cannot be combined with input gradients");
            return DRMB200_EINVAL;
        }
        constexpr int TI = 128;
        const size_t sb = (size_t)RneaInertialSmem(TI, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float);
        if (sb > SMEM_CTA_MAX) { set_error("rnea inertial backward needs %zu B of shared memory (> 227 KB)", sb); return DRMB200_ELIMIT; }
        int g = 0;
        rc = launch_persistent<rnea_backward_inertial_kernel<TI>>(TI, sb, (batch + TI - 1) / TI, stream, "rnea inertial backward", &g,
                                                                  prog, args);
        if (rc != DRMB200_OK) return rc;
        return launch_reduce(args.partials, g, topo, table_grad, stream);
    }

    int grid = 0;
    const bool need_table = table_grad != nullptr;
    // a serial chain (every link's parent is the link before it): the two-sweep kernel
    bool chain = get_option(13) != 0 && prog.n_links >= 2;
    for (int i = 1; i < prog.n_links && chain; ++i) chain = prog.parent[i] == i - 1;
    if (chain) {
        // 64 rows per CTA: registers allow 7 CTAs (448 configurations) per SM; 128 only when 64 does not fit in shared memory
        int tile = 64;
        size_t sb = (size_t)RneaChainSmem(64, prog.n_dofs, prog.n_links).total_floats * sizeof(float);
        if (7 * (sb + 1024) > 228 * 1024 && (size_t)RneaChainSmem(32, prog.n_dofs, prog.n_links).total_floats * sizeof(float) <= SMEM_CTA_MAX) {
            tile = 32;
            sb = (size_t)RneaChainSmem(32, prog.n_dofs, prog.n_links).total_floats * sizeof(float);
        }
        if (sb <= SMEM_CTA_MAX) {
            const int64_t tiles = (batch + tile - 1) / tile;
#define DRM_LAUNCH_IDC(NT, TT) \
    rc = launch_persistent<rnea_backward_chain_kernel<NT, TT>>(TT, sb, tiles, stream, "rnea chain backward", &grid, prog, args)
            if (need_table) { if (tile == 64) DRM_LAUNCH_IDC(true, 64); else DRM_LAUNCH_IDC(true, 32); }
            else            { if (tile == 64) DRM_LAUNCH_IDC(false, 64); else DRM_LAUNCH_IDC(false, 32); }
#undef DRM_LAUNCH_IDC
            if (rc != DRMB200_OK) return rc;
            return need_table ? launch_reduce(args.partials, grid, topo, table_grad, stream) : DRMB200_OK;
        }
    }

    // shared memory (8 floats per link + 12 per chain end, per configuration) is the occupancy limiter: pick the
    // tile that keeps the most warps resident per SM, larger tile on ties
    int tile = 32, best_warps = 0;
    for (int t = 128; t >= 32; t >>= 1) {
        const size_t b = (size_t)RneaBwdSmem(t, prog.n_dofs, prog.n_links, prog.n_slots, prog.n_tips).total_floats * sizeof(float) + 1024;
        const int warps = b > SMEM_CTA_MAX ? 0 : (int)(SMEM_CTA_MAX / b) * (t / 32);
        if (warps > best_warps) { best_warps = warps; tile = t; }
    }
    const size_t smem_bytes = (size_t)RneaBwdSmem(tile, prog.n_dofs, prog.n_links, prog.n_slots, prog.n_tips).total_floats * sizeof(float);
    if (smem_bytes > SMEM_CTA_MAX) { set_error("rnea backward needs %zu B of shared memory per CTA (> 227 KB): model too large", smem_bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (batch + tile - 1) / tile;
#define DRM_LAUNCH_IDB(NT, TT) \
    rc = launch_persistent<rnea_backward_kernel<NT, TT>>(TT, smem_bytes, tiles, stream, "rnea backward", &grid, prog, args)
    if (need_table) { if (tile == 128) DRM_LAUNCH_IDB(true, 128); else if (tile == 64) DRM_LAUNCH_IDB(true, 64); else DRM_LAUNCH_IDB(true, 32); }
    else            { if (tile == 128) DRM_LAUNCH_IDB(false, 128); else if (tile == 64) DRM_LAUNCH_IDB(false, 64); else DRM_LAUNCH_IDB(false, 32); }
#undef DRM_LAUNCH_IDB
    if (rc != DRMB200_OK) return rc;
    return need_table ? launch_reduce(args.partials, grid, topo, table_grad, stream) : DRMB200_OK;
}

}  // namespace drm
