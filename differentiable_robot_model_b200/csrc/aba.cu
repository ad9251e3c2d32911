// aba.cu -- batched articulated-body forward dynamics (sm_90a).
//
// Replaces, in ONE launch, DifferentiableRobotModel.compute_forward_dynamics (robot_model.py:488-624):
// update_kinematic_state (robot_model.py:140-195), the bias pass (:537-545), the articulated-inertia pass
// leaves->root with its per-link 6x6 matrices (:547-596) and the acceleration pass root->leaves (:604-622).
//
// The reference's arithmetic is kept, including where it departs from the textbook algorithm:
//   * U = IA S is used as a COLUMN both in the rank-1 update IA - U U^T/(d + 1e-37) and in
//     qdd = (u - U . a')/d (:555-557, :569-577, :621), so a non-symmetric inertia_mat (which the reference never
//     symmetrises and its forward-dynamics example learns freely) gives the reference's answer, not H^-1 (f - nle);
//     the articulated inertia is therefore carried as a GENERAL 6x6 (four 3x3 blocks), not a symmetric 21-vector;
//   * the +1e-37 regularisers (:570, :582);
//   * fixed links are "joints" with a zero axis: U = 0, d = 0, u = 0 and nothing is eliminated (:550-561).
//
// Closed form, link i with parent p, canonical joint frames of drm_common.cuh (joint axis e_z, spatial vectors
// [ang; lin], M = F~ Rz(q), E = M^T, r = r~, motion transform X = [[E, 0], [-E r^, E]]):
//   pass 1  w_i = E w_p + (0,0,qd), v_i = E (v_p + w_p x r);  c_i = (w_i x (0,0,qd); v_i x (0,0,qd))
//           h = I_i (w_i; v_i);  pA_i = (w x h_ang + v x h_lin; w x h_lin);  IA_i = [[Io, mc^], [mc^T, m 1]]
//   pass 2  U = IA e_z(ang), d = U_z(ang), u = f_i - pA_i,z(ang);  IA' = IA - U U^T / (d + eps)
//           pa = pA + IA' c + U u / (d + eps);  IA_p += X^T IA' X;  pA_p += X^T pa
//   pass 3  a' = X a_p + c_i;  qdd_i = (u - U . a') / d;  a_i = a' + e_z(ang) qdd_i          (a_0 = (0; 0,0,9.81))
//
// Mapping: one thread per configuration, T per CTA.  The articulated inertia of the link being eliminated lives in
// registers (36 + 6 floats) and is handed to the parent through registers when the parent is the previous link; only
// branch points accumulate in shared-memory slots (the tree program's save / accw fields).  Per link the kernel
// keeps 14 floats in shared memory, slot-major: cos, sin, the 4 non-zero entries of c, pA (later overwritten by U),
// u and d.  q / qd / f tiles in and the qdd tile out move as TMA 1-D bulk copies.
//
// Algorithmic HBM bytes per configuration: 12n in + 4n out = 16n (112 B at n = 7); at roughly 6 kflop per 7-DoF
// configuration the kernel is FP32-issue-bound, like RNEA.
#include "drm_common.cuh"

namespace drm {

constexpr float ABA_GRAVITY = 9.81f;     // robot_model.py:530
constexpr float ABA_EPS = 1e-37f;        // robot_model.py:570, 582
constexpr int ABA_LINK = 14;             // floats per link in shared memory
constexpr int ABA_SLOT = 42;             // floats per branch slot (6x6 + 6)

struct AbaArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ f;
    float* __restrict__ qdd;
    int64_t batch;
    uint32_t flags;
    int32_t aligned;
};

struct AbaSmemLayout {
    int q, qd, f, qdd, table, link, slots, total_floats;
    __host__ __device__ AbaSmemLayout(int T, int n, int n_links, int n_slots) {
        int o = 0;
        q = o;   o += T * n;
        qd = o;  o += T * n;
        f = o;   o += T * n;
        qdd = o; o += T * n;
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o;  o += n_links * ABA_LINK * T;
        slots = o; o += n_slots * ABA_SLOT * T;
        total_floats = o;
    }
};

struct M6 { M3 A, B, C, D; };       // [[A, B], [C, D]] acting on [ang; lin]

__device__ __forceinline__ M3 operator+(const M3& a, const M3& b) {
    M3 r;
    r.a00 = a.a00 + b.a00; r.a01 = a.a01 + b.a01; r.a02 = a.a02 + b.a02;
    r.a10 = a.a10 + b.a10; r.a11 = a.a11 + b.a11; r.a12 = a.a12 + b.a12;
    r.a20 = a.a20 + b.a20; r.a21 = a.a21 + b.a21; r.a22 = a.a22 + b.a22;
    return r;
}
__device__ __forceinline__ M3 operator-(const M3& a, const M3& b) {
    M3 r;
    r.a00 = a.a00 - b.a00; r.a01 = a.a01 - b.a01; r.a02 = a.a02 - b.a02;
    r.a10 = a.a10 - b.a10; r.a11 = a.a11 - b.a11; r.a12 = a.a12 - b.a12;
    r.a20 = a.a20 - b.a20; r.a21 = a.a21 - b.a21; r.a22 = a.a22 - b.a22;
    return r;
}
__device__ __forceinline__ M3 skew(V3 a) {          // skew(a) b = a x b
    M3 r;
    r.a00 = 0.f;  r.a01 = -a.z; r.a02 = a.y;
    r.a10 = a.z;  r.a11 = 0.f;  r.a12 = -a.x;
    r.a20 = -a.y; r.a21 = a.x;  r.a22 = 0.f;
    return r;
}
__device__ __forceinline__ M3 from_cols(V3 c0, V3 c1, V3 c2) {
    M3 r;
    r.a00 = c0.x; r.a10 = c0.y; r.a20 = c0.z; r.a01 = c1.x; r.a11 = c1.y; r.a21 = c1.z; r.a02 = c2.x; r.a12 = c2.y; r.a22 = c2.z;
    return r;
}
__device__ __forceinline__ M3 from_rows(V3 r0, V3 r1, V3 r2) {
    M3 r;
    r.a00 = r0.x; r.a01 = r0.y; r.a02 = r0.z; r.a10 = r1.x; r.a11 = r1.y; r.a12 = r1.z; r.a20 = r2.x; r.a21 = r2.y; r.a22 = r2.z;
    return r;
}
__device__ __forceinline__ V3 row0(const M3& m) { return v3(m.a00, m.a01, m.a02); }
__device__ __forceinline__ V3 row1(const M3& m) { return v3(m.a10, m.a11, m.a12); }
__device__ __forceinline__ V3 row2(const M3& m) { return v3(m.a20, m.a21, m.a22); }
// skew(r) Y: every column crossed from the left;  Y skew(r): every row crossed from the right
__device__ __forceinline__ M3 left_cross(V3 r, const M3& Y) { return from_cols(cross(r, col0(Y)), cross(r, col1(Y)), cross(r, col2(Y))); }
__device__ __forceinline__ M3 right_cross(const M3& Y, V3 r) { return from_rows(cross(row0(Y), r), cross(row1(Y), r), cross(row2(Y), r)); }
__device__ __forceinline__ void sub_outer(M3& m, V3 x, V3 y) {      // m -= x y^T
    m.a00 = fmaf(-x.x, y.x, m.a00); m.a01 = fmaf(-x.x, y.y, m.a01); m.a02 = fmaf(-x.x, y.z, m.a02);
    m.a10 = fmaf(-x.y, y.x, m.a10); m.a11 = fmaf(-x.y, y.y, m.a11); m.a12 = fmaf(-x.y, y.z, m.a12);
    m.a20 = fmaf(-x.z, y.x, m.a20); m.a21 = fmaf(-x.z, y.y, m.a21); m.a22 = fmaf(-x.z, y.z, m.a22);
}
__device__ __forceinline__ M3 conj_by(const M3& M, const M3& Y) { return mulNT(mul(M, Y), M); }   // M Y M^T

// ---- element-wise PAIR of two 3x3 blocks (lo | hi) as f32x2 lanes --------------------------------------------------
struct M3PP { f32x2 a00, a01, a02, a10, a11, a12, a20, a21, a22; };
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return pk2(__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)); }
__device__ __forceinline__ float hsum2(f32x2 v) { float lo, hi; upk2(v, lo, hi); return lo + hi; }
__device__ __forceinline__ M3PP pkm(const M3& lo, const M3& hi) {
    M3PP r;
    r.a00 = pk2(lo.a00, hi.a00); r.a01 = pk2(lo.a01, hi.a01); r.a02 = pk2(lo.a02, hi.a02);
    r.a10 = pk2(lo.a10, hi.a10); r.a11 = pk2(lo.a11, hi.a11); r.a12 = pk2(lo.a12, hi.a12);
    r.a20 = pk2(lo.a20, hi.a20); r.a21 = pk2(lo.a21, hi.a21); r.a22 = pk2(lo.a22, hi.a22);
    return r;
}
__device__ __forceinline__ void upkm(const M3PP& p, M3& lo, M3& hi) {
    upk2(p.a00, lo.a00, hi.a00); upk2(p.a01, lo.a01, hi.a01); upk2(p.a02, lo.a02, hi.a02);
    upk2(p.a10, lo.a10, hi.a10); upk2(p.a11, lo.a11, hi.a11); upk2(p.a12, lo.a12, hi.a12);
    upk2(p.a20, lo.a20, hi.a20); upk2(p.a21, lo.a21, hi.a21); upk2(p.a22, lo.a22, hi.a22);
}
__device__ __forceinline__ M3PP zero_pp() { const M3 z = zero3(); return pkm(z, z); }
__device__ __forceinline__ M3PP add_pp(const M3PP& a, const M3PP& b) {
    M3PP r;
    r.a00 = add2(a.a00, b.a00); r.a01 = add2(a.a01, b.a01); r.a02 = add2(a.a02, b.a02);
    r.a10 = add2(a.a10, b.a10); r.a11 = add2(a.a11, b.a11); r.a12 = add2(a.a12, b.a12);
    r.a20 = add2(a.a20, b.a20); r.a21 = add2(a.a21, b.a21); r.a22 = add2(a.a22, b.a22);
    return r;
}
// (M Y_lo | M Y_hi): scalar matrix from the left, same association order as mul(M3, M3)
__device__ __forceinline__ M3PP mul_left_pp(const M3& m, const M3PP& y) {
    M3PP r;
    r.a00 = fma2(bc2(m.a00), y.a00, fma2(bc2(m.a01), y.a10, mul2(bc2(m.a02), y.a20)));
    r.a01 = fma2(bc2(m.a00), y.a01, fma2(bc2(m.a01), y.a11, mul2(bc2(m.a02), y.a21)));
    r.a02 = fma2(bc2(m.a00), y.a02, fma2(bc2(m.a01), y.a12, mul2(bc2(m.a02), y.a22)));
    r.a10 = fma2(bc2(m.a10), y.a00, fma2(bc2(m.a11), y.a10, mul2(bc2(m.a12), y.a20)));
    r.a11 = fma2(bc2(m.a10), y.a01, fma2(bc2(m.a11), y.a11, mul2(bc2(m.a12), y.a21)));
    r.a12 = fma2(bc2(m.a10), y.a02, fma2(bc2(m.a11), y.a12, mul2(bc2(m.a12), y.a22)));
    r.a20 = fma2(bc2(m.a20), y.a00, fma2(bc2(m.a21), y.a10, mul2(bc2(m.a22), y.a20)));
    r.a21 = fma2(bc2(m.a20), y.a01, fma2(bc2(m.a21), y.a11, mul2(bc2(m.a22), y.a21)));
    r.a22 = fma2(bc2(m.a20), y.a02, fma2(bc2(m.a21), y.a12, mul2(bc2(m.a22), y.a22)));
    return r;
}
// (Y_lo M^T | Y_hi M^T)
__device__ __forceinline__ M3PP mul_rightT_pp(const M3PP& y, const M3& m) {
    M3PP r;
    r.a00 = fma2(y.a00, bc2(m.a00), fma2(y.a01, bc2(m.a01), mul2(y.a02, bc2(m.a02))));
    r.a01 = fma2(y.a00, bc2(m.a10), fma2(y.a01, bc2(m.a11), mul2(y.a02, bc2(m.a12))));
    r.a02 = fma2(y.a00, bc2(m.a20), fma2(y.a01, bc2(m.a21), mul2(y.a02, bc2(m.a22))));
    r.a10 = fma2(y.a10, bc2(m.a00), fma2(y.a11, bc2(m.a01), mul2(y.a12, bc2(m.a02))));
    r.a11 = fma2(y.a10, bc2(m.a10), fma2(y.a11, bc2(m.a11), mul2(y.a12, bc2(m.a12))));
    r.a12 = fma2(y.a10, bc2(m.a20), fma2(y.a11, bc2(m.a21), mul2(y.a12, bc2(m.a22))));
    r.a20 = fma2(y.a20, bc2(m.a00), fma2(y.a21, bc2(m.a01), mul2(y.a22, bc2(m.a02))));
    r.a21 = fma2(y.a20, bc2(m.a10), fma2(y.a21, bc2(m.a11), mul2(y.a22, bc2(m.a12))));
    r.a22 = fma2(y.a20, bc2(m.a20), fma2(y.a21, bc2(m.a21), mul2(y.a22, bc2(m.a22))));
    return r;
}
__device__ __forceinline__ M3PP conj_pp(const M3& m, const M3PP& y) { return mul_rightT_pp(mul_left_pp(m, y), m); }   // M Y M^T
// skew(r) Y on both lanes: column j of the result = r x column j
__device__ __forceinline__ M3PP left_cross_pp(V3 r, const M3PP& y) {
    M3PP o;
    o.a00 = fma2(bc2(r.y), y.a20, mul2(bc2(-r.z), y.a10)); o.a10 = fma2(bc2(r.z), y.a00, mul2(bc2(-r.x), y.a20)); o.a20 = fma2(bc2(r.x), y.a10, mul2(bc2(-r.y), y.a00));
    o.a01 = fma2(bc2(r.y), y.a21, mul2(bc2(-r.z), y.a11)); o.a11 = fma2(bc2(r.z), y.a01, mul2(bc2(-r.x), y.a21)); o.a21 = fma2(bc2(r.x), y.a11, mul2(bc2(-r.y), y.a01));
    o.a02 = fma2(bc2(r.y), y.a22, mul2(bc2(-r.z), y.a12)); o.a12 = fma2(bc2(r.z), y.a02, mul2(bc2(-r.x), y.a22)); o.a22 = fma2(bc2(r.x), y.a12, mul2(bc2(-r.y), y.a02));
    return o;
}
// Y -= x yp^T with a scalar left vector x and a PAIR right vector yp (one vector per lane)
__device__ __forceinline__ void sub_outer_pp(M3PP& m, V3 x, const V3P& yp) {
    m.a00 = fma2(bc2(-x.x), yp.x, m.a00); m.a01 = fma2(bc2(-x.x), yp.y, m.a01); m.a02 = fma2(bc2(-x.x), yp.z, m.a02);
    m.a10 = fma2(bc2(-x.y), yp.x, m.a10); m.a11 = fma2(bc2(-x.y), yp.y, m.a11); m.a12 = fma2(bc2(-x.y), yp.z, m.a12);
    m.a20 = fma2(bc2(-x.z), yp.x, m.a20); m.a21 = fma2(bc2(-x.z), yp.y, m.a21); m.a22 = fma2(bc2(-x.z), yp.z, m.a22);
}

template <int T>
__global__ void __launch_bounds__(T)
aba_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const AbaArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = prog.n_dofs;
    const int N = prog.n_links;
    const AbaSmemLayout L(T, n, N, prog.n_slots);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_f = smem + L.f;
    float* s_qdd = smem + L.qdd;
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_slot = smem + L.slots;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, args.batch - tile_start);
    const bool vec_ok = args.aligned;
    const bool bulk = args.aligned && ((valid & 3) == 0);

    if (bulk) {
        if (tid == 0) {
            mbar_init(&mbar, 1);
            fence_mbar_init();
            const uint32_t bytes = (uint32_t)valid * n * 4u;
            mbar_arrive_expect_tx(&mbar, 3u * bytes);
            bulk_g2s(s_q, args.q + tile_start * n, bytes, &mbar);
            bulk_g2s(s_qd, args.qd + tile_start * n, bytes, &mbar);
            bulk_g2s(s_f, args.f + tile_start * n, bytes, &mbar);
        }
    } else {
        coop_copy(s_q, args.q + tile_start * n, valid * n, vec_ok);
        coop_copy(s_qd, args.qd + tile_start * n, valid * n, vec_ok);
        coop_copy(s_f, args.f + tile_start * n, valid * n, vec_ok);
    }
    // fold.n_red > 0: fixed links folded into their movable ancestors, prog is the reduced tree (drm_common.cuh): a fixed
    // joint has S = 0, so its articulated inertia and bias force pass to the parent through a constant transform -- the fold
    if (fold.n_red > 0 && fold.n_full == 0) {                // args.table holds rows folded beforehand (drmb200_fold_link_table)
        for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) s_tab[i] = __ldg(args.table + i);
    } else if (fold.n_red > 0) {
        stage_folded_table(s_tab, s_link, args.table, fold, prog, T);
    } else {
        stage_canonical_table(s_tab, args.table, prog, T);
    }
    __syncthreads();
    if (bulk) mbar_wait(&mbar, 0);

    if (tid < valid) {
        const float* qrow = s_q + tid * n;
        const float* qdrow = s_qd + tid * n;
        const float* frow = s_f + tid * n;
        float* outrow = s_qdd + tid * n;
        float* lk0 = s_link + tid;
        float* sl0 = s_slot + tid;
        const float g = (args.flags & DRMB200_GRAVITY) ? ABA_GRAVITY : 0.f;
        const bool damp = (args.flags & DRMB200_DAMPING) != 0;
        const V3 zero = v3(0.f, 0.f, 0.f);

        // ---- pass 1: root -> leaves, velocities, velocity-product terms c and bias forces pA ----------------
        {
            V3 w = zero, v = zero;
            for (int i = 1; i < N; ++i) {
                const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
                const int src = prog.psrc[i];
                V3 wp, vp;
                if (src == 0) { wp = w; vp = v; }
                else if (src < 0) { wp = vp = zero; }
                else { const float* sl = sl0 + (src - 1) * ABA_SLOT * T; wp = ldv(sl, T); vp = ldv(sl + 3 * T, T); }
                M3 M = C.F;
                const int c = prog.dof[i];
                float cs = 1.f, sn = 0.f, qd_k = 0.f;
                if (c >= 0) {
                    qd_k = qdrow[c];
                    sincos_pi2(qrow[c], sn, cs);
                    rotate_z(M, cs, sn);
                }
                w = mulT(M, wp); w.z += qd_k;                                    // robot_model.py:183-193
                v = mulT(M, cross_add(wp, C.r, vp));
                const V3 ca = cross_z(w, qd_k), cl = cross_z(v, qd_k);           // robot_model.py:541
                const V3 hl = C.m * v - cross(C.mc, w);                          // sva:321-338
                const V3 ha = mul_add(C.Io, w, cross(C.mc, v));
                const V3 pa_ang = cross_add(w, ha, cross(v, hl));                // robot_model.py:543, sva:215-224
                const V3 pa_lin = cross(w, hl);
                float* lk = lk0 + i * ABA_LINK * T;
                lk[0] = cs; lk[T] = sn; lk[2 * T] = ca.x; lk[3 * T] = ca.y; lk[4 * T] = cl.x; lk[5 * T] = cl.y;
                stv(lk + 6 * T, T, pa_ang); stv(lk + 9 * T, T, pa_lin);
                const int sv = prog.save[i];
                if (sv >= 0) { float* sl = sl0 + sv * ABA_SLOT * T; stv(sl, T, w); stv(sl + 3 * T, T, v); }
            }
        }

        // ---- pass 2: leaves -> root, articulated inertias (robot_model.py:547-596) ---------------------------
        // f32x2 pairs: the 6x6 travels as two element-wise PAIRS of 3x3 blocks, AB = (A | B) and CD = (C | D) -- both
        // blocks of a pair see the same rotation M . M^T, the same left cross product with r and the same left factor of
        // the rank-1 update, so each of those operations is written once for both blocks.
        {
            M3PP cAB = zero_pp(), cCD = zero_pp();       // contribution of link i+1 to its parent i, through registers
            V3 c_pang = zero, c_plin = zero;
            for (int i = N - 1; i >= 1; --i) {
                const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
                float* lk = lk0 + i * ABA_LINK * T;
                M3 D0 = zero3(); D0.a00 = D0.a11 = D0.a22 = C.m;
                const M3 B0 = skew(C.mc);
                M3PP AB = pkm(C.Io, B0), CD = pkm(transpose(B0), D0);               // sva:340-372
                V3 p_ang = ldv(lk + 6 * T, T), p_lin = ldv(lk + 9 * T, T);
                if (i + 1 < N && prog.psrc[i + 1] == 0) {
                    AB = add_pp(AB, cAB); CD = add_pp(CD, cCD);
                    p_ang = p_ang + c_pang; p_lin = p_lin + c_plin;
                }
                const int sv = prog.save[i];
                if (sv >= 0) {
                    const float* sl = sl0 + sv * ABA_SLOT * T;
                    AB = add_pp(AB, pkm(ldm(sl, T), ldm(sl + 9 * T, T)));
                    CD = add_pp(CD, pkm(ldm(sl + 18 * T, T), ldm(sl + 27 * T, T)));
                    p_ang = p_ang + ldv(sl + 36 * T, T); p_lin = p_lin + ldv(sl + 39 * T, T);
                }
                const int c = prog.dof[i];
                V3 Ua = zero, Ul = zero;
                float d = 0.f, u = 0.f;
                if (c >= 0) {
                    float t;
                    upk2(AB.a02, Ua.x, t); upk2(AB.a12, Ua.y, t); upk2(AB.a22, Ua.z, t);    // U = IA S, S = e_z(ang)   (:555)
                    upk2(CD.a02, Ul.x, t); upk2(CD.a12, Ul.y, t); upk2(CD.a22, Ul.z, t);
                    d = Ua.z;                                                      // S . U                    (:557)
                    float fk = frow[c];
                    if (damp) fk = fmaf(-C.d, qdrow[c], fk);                       // f -= damping * qd        (:516-521)
                    u = fk - p_ang.z;                                              // (:559)
                }
                const int P = prog.parent[i];
                if (P > 0) {
                    const float cs = lk[0], sn = lk[T];
                    V3 pa_ang = p_ang, pa_lin = p_lin;
                    if (c >= 0) {
                        const float inv = 1.f / (d + ABA_EPS);                     // (:569-571, :581-583)
                        const V3P Ud = pk3(inv * Ua, inv * Ul);                    // (Ud_ang | Ud_lin)
                        sub_outer_pp(AB, Ua, Ud);                                  // IA - U Ud^T              (:575-577)
                        sub_outer_pp(CD, Ul, Ud);
                        const f32x2 cx = pk2(lk[2 * T], lk[4 * T]), cy = pk2(lk[3 * T], lk[5 * T]);   // (c_ang | c_lin), z = 0
                        const float ud = u * inv;
                        // pa = pA + IA' c + U ud                                                               (:579-585)
                        pa_ang.x += hsum2(fma2(AB.a00, cx, mul2(AB.a01, cy))) + Ua.x * ud;
                        pa_ang.y += hsum2(fma2(AB.a10, cx, mul2(AB.a11, cy))) + Ua.y * ud;
                        pa_ang.z += hsum2(fma2(AB.a20, cx, mul2(AB.a21, cy))) + Ua.z * ud;
                        pa_lin.x += hsum2(fma2(CD.a00, cx, mul2(CD.a01, cy))) + Ul.x * ud;
                        pa_lin.y += hsum2(fma2(CD.a10, cx, mul2(CD.a11, cy))) + Ul.y * ud;
                        pa_lin.z += hsum2(fma2(CD.a20, cx, mul2(CD.a21, cy))) + Ul.z * ud;
                    }
                    // X^T IA' X = T^T (M IA' M^T) T with T = [[1, 0], [-r^, 1]]                                 (:587-595)
                    M3 M = C.F;
                    if (c >= 0) rotate_z(M, cs, sn);
                    M3PP Yab = conj_pp(M, AB);                                     // (A^ | B^)
                    M3PP Ycd = conj_pp(M, CD);                                     // (C^ | D^)
                    Yab = add_pp(Yab, left_cross_pp(C.r, Ycd));                    // (A^ + r^ C^ | B^ + r^ D^) = (. | Y_B)
                    {
                        M3 Ya, Yb, Yc, Yd;
                        upkm(Yab, Ya, Yb); upkm(Ycd, Yc, Yd);
                        Ya = Ya - right_cross(Yb, C.r);                            // Y_A = A^ + r^ C^ - Y_B r^
                        Yc = Yc - right_cross(Yd, C.r);                            // Y_C = C^ - D^ r^
                        Yab = pkm(Ya, Yb); Ycd = pkm(Yc, Yd);
                    }
                    // force transform (sva:281-291)
                    const V3 q_lin = mul(M, pa_lin);
                    const V3 q_ang = cross_add(C.r, q_lin, mul(M, pa_ang));
                    if (P == i - 1) { cAB = Yab; cCD = Ycd; c_pang = q_ang; c_plin = q_lin; }
                    else {
                        float* sl = sl0 + (int)prog.save[P] * ABA_SLOT * T;
                        M3 Ya, Yb, Yc, Yd;
                        upkm(Yab, Ya, Yb); upkm(Ycd, Yc, Yd);
                        if (prog.accw[i] != 2) {
                            Ya = Ya + ldm(sl, T); Yb = Yb + ldm(sl + 9 * T, T);
                            Yc = Yc + ldm(sl + 18 * T, T); Yd = Yd + ldm(sl + 27 * T, T);
                            stv(sl + 36 * T, T, ldv(sl + 36 * T, T) + q_ang); stv(sl + 39 * T, T, ldv(sl + 39 * T, T) + q_lin);
                        } else {
                            stv(sl + 36 * T, T, q_ang); stv(sl + 39 * T, T, q_lin);
                        }
                        stm(sl, T, Ya); stm(sl + 9 * T, T, Yb); stm(sl + 18 * T, T, Yc); stm(sl + 27 * T, T, Yd);
                    }
                }
                stv(lk + 6 * T, T, Ua); stv(lk + 9 * T, T, Ul);                    // pA_i is dead: keep U, u, d for pass 3
                lk[12 * T] = u; lk[13 * T] = d;
            }
        }

        // ---- pass 3: root -> leaves, accelerations (robot_model.py:604-622) ----------------------------------
        {
            V3 al = zero, a = zero;
            for (int i = 1; i < N; ++i) {
                const float* row = s_tab + i * DRMB200_TABLE_STRIDE;
                M3 M; V3 r;
                load_Fr(row, M, r);
                const float* lk = lk0 + i * ABA_LINK * T;
                const int src = prog.psrc[i];
                V3 alp, ap;
                if (src == 0) { alp = al; ap = a; }
                else if (src < 0) { alp = zero; ap = v3(0.f, 0.f, g); }
                else { const float* sl = sl0 + (src - 1) * ABA_SLOT * T; alp = ldv(sl, T); ap = ldv(sl + 3 * T, T); }
                const int c = prog.dof[i];
                if (c >= 0) rotate_z(M, lk[0], lk[T]);
                al = mulT(M, alp);                                                 // acc_parent.transform(inv_pose)  (:611-614)
                a = mulT(M, cross_add(alp, r, ap));
                if (c >= 0) {
                    al.x += lk[2 * T]; al.y += lk[3 * T]; a.x += lk[4 * T]; a.y += lk[5 * T];     // + c   (:616)
                    const V3 Ua = ldv(lk + 6 * T, T), Ul = ldv(lk + 9 * T, T);
                    const float u = lk[12 * T], d = lk[13 * T];
                    const float qdd = (1.0f / d) * (u - (dot(Ua, al) + dot(Ul, a)));             // (:621)
                    outrow[c] = qdd;
                    al.z += qdd;                                                                  // (:622)
                }
                const int sv = prog.save[i];
                if (sv >= 0) { float* sl = sl0 + sv * ABA_SLOT * T; stv(sl, T, al); stv(sl + 3 * T, T, a); }
            }
        }
    }

    if (bulk) {
        fence_proxy_async();
        __syncthreads();
        if (tid == 0) {
            bulk_s2g(args.qdd + tile_start * n, s_qdd, (uint32_t)valid * n * 4u);
            bulk_commit();
            bulk_wait_read<0>();
        }
    } else {
        __syncthreads();
        coop_copy(args.qdd + tile_start * n, s_qdd, valid * n, vec_ok);
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <int T>
static int launch_aba(const TreeProgram& prog, const FoldProgram& fold, const AbaArgs& args, size_t smem_bytes, cudaStream_t stream) {
    static size_t configured_by_dev[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    size_t& configured = configured_by_dev[dev & 63];
    if (smem_bytes > configured) {
        cudaError_t e = cudaFuncSetAttribute(aba_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%zu B smem): %s", smem_bytes, cudaGetErrorString(e)); return DRMB200_ECUDA; }
        configured = smem_bytes;
    }
    const int64_t tiles = (args.batch + T - 1) / T;
    if (tiles > 0x7fffffffLL) { set_error("batch too large for one launch"); return DRMB200_EINVAL; }
    aba_kernel<T><<<(unsigned)tiles, T, smem_bytes, stream>>>(prog, fold, args);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("aba launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}

static int forward_dynamics_device_impl(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                       const float* f, int64_t batch, uint32_t flags, float* qdd, cudaStream_t stream,
                                       bool prefolded) {
    int rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);
    if (cp == nullptr) return rc;
    if (prefolded && !cp->foldable) { set_error("this topology has no link behind a fixed joint to fold"); return DRMB200_EINVAL; }
    const bool folded = prefolded || (cp->foldable && get_option(11) != 0);      // "rnea_fold"
    const TreeProgram& prog = folded ? cp->red : cp->full;
    FoldProgram fold = cp->fold;
    if (!folded) fold.n_red = 0;
    if (prefolded) fold.n_full = 0;                     // `table` holds the rows of drmb200_fold_link_table
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || f == nullptr || qdd == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }

    AbaArgs args;
    args.table = table; args.q = q; args.qd = qd; args.f = f; args.qdd = qdd; args.batch = batch; args.flags = flags;
    auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    args.aligned = (al16(q) && al16(qd) && al16(f) && al16(qdd)) ? 1 : 0;

    // 64 configurations per CTA unless the model's per-link state would leave a single CTA per SM
    auto bytes_of = [&](int T) { return (size_t)AbaSmemLayout(T, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float); };
    const int tile = bytes_of(64) <= 113 * 1024 ? 64 : 32;
    const size_t smem_bytes = bytes_of(tile);
    if (smem_bytes > 227 * 1024) { set_error("model needs %zu B of shared memory per CTA (> 227 KB)", smem_bytes); return DRMB200_ELIMIT; }
    return tile == 64 ? launch_aba<64>(prog, fold, args, smem_bytes, stream) : launch_aba<32>(prog, fold, args, smem_bytes, stream);
}

int forward_dynamics_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                            const float* f, int64_t batch, uint32_t flags, float* qdd, cudaStream_t stream) {
    return forward_dynamics_device_impl(topo, table, q, qd, f, batch, flags, qdd, stream, false);
}
int forward_dynamics_prefolded_device(const drmb200_topology_t* topo, const float* folded, const float* q, const float* qd,
                                      const float* f, int64_t batch, uint32_t flags, float* qdd, cudaStream_t stream) {
    return forward_dynamics_device_impl(topo, folded, q, qd, f, batch, flags, qdd, stream, true);
}

}  // namespace drm
