// backward_aba.cu -- analytic adjoint of the articulated-body forward-dynamics kernel (sm_90a).
//
// The reference differentiates its per-link op graph of compute_forward_dynamics (robot_model.py:488-624) with
// autograd; this kernel evaluates the hand-derived reverse-mode recursions instead (stated and verified against
// autograd in oracle/adjoint_proto.py: forward_dynamics_with_backward), one thread per configuration:
//
//   forward recompute   F1 root->leaves: cos/sin, (w, v), pA0, IA0        (aba.cu pass 1)
//                       F2 leaves->root: IA_i, pA_i accumulated, u        (aba.cu pass 2; parents accumulate in place)
//                       F3 root->leaves: (al, a)                          (aba.cu pass 3)
//   adjoint             R3 leaves->root: reverse of F3 -> U-bar, d-bar, u-bar, c-bar, acceleration adjoints
//                       R2 root->leaves: reverse of F2 -> IA-bar_i (6x6), pA-bar_i, f-bar, inertial table columns
//                       R1 leaves->root: reverse of F1 -> velocity adjoints, qd-bar
//   every reverse pass adds its share of M-bar (-> q-bar, F-bar) and r-bar.
//
// Per link and configuration 33 floats stay in shared memory (slot-major): cos sin | w v | pA -> pA-bar | u |
// al a -> U-bar | adjoint accumulator (6) | d-bar u-bar | c-bar (4).  The 6x6 articulated inertia IA_i (36 floats, later
// overwritten by its adjoint) lives in a per-CTA slice of a GLOBAL scratch instead: the CTAs are persistent, so the whole
// scratch is (#CTAs x links x 36 x 32 floats, about 21 MB for the Kuka at five CTAs on each of 132 SMs) and stays
// resident in the 50 MB L2; every access is a
// coalesced 128-byte line of lane-private values.  With IA in shared memory (69 floats per link) only two single-warp CTAs
// fit per SM -- two of the four schedulers idle; this layout runs four to five.
// Table gradients: per-CTA accumulators in canonical frames, un-permuted into per-CTA partial tables, then the
// fixed-order reduce kernel of backward.cu (deterministic, no atomics).
#include "backward_common.cuh"

namespace drm {

constexpr float ABA_EPS_B = 1e-37f;
constexpr int AL = 33;            // floats per link in shared memory (+ 36 per link in the L2-resident scratch)
constexpr int O_CS = 0, O_W = 2, O_PA = 8, O_U = 14, O_AL = 15, O_ADJ = 21, O_DB = 27, O_UB = 28, O_CB = 29;
constexpr int IA_FLOATS = 36;     // the 6x6 articulated inertia (-> its adjoint) of a link, global scratch

struct AbaBwdArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ f;
    const float* __restrict__ g_qdd;
    float* __restrict__ q_grad;
    float* __restrict__ qd_grad;
    float* __restrict__ f_grad;
    float* __restrict__ partials;
    float* __restrict__ scratch;       // [grid][n_links - 1][36][T]: IA_i, later IA-bar_i (stays in L2)
    int64_t batch;
    uint32_t flags;
    int32_t vec_ok;
};

struct AbaBwdSmem {
    int q, qd, f, g, qg, qdg, fg, table, link, scratch, acc, total_floats;
    __host__ __device__ AbaBwdSmem(int T, int n, int n_links) {
        const int TB = T < 32 ? 32 : T;
        int o = 0;
        q = o; o += T * n;
        qd = o; o += T * n;
        f = o; o += T * n;
        g = o; o += T * n;
        qg = g;                       // g_qdd_c is last read in R3 just before q-bar_c is first written
        qdg = o; o += T * n;
        fg = f;                       // f is last read in F2, f-bar is written in R2
        o = (o + 3) & ~3;
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o; o += (n_links - 1) * AL * T;
        scratch = o; o += 26 * (TB + 1);
        acc = o; o += n_links * DRMB200_TABLE_STRIDE;
        total_floats = o;
    }
};

// ---- small 3x3 helpers (local to this file) ------------------------------------------------------
__device__ __forceinline__ M3 madd(const M3& a, const M3& b) {
    M3 r;
    r.a00 = a.a00 + b.a00; r.a01 = a.a01 + b.a01; r.a02 = a.a02 + b.a02;
    r.a10 = a.a10 + b.a10; r.a11 = a.a11 + b.a11; r.a12 = a.a12 + b.a12;
    r.a20 = a.a20 + b.a20; r.a21 = a.a21 + b.a21; r.a22 = a.a22 + b.a22;
    return r;
}
__device__ __forceinline__ M3 msub(const M3& a, const M3& b) {
    M3 r;
    r.a00 = a.a00 - b.a00; r.a01 = a.a01 - b.a01; r.a02 = a.a02 - b.a02;
    r.a10 = a.a10 - b.a10; r.a11 = a.a11 - b.a11; r.a12 = a.a12 - b.a12;
    r.a20 = a.a20 - b.a20; r.a21 = a.a21 - b.a21; r.a22 = a.a22 - b.a22;
    return r;
}
__device__ __forceinline__ M3 skew_b(V3 a) {
    M3 r;
    r.a00 = 0.f;  r.a01 = -a.z; r.a02 = a.y;
    r.a10 = a.z;  r.a11 = 0.f;  r.a12 = -a.x;
    r.a20 = -a.y; r.a21 = a.x;  r.a22 = 0.f;
    return r;
}
__device__ __forceinline__ V3 unskew(const M3& s) { return v3(s.a21 - s.a12, s.a02 - s.a20, s.a10 - s.a01); }
__device__ __forceinline__ V3 rw0(const M3& m) { return v3(m.a00, m.a01, m.a02); }
__device__ __forceinline__ V3 rw1(const M3& m) { return v3(m.a10, m.a11, m.a12); }
__device__ __forceinline__ V3 rw2(const M3& m) { return v3(m.a20, m.a21, m.a22); }
__device__ __forceinline__ M3 cols3(V3 c0, V3 c1, V3 c2) {
    M3 r;
    r.a00 = c0.x; r.a10 = c0.y; r.a20 = c0.z; r.a01 = c1.x; r.a11 = c1.y; r.a21 = c1.z; r.a02 = c2.x; r.a12 = c2.y; r.a22 = c2.z;
    return r;
}
__device__ __forceinline__ M3 rows3(V3 r0, V3 r1, V3 r2) {
    M3 r;
    r.a00 = r0.x; r.a01 = r0.y; r.a02 = r0.z; r.a10 = r1.x; r.a11 = r1.y; r.a12 = r1.z; r.a20 = r2.x; r.a21 = r2.y; r.a22 = r2.z;
    return r;
}
__device__ __forceinline__ M3 lcross(V3 r, const M3& Y) { return cols3(cross(r, col0(Y)), cross(r, col1(Y)), cross(r, col2(Y))); }   // skew(r) Y
__device__ __forceinline__ M3 rcross(const M3& Y, V3 r) { return rows3(cross(rw0(Y), r), cross(rw1(Y), r), cross(rw2(Y), r)); }      // Y skew(r)
__device__ __forceinline__ void sub_outer_b(M3& m, V3 x, V3 y) {
    m.a00 = fmaf(-x.x, y.x, m.a00); m.a01 = fmaf(-x.x, y.y, m.a01); m.a02 = fmaf(-x.x, y.z, m.a02);
    m.a10 = fmaf(-x.y, y.x, m.a10); m.a11 = fmaf(-x.y, y.y, m.a11); m.a12 = fmaf(-x.y, y.z, m.a12);
    m.a20 = fmaf(-x.z, y.x, m.a20); m.a21 = fmaf(-x.z, y.y, m.a21); m.a22 = fmaf(-x.z, y.z, m.a22);
}
__device__ __forceinline__ M3 conj_b(const M3& M, const M3& Y) { return mulNT(mul(M, Y), M); }     // M Y M^T
__device__ __forceinline__ M3 conjT_b(const M3& M, const M3& Y) { return mul(mulTN(M, Y), M); }    // M^T Y M
__device__ __forceinline__ float quad(V3 x, const M3& Y, V3 y) { return dot(x, mul(Y, y)); }       // x^T Y y

// Sum of NV <= 32 per-thread values over the (single-warp) CTA into acc_row[0..NV): transposed through a padded
// scratch so that lane j adds up value j of all 32 threads -- 32 independent short chains instead of NV serial
// shuffle trees (the kernel runs at 2-3 warps per SM, latency is what it pays for).  Fixed order: deterministic.
template <int NV>
__device__ __forceinline__ void warp_accumulate(float* scratch, float* acc_row, const float (&vals)[NV], bool active) {
    static_assert(NV <= 32, "one lane per value");
    const int lane = threadIdx.x;
#pragma unroll
    for (int j = 0; j < NV; ++j) scratch[j * 33 + lane] = active ? vals[j] : 0.f;
    __syncwarp();
    if (lane < NV) {
        const float* row = scratch + lane * 33;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int c = 0; c < 32; c += 4) { s0 += row[c]; s1 += row[c + 1]; s2 += row[c + 2]; s3 += row[c + 3]; }
        acc_row[lane] += (s0 + s1) + (s2 + s3);
    }
    __syncwarp();
}

struct Blocks { M3 A, B, C, D; };
__device__ __forceinline__ Blocks ld_blocks(const float* p, int T) {
    Blocks b;
    b.A = ldm(p, T); b.B = ldm(p + 9 * T, T); b.C = ldm(p + 18 * T, T); b.D = ldm(p + 27 * T, T);
    return b;
}
__device__ __forceinline__ void st_blocks(float* p, int T, const Blocks& b) {
    stm(p, T, b.A); stm(p + 9 * T, T, b.B); stm(p + 18 * T, T, b.C); stm(p + 27 * T, T, b.D);
}

template <bool NEED_TABLE, int T>
__global__ void __launch_bounds__(T < 32 ? 32 : T)
aba_backward_kernel(const __grid_constant__ TreeProgram prog, const AbaBwdArgs args) {
    constexpr int TB = T < 32 ? 32 : T;
    static_assert(TB == 32, "warp_accumulate assumes a single-warp CTA");
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs, N = prog.n_links;
    const AbaBwdSmem L(T, n, N);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_f = smem + L.f;
    float* s_g = smem + L.g;
    float* s_qg = smem + L.qg;
    float* s_qdg = smem + L.qdg;
    float* s_fg = smem + L.fg;
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_scr = smem + L.scratch;
    float* s_acc = smem + L.acc;
    const int tid = threadIdx.x;
    const bool vec_ok = args.vec_ok;
    const float grav = (args.flags & DRMB200_GRAVITY) ? GRAVITY_B : 0.f;
    const bool damp = (args.flags & DRMB200_DAMPING) != 0;

    for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += TB) {
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
        coop_copy(s_f, args.f + start * n, valid * n, vec_ok);
        coop_copy(s_g, args.g_qdd + start * n, valid * n, vec_ok);
        for (int i = tid; i < T * n; i += TB) s_qdg[i] = 0.f;      // q-bar and f-bar tiles alias inputs and are assigned, not accumulated
        __syncthreads();

        const bool active = tid < valid;
        const int lane = tid < T ? tid : 0;             // threads beyond the tile (T = 16) shadow row 0, never active
        const float* qrow = s_q + lane * n;
        const float* qdrow = s_qd + lane * n;
        const float* frow = s_f + lane * n;
        const float* grow = s_g + lane * n;
        float* qg = s_qg + lane * n;
        float* qdg = s_qdg + lane * n;
        float* fg = s_fg + lane * n;
        float* lk0 = s_link + lane - AL * T;            // link i lives at lk0 + i * AL * T   (i >= 1)
        float* gia0 = args.scratch + ((int64_t)blockIdx.x * (N - 1) - 1) * IA_FLOATS * T + lane;     // IA of link i at gia0 + i * 36 * T
        const V3 zero = v3(0.f, 0.f, 0.f);
        const bool writer = tid < T;                    // shadows must not store

        // ================= F1: velocities, bias forces, rigid-body inertias =====================
        for (int i = 1; i < N; ++i) {
            const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
            float* lk = lk0 + i * AL * T;
            const int P = prog.parent[i];
            V3 wp = zero, vp = zero;
            if (P > 0) { const float* pk = lk0 + P * AL * T; wp = ldv(pk + O_W * T, T); vp = ldv(pk + (O_W + 3) * T, T); }
            M3 M = C.F;
            const int c = prog.dof[i];
            float cs = 1.f, sn = 0.f, qd_k = 0.f;
            if (c >= 0) { qd_k = qdrow[c]; sincos_pi2(qrow[c], sn, cs); rotate_z(M, cs, sn); }
            V3 w = mulT(M, wp); w.z += qd_k;
            const V3 v = mulT(M, cross_add(wp, C.r, vp));
            const V3 hl = C.m * v - cross(C.mc, w);
            const V3 ha = mul_add(C.Io, w, cross(C.mc, v));
            if (writer) {
                lk[O_CS * T] = cs; lk[(O_CS + 1) * T] = sn;
                stv(lk + O_W * T, T, w); stv(lk + (O_W + 3) * T, T, v);
                stv(lk + O_PA * T, T, cross_add(w, ha, cross(v, hl))); stv(lk + (O_PA + 3) * T, T, cross(w, hl));
                Blocks I;
                I.A = C.Io; I.B = skew_b(C.mc); I.C = transpose(I.B);
                I.D = zero3(); I.D.a00 = I.D.a11 = I.D.a22 = C.m;
                st_blocks(gia0 + i * IA_FLOATS * T, T, I);
                stv(lk + O_ADJ * T, T, zero); stv(lk + (O_ADJ + 3) * T, T, zero);
                stv(lk + O_AL * T, T, zero); stv(lk + (O_AL + 3) * T, T, zero);
                lk[O_DB * T] = 0.f; lk[O_UB * T] = 0.f; lk[O_U * T] = 0.f;
            }
        }

        // ================= F2: articulated inertias, parents accumulate in place =================
        for (int i = N - 1; i >= 1; --i) {
            const int P = prog.parent[i];
            const int c = prog.dof[i];
            float* lk = lk0 + i * AL * T;
            Blocks I = ld_blocks(gia0 + i * IA_FLOATS * T, T);
            V3 pa_ang = ldv(lk + O_PA * T, T), pa_lin = ldv(lk + (O_PA + 3) * T, T);
            V3 Ua = zero, Ul = zero;
            float d = 0.f, u = 0.f;
            if (c >= 0) {
                Ua = col2(I.A); Ul = col2(I.C); d = Ua.z;
                float fk = frow[c];
                if (damp) fk = fmaf(-s_tab[i * DRMB200_TABLE_STRIDE + 25], qdrow[c], fk);
                u = fk - pa_ang.z;
                if (writer) lk[O_U * T] = u;
            }
            if (P > 0) {
                M3 M; V3 r;
                load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
                if (c >= 0) {
                    const float inv = 1.f / (d + ABA_EPS_B);
                    const V3 Uda = inv * Ua, Udl = inv * Ul;
                    sub_outer_b(I.A, Ua, Uda); sub_outer_b(I.B, Ua, Udl); sub_outer_b(I.C, Ul, Uda); sub_outer_b(I.D, Ul, Udl);
                    const V3 w = ldv(lk + O_W * T, T), v = ldv(lk + (O_W + 3) * T, T);
                    const float qd_k = qdrow[c];
                    const V3 ca = cross_z(w, qd_k), cl = cross_z(v, qd_k);
                    const float ud = u * inv;
                    pa_ang = pa_ang + mul(I.A, ca) + mul(I.B, cl) + ud * Ua;
                    pa_lin = pa_lin + mul(I.C, ca) + mul(I.D, cl) + ud * Ul;
                    rotate_z(M, lk[O_CS * T], lk[(O_CS + 1) * T]);
                }
                Blocks Y;
                const M3 Bh = conj_b(M, I.B);
                Y.D = conj_b(M, I.D);
                Y.B = madd(Bh, lcross(r, Y.D));
                Y.C = msub(conj_b(M, I.C), rcross(Y.D, r));
                Y.A = msub(madd(conj_b(M, I.A), lcross(r, Y.C)), rcross(Bh, r));
                const V3 q_lin = mul(M, pa_lin);
                const V3 q_ang = cross_add(r, q_lin, mul(M, pa_ang));
                if (writer) {
                    float* pk = lk0 + P * AL * T;
                    const Blocks Pk = ld_blocks(gia0 + P * IA_FLOATS * T, T);
                    Y.A = madd(Y.A, Pk.A); Y.B = madd(Y.B, Pk.B); Y.C = madd(Y.C, Pk.C); Y.D = madd(Y.D, Pk.D);
                    st_blocks(gia0 + P * IA_FLOATS * T, T, Y);
                    stv(pk + O_PA * T, T, ldv(pk + O_PA * T, T) + q_ang);
                    stv(pk + (O_PA + 3) * T, T, ldv(pk + (O_PA + 3) * T, T) + q_lin);
                }
            }
        }

        // ================= F3: accelerations ======================================================
        for (int i = 1; i < N; ++i) {
            const int P = prog.parent[i];
            const int c = prog.dof[i];
            float* lk = lk0 + i * AL * T;
            M3 M; V3 r;
            load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
            V3 alp = zero, ap = v3(0.f, 0.f, grav);
            if (P > 0) { const float* pk = lk0 + P * AL * T; alp = ldv(pk + O_AL * T, T); ap = ldv(pk + (O_AL + 3) * T, T); }
            if (c >= 0) rotate_z(M, lk[O_CS * T], lk[(O_CS + 1) * T]);
            V3 al = mulT(M, alp);
            V3 a = mulT(M, cross_add(alp, r, ap));
            if (c >= 0) {
                const float qd_k = qdrow[c];
                const V3 w = ldv(lk + O_W * T, T), v = ldv(lk + (O_W + 3) * T, T);
                al = al + cross_z(w, qd_k); a = a + cross_z(v, qd_k);
                const V3 Ua = v3(gia0[(i * IA_FLOATS + 2) * T], gia0[(i * IA_FLOATS + 5) * T], gia0[(i * IA_FLOATS + 8) * T]);
                const V3 Ul = v3(gia0[(i * IA_FLOATS + 20) * T], gia0[(i * IA_FLOATS + 23) * T], gia0[(i * IA_FLOATS + 26) * T]);
                const float qdd = (1.0f / Ua.z) * (lk[O_U * T] - (dot(Ua, al) + dot(Ul, a)));
                al.z += qdd;
            }
            if (writer) { stv(lk + O_AL * T, T, al); stv(lk + (O_AL + 3) * T, T, a); }
        }

        // ================= R3: reverse of the acceleration pass ==================================
        for (int i = N - 1; i >= 1; --i) {
            const int P = prog.parent[i];
            const int c = prog.dof[i];
            float* lk = lk0 + i * AL * T;
            M3 M; V3 r;
            load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
            const float cs = lk[O_CS * T], sn = lk[(O_CS + 1) * T];
            V3 alp = zero, ap = v3(0.f, 0.f, grav);
            if (P > 0) { const float* pk = lk0 + P * AL * T; alp = ldv(pk + O_AL * T, T); ap = ldv(pk + (O_AL + 3) * T, T); }
            V3 alq_b = ldv(lk + O_ADJ * T, T), aq_b = ldv(lk + (O_ADJ + 3) * T, T);
            if (c >= 0) {
                rotate_z(M, cs, sn);
                const float qd_k = qdrow[c];
                const V3 w = ldv(lk + O_W * T, T), v = ldv(lk + (O_W + 3) * T, T);
                const V3 alq = mulT(M, alp) + cross_z(w, qd_k);
                const V3 aq = mulT(M, cross_add(alp, r, ap)) + cross_z(v, qd_k);
                const V3 Ua = v3(gia0[(i * IA_FLOATS + 2) * T], gia0[(i * IA_FLOATS + 5) * T], gia0[(i * IA_FLOATS + 8) * T]);
                const V3 Ul = v3(gia0[(i * IA_FLOATS + 20) * T], gia0[(i * IA_FLOATS + 23) * T], gia0[(i * IA_FLOATS + 26) * T]);
                const float dinv = 1.0f / Ua.z;
                const float qdd = dinv * (lk[O_U * T] - (dot(Ua, alq) + dot(Ul, aq)));
                const float k = (grow[c] + alq_b.z) * dinv;
                if (writer) {
                    lk[O_UB * T] = k;
                    lk[O_DB * T] = -k * qdd;
                    stv(lk + O_AL * T, T, (-k) * alq); stv(lk + (O_AL + 3) * T, T, (-k) * aq);      // U-bar (al, a of link i are dead)
                }
                alq_b = alq_b - k * Ua;
                aq_b = aq_b - k * Ul;
            }
            if (writer) {
                lk[O_CB * T] = alq_b.x; lk[(O_CB + 1) * T] = alq_b.y; lk[(O_CB + 2) * T] = aq_b.x; lk[(O_CB + 3) * T] = aq_b.y;
                stv(lk + O_ADJ * T, T, zero); stv(lk + (O_ADJ + 3) * T, T, zero);                    // reused by R1
            }
            const V3 ua = mul(M, aq_b);
            if (P > 0 && writer) {
                float* pk = lk0 + P * AL * T;
                stv(pk + O_ADJ * T, T, ldv(pk + O_ADJ * T, T) + cross_add(r, ua, mul(M, alq_b)));
                stv(pk + (O_ADJ + 3) * T, T, ldv(pk + (O_ADJ + 3) * T, T) + ua);
            }
            M3 Mbar = zero3();
            add_outer(Mbar, cross_add(alp, r, ap), aq_b);
            add_outer(Mbar, alp, alq_b);
            if (c >= 0 && writer) qg[c] = theta_grad_z(Mbar, M);     // first touch of q-bar_c (its tile aliases g_qdd, read above)
            if (NEED_TABLE) {
                float vals[12];
                if (c >= 0) rotate_z(Mbar, cs, -sn);
                m3_to_array(Mbar, vals);
                const V3 rbar = cross(ua, alp);
                vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z;
                warp_accumulate<12>(s_scr, s_acc + i * DRMB200_TABLE_STRIDE, vals, active);
            }
        }

        // ================= R2: reverse of the articulated-inertia pass ===========================
        for (int i = 1; i < N; ++i) {
            const int P = prog.parent[i];
            const int c = prog.dof[i];
            float* lk = lk0 + i * AL * T;
            const float cs = lk[O_CS * T], sn = lk[(O_CS + 1) * T];
            Blocks Ib;                                    // IA-bar_i
            Ib.A = Ib.B = Ib.C = Ib.D = zero3();
            V3 pb_ang = zero, pb_lin = zero;              // pA-bar_i
            V3 Uab = zero, Ulb = zero;
            float db = 0.f, ub = 0.f;
            V3 Ua = zero, Ul = zero;
            if (c >= 0) {
                Ua = v3(gia0[(i * IA_FLOATS + 2) * T], gia0[(i * IA_FLOATS + 5) * T], gia0[(i * IA_FLOATS + 8) * T]);
                Ul = v3(gia0[(i * IA_FLOATS + 20) * T], gia0[(i * IA_FLOATS + 23) * T], gia0[(i * IA_FLOATS + 26) * T]);
                Uab = ldv(lk + O_AL * T, T); Ulb = ldv(lk + (O_AL + 3) * T, T);
                db = lk[O_DB * T]; ub = lk[O_UB * T];
            }
            float vals[26];
#pragma unroll
            for (int j = 0; j < 26; ++j) vals[j] = 0.f;
            if (P > 0) {
                M3 M; V3 r;
                load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
                if (c >= 0) rotate_z(M, cs, sn);
                const float* pk = lk0 + P * AL * T;
                const Blocks Y = ld_blocks(gia0 + P * IA_FLOATS * T, T);                     // IA-bar of the parent
                const V3 Qa_b = ldv(pk + O_PA * T, T), Ql_b = ldv(pk + (O_PA + 3) * T, T);
                // recompute IA', pa of this link
                Blocks I = ld_blocks(gia0 + i * IA_FLOATS * T, T);
                V3 pa_ang = ldv(lk + O_PA * T, T), pa_lin = ldv(lk + (O_PA + 3) * T, T);
                float inv = 0.f, u = 0.f;
                V3 ca = zero, cl = zero;
                if (c >= 0) {
                    inv = 1.f / (Ua.z + ABA_EPS_B);
                    u = lk[O_U * T];
                    const V3 Uda = inv * Ua, Udl = inv * Ul;
                    sub_outer_b(I.A, Ua, Uda); sub_outer_b(I.B, Ua, Udl); sub_outer_b(I.C, Ul, Uda); sub_outer_b(I.D, Ul, Udl);
                    const float qd_k = qdrow[c];
                    ca = cross_z(ldv(lk + O_W * T, T), qd_k); cl = cross_z(ldv(lk + (O_W + 3) * T, T), qd_k);
                    const float ud = u * inv;
                    pa_ang = pa_ang + mul(I.A, ca) + mul(I.B, cl) + ud * Ua;
                    pa_lin = pa_lin + mul(I.C, ca) + mul(I.D, cl) + ud * Ul;
                }
                // force transform
                const V3 t = Ql_b + cross(Qa_b, r);
                const V3 pal_b = mulT(M, t), paa_b = mulT(M, Qa_b);
                V3 rbar = cross(mul(M, pa_lin), Qa_b);
                M3 Mbar = zero3();
                add_outer(Mbar, t, pa_lin);
                add_outer(Mbar, Qa_b, pa_ang);
                // congruence: hatted blocks and their adjoints
                const M3 Ah = conj_b(M, I.A), Bh = conj_b(M, I.B), Ch = conj_b(M, I.C), Dh = conj_b(M, I.D);
                const M3 YAS = rcross(Y.A, r);                                    // YA S
                const M3 Ah_b = Y.A;
                const M3 Bh_b = madd(Y.B, YAS);
                const M3 Ch_b = msub(Y.C, lcross(r, Y.A));
                const M3 Dh_b = msub(madd(msub(Y.D, lcross(r, Y.B)), rcross(Y.C, r)), lcross(r, YAS));
                {
                    const M3 DhT = transpose(Dh);
                    M3 Sb = mul(Y.B, DhT);
                    Sb = msub(Sb, mul(DhT, Y.C));
                    Sb = madd(Sb, mulNT(Y.A, Ch));
                    Sb = msub(Sb, mulTN(Bh, Y.A));
                    Sb = madd(Sb, mul(YAS, DhT));
                    Sb = madd(Sb, mul(DhT, lcross(r, Y.A)));
                    rbar = rbar + unskew(Sb);
                }
                {
                    M3 G = madd(mulNT(Ah_b, Ah), mulTN(Ah_b, Ah));
                    G = madd(G, madd(mulNT(Bh_b, Bh), mulTN(Bh_b, Bh)));
                    G = madd(G, madd(mulNT(Ch_b, Ch), mulTN(Ch_b, Ch)));
                    G = madd(G, madd(mulNT(Dh_b, Dh), mulTN(Dh_b, Dh)));
                    Mbar = madd(Mbar, mul(G, M));
                }
                Ib.A = conjT_b(M, Ah_b); Ib.B = conjT_b(M, Bh_b); Ib.C = conjT_b(M, Ch_b); Ib.D = conjT_b(M, Dh_b);
                pb_ang = paa_b; pb_lin = pal_b;
                if (c >= 0) {
                    add_outer(Ib.A, paa_b, ca); add_outer(Ib.B, paa_b, cl); add_outer(Ib.C, pal_b, ca); add_outer(Ib.D, pal_b, cl);
                    const V3 cab = mulT(I.A, paa_b) + mulT(I.C, pal_b);
                    const V3 clb = mulT(I.B, paa_b) + mulT(I.D, pal_b);
                    if (writer) {
                        lk[O_CB * T] += cab.x; lk[(O_CB + 1) * T] += cab.y; lk[(O_CB + 2) * T] += clb.x; lk[(O_CB + 3) * T] += clb.y;
                    }
                    const float sig = dot(Ua, paa_b) + dot(Ul, pal_b);
                    Uab = Uab + (u * inv) * paa_b;
                    Ulb = Ulb + (u * inv) * pal_b;
                    ub = fmaf(sig, inv, ub);
                    float inv_b = sig * u;
                    Uab = Uab - inv * (mul(Ib.A, Ua) + mulT(Ib.A, Ua) + mul(Ib.B, Ul) + mulT(Ib.C, Ul));
                    Ulb = Ulb - inv * (mulT(Ib.B, Ua) + mul(Ib.C, Ua) + mul(Ib.D, Ul) + mulT(Ib.D, Ul));
                    inv_b -= quad(Ua, Ib.A, Ua) + quad(Ua, Ib.B, Ul) + quad(Ul, Ib.C, Ua) + quad(Ul, Ib.D, Ul);
                    db = fmaf(-inv_b * inv, inv, db);
                }
                if (c >= 0 && writer) qg[c] += theta_grad_z(Mbar, M);
                if (NEED_TABLE) {
                    if (c >= 0) rotate_z(Mbar, cs, -sn);
                    m3_to_array(Mbar, vals);
                    vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z;
                }
            }
            if (c >= 0) {
                if (writer) fg[c] = ub;
                if (damp) {
                    if (writer) qdg[c] = fmaf(-s_tab[i * DRMB200_TABLE_STRIDE + 25], ub, qdg[c]);
                    vals[25] = -ub * qdrow[c];
                }
                pb_ang.z -= ub;
                Uab.z += db;
                Ib.A.a02 += Uab.x; Ib.A.a12 += Uab.y; Ib.A.a22 += Uab.z;           // Ua = A e_z, Ul = C e_z
                Ib.C.a02 += Ulb.x; Ib.C.a12 += Ulb.y; Ib.C.a22 += Ulb.z;
            }
            if (writer) {
                st_blocks(gia0 + i * IA_FLOATS * T, T, Ib);                                    // IA_i is dead: keep IA-bar_i for the children
                stv(lk + O_PA * T, T, pb_ang); stv(lk + (O_PA + 3) * T, T, pb_lin);
            }
            if (NEED_TABLE) {
                m3_to_array(Ib.A, vals + 12);                                       // Io-bar
                const V3 mcb = unskew(madd(Ib.B, transpose(Ib.C)));                 // B = mc^, C = (mc^)^T
                vals[21] = mcb.x; vals[22] = mcb.y; vals[23] = mcb.z;
                vals[24] = Ib.D.a00 + Ib.D.a11 + Ib.D.a22;
                warp_accumulate<26>(s_scr, s_acc + i * DRMB200_TABLE_STRIDE, vals, active);
            }
        }

        // ================= R1: reverse of the velocity / bias pass ================================
        for (int i = N - 1; i >= 1; --i) {
            const int P = prog.parent[i];
            const int c = prog.dof[i];
            float* lk = lk0 + i * AL * T;
            const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
            const float cs = lk[O_CS * T], sn = lk[(O_CS + 1) * T];
            M3 M = C.F;
            float qd_k = 0.f;
            if (c >= 0) { rotate_z(M, cs, sn); qd_k = qdrow[c]; }
            const V3 w = ldv(lk + O_W * T, T), v = ldv(lk + (O_W + 3) * T, T);
            V3 wp = zero, vp = zero;
            if (P > 0) { const float* pk = lk0 + P * AL * T; wp = ldv(pk + O_W * T, T); vp = ldv(pk + (O_W + 3) * T, T); }
            V3 wb = ldv(lk + O_ADJ * T, T), vb = ldv(lk + (O_ADJ + 3) * T, T);
            const V3 pi = ldv(lk + O_PA * T, T), rho = ldv(lk + (O_PA + 3) * T, T);
            const V3 hl = C.m * v - cross(C.mc, w);
            const V3 ha = mul_add(C.Io, w, cross(C.mc, v));
            const V3 hab = cross(pi, w);
            const V3 hlb = cross_add(pi, v, cross(rho, w));
            wb = wb + cross_add(ha, pi, cross(hl, rho)) + cross_add(C.mc, hlb, mulT(C.Io, hab));
            vb = vb + cross_add(hl, pi, cross_add(hab, C.mc, C.m * hlb));
            float wJb = 0.f;
            if (c >= 0) {
                const V3 cab = v3(lk[O_CB * T], lk[(O_CB + 1) * T], 0.f), clb = v3(lk[(O_CB + 2) * T], lk[(O_CB + 3) * T], 0.f);
                wb = wb + z_cross(qd_k, cab);
                vb = vb + z_cross(qd_k, clb);
                wJb = (cab.x * w.y - cab.y * w.x) + (clb.x * v.y - clb.y * v.x) + wb.z;
                if (writer) qdg[c] += wJb;
            }
            const V3 uv = mul(M, vb);
            if (P > 0 && writer) {
                float* pk = lk0 + P * AL * T;
                stv(pk + O_ADJ * T, T, ldv(pk + O_ADJ * T, T) + cross_add(C.r, uv, mul(M, wb)));
                stv(pk + (O_ADJ + 3) * T, T, ldv(pk + (O_ADJ + 3) * T, T) + uv);
            }
            M3 Mbar = zero3();
            add_outer(Mbar, cross_add(wp, C.r, vp), vb);
            add_outer(Mbar, wp, wb);
            if (c >= 0 && writer) qg[c] += theta_grad_z(Mbar, M);
            if (NEED_TABLE) {
                float vals[25];
                if (c >= 0) rotate_z(Mbar, cs, -sn);
                m3_to_array(Mbar, vals);
                const V3 rbar = cross(uv, wp);
                vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z;
                M3 Iob = zero3();
                add_outer(Iob, hab, w);
                m3_to_array(Iob, vals + 12);
                const V3 mcb = cross_add(hlb, w, cross(v, hab));
                vals[21] = mcb.x; vals[22] = mcb.y; vals[23] = mcb.z;
                vals[24] = dot(hlb, v);
                warp_accumulate<25>(s_scr, s_acc + i * DRMB200_TABLE_STRIDE, vals, active);
            }
        }

        __syncthreads();
        if (args.q_grad != nullptr) coop_copy(args.q_grad + start * n, s_qg, valid * n, vec_ok);
        if (args.qd_grad != nullptr) coop_copy(args.qd_grad + start * n, s_qdg, valid * n, vec_ok);
        if (args.f_grad != nullptr) coop_copy(args.f_grad + start * n, s_fg, valid * n, vec_ok);
    }
    if (NEED_TABLE) {
        __syncthreads();
        float* out = args.partials + (size_t)blockIdx.x * N * DRMB200_TABLE_STRIDE;
        for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += TB) {       // canonical -> natural (bijection per row)
            const int l = i / DRMB200_TABLE_STRIDE, e = i - l * DRMB200_TABLE_STRIDE;
            const int p = prog.parent[l];
            int src;
            const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
            out[l * DRMB200_TABLE_STRIDE + src] = sg * s_acc[i];
        }
    }
}

// workspace = per-CTA partial tables (as for the other backward kernels) + the per-CTA articulated-inertia scratch
int64_t forward_dynamics_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    if (topo == nullptr || topo->n_links < 1 || topo->n_links > DRMB200_MAX_LINKS) return 0;
    int64_t tiles = (batch + 15) / 16;
    if (tiles < 1) tiles = 1;
    const int64_t grid = tiles < BWD_MAX_GRID ? tiles : BWD_MAX_GRID;
    return table_grad_workspace_bytes(topo, batch) + grid * (topo->n_links - 1) * IA_FLOATS * 32 * (int64_t)sizeof(float);
}

int forward_dynamics_backward_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                     const float* f, int64_t batch, uint32_t flags, const float* g_qdd,
                                     float* q_grad, float* qd_grad, float* f_grad, float* table_grad, void* workspace,
                                     cudaStream_t stream) {
    TreeProgram prog;
    int rc = build_tree_program(topo, &prog);
    if (rc != DRMB200_OK) return rc;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (q_grad == nullptr && qd_grad == nullptr && f_grad == nullptr && table_grad == nullptr) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || f == nullptr || g_qdd == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    if (workspace == nullptr) { set_error("forward-dynamics backward needs its workspace (drmb200_forward_dynamics_backward_workspace_bytes)"); return DRMB200_EINVAL; }

    AbaBwdArgs args;
    args.table = table; args.q = q; args.qd = qd; args.f = f; args.g_qdd = g_qdd;
    args.q_grad = q_grad; args.qd_grad = qd_grad; args.f_grad = f_grad;
    args.partials = static_cast<float*>(workspace);
    args.scratch = reinterpret_cast<float*>(static_cast<char*>(workspace) + table_grad_workspace_bytes(topo, batch));
    args.batch = batch; args.flags = flags;
    auto al16 = [](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    args.vec_ok = (al16(q) && al16(qd) && al16(f) && al16(g_qdd) && al16(q_grad) && al16(qd_grad) && al16(f_grad)) ? 1 : 0;

    auto bytes_of = [&](int t) { return (size_t)AbaBwdSmem(t, prog.n_dofs, prog.n_links).total_floats * sizeof(float); };
    const int tile = bytes_of(32) <= 200 * 1024 ? 32 : 16;
    const size_t smem_bytes = bytes_of(tile);
    if (smem_bytes > 227 * 1024) { set_error("forward-dynamics backward needs %zu B of shared memory per CTA (> 227 KB): model too large", smem_bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (batch + tile - 1) / tile;
    int grid = 0;
    const bool need_table = table_grad != nullptr;
#define DRM_LAUNCH_ABAB(NT, TT)                                                                                   \
    do {                                                                                                          \
        rc = persistent_grid(aba_backward_kernel<NT, TT>, TT < 32 ? 32 : TT, smem_bytes, tiles, &grid, "aba backward"); \
        if (rc != DRMB200_OK) return rc;                                                                          \
        aba_backward_kernel<NT, TT><<<grid, TT < 32 ? 32 : TT, smem_bytes, stream>>>(prog, args);                 \
    } while (0)
    if (need_table) { if (tile == 32) DRM_LAUNCH_ABAB(true, 32); else DRM_LAUNCH_ABAB(true, 16); }
    else            { if (tile == 32) DRM_LAUNCH_ABAB(false, 32); else DRM_LAUNCH_ABAB(false, 16); }
#undef DRM_LAUNCH_ABAB
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("aba backward launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return need_table ? launch_reduce(args.partials, grid, topo, table_grad, stream) : DRMB200_OK;
}

}  // namespace drm
