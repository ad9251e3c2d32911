// contact_backward.cu -- the adjoint of the contact dynamics and of the contact impulse (sm_90a).
//
// With J, G, A = J G J^T + mu I as in contact_dynamics.cu and the forward's outputs (qdd or qd_plus, lambda, solved), the
// upstream gradients g_qdd [n] and g_lambda [M] (NULL: zero) give, per row (the derivation is in include/drm_b200.h):
//   s = g_lambda + J G^T g_qdd;   A^T nu = s;   g^ = g_qdd - J^T nu;   accel_ref_grad = nu
//   (q1, qd1, theta1, tau^) = forward-dynamics adjoint at (q, qd, tau_c = f + J^T lambda) with upstream g^;  f_grad = tau^
//   phi(q, qd; theta) = lambda^T J tau^ - nu^T (J qdd + Jdot qd), lambda, nu, tau^, qdd held constant
//   q_grad = q1 + dphi/dq,  qd_grad = qd1 + dphi/dqd,  table_grad += theta1 + dphi/dtheta
// The impulse: qdd -> qd_plus, lambda -> Lambda, the adjoint at (q, 0, J^T Lambda) without flags, phi without the Jdot qd
// term (a walk at zero velocity), qd_grad = g^ and velocity_ref_grad = nu.
//
// Three stages in stream order, no allocation and no synchronisation:
//   1. contact_backward_kernel<T, IMPULSE>: one thread per row with the forward's slot-major row state.  It recomputes the
//      walk, the ABA's articulated inertias and A with the forward's device code (osd_inverse_inertia with the g_qdd dot
//      products beside its sweeps), factors S A S with contact_factor -- the forward's float operations, so its pivots and
//      solved decision are the forward's bit for bit -- and solves the transposed system.  Outputs (nu, g^, tau_c) leave
//      through store_transposed, with copies of q and qd that are zero on the rows it finds unsolved; those rows get
//      nu = g^ = tau_c = 0, so they contribute exactly zero to every gradient, even when their inputs are not finite.
//   2. the forward-dynamics adjoint (backward_aba.cu) at (q, qd, tau_c) with upstream g^.
//   3. contact_kinematic_backward_kernel<T, IMPULSE>: dphi/dq, dphi/dqd and dphi/d(F, r) in one forward walk of the union of
//      the contact links' paths (osd_walk's MultiProgram order) that keeps every step's parent state, then one reverse sweep.
//      It adds into q_grad / qd_grad and writes per-CTA partial table gradients in the canonical +z frames, mapped back to
//      table columns through canon_map and reduced in fixed order by reduce_partials_kernel: bitwise reproducible.
#include <cmath>
#include "backward_common.cuh"
#include "contact_common.cuh"

namespace drm {

int contact_programs(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, float regularization,
                     int64_t batch, UnionProgram* P, const TreeProgram** prog);      // contact_dynamics.cu
int forward_dynamics_backward_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*,
                                     int64_t, uint32_t, const float*, float*, float*, float*, float*, void*, cudaStream_t);
int64_t forward_dynamics_backward_workspace_bytes(const drmb200_topology_t*, int64_t);

// =============================================================================================
// stage 1: nu, g^ and tau_c
// =============================================================================================
struct ContactBwdArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ f;         // [B, n]; null for the impulse
    const float* __restrict__ lam;       // [B, M] the forward's force / impulse
    const float* __restrict__ g_out;     // [B, n] upstream of qdd / qd_plus, or null (0)
    const float* __restrict__ g_lam;     // [B, M] upstream of force / impulse, or null (0)
    const uint8_t* __restrict__ solved;  // [B] the forward's decision
    float* __restrict__ nu;              // [B, M]
    float* __restrict__ ghat;            // [B, n]
    float* __restrict__ tauc;            // [B, n]
    float* __restrict__ q_safe;          // [B, n] q, zero on unsolved rows: where the forward-dynamics adjoint runs
    float* __restrict__ qd_safe;         // [B, n] qd (the impulse: 0), zero on unsolved rows
    uint8_t* __restrict__ ok;            // [B] this stage's solved decision
    int64_t batch;
    uint32_t flags;
    int32_t M;
    float mu;
    int32_t aligned;
};

struct ContactBwdSmemLayout {
    AbaSmemLayout aba;
    int lam, g, glam, jac, jscr, state, vel, bias, sdot, scale, piv, a, nu, ghat, tauc, okf, total_floats;
    __host__ __device__ ContactBwdSmemLayout(int T, const TreeProgram& tp, const UnionProgram& P, int M)
        : aba(T, tp.n_dofs, tp.n_links, tp.n_slots) {
        const int n = tp.n_dofs;
        int o = (aba.total_floats + 3) & ~3;   // row-major tiles staged with float4 copies
        lam = o;   o += ((M * T + 3) & ~3);
        g = o;     o += ((n * T + 3) & ~3);
        glam = o;  o += M * T;
        jac = o;   o += M * P.n_u * T;
        jscr = o;  o += 6 * P.walk.n_jslots * T;
        state = o; o += OSD_STATE * P.walk.n_state_slots * T;
        vel = o;   o += M * T;
        bias = o;  o += M * T;
        sdot = o;  o += M * T;
        scale = o; o += M * T;
        piv = o;   o += M * T;
        a = o;     o += M * M * T;
        nu = o;    o += M * T;
        ghat = o;  o += n * T;
        tauc = o;  o += n * T;
        okf = o;   o += T;
        total_floats = o;
    }
};

template <int T, bool IMPULSE>
__global__ void __launch_bounds__(T)
contact_backward_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ UnionProgram P, const ContactBwdArgs args) {
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs;
    const int M = args.M;
    const int MR = M / P.walk.n_ee;
    const int n_u = P.n_u;
    const ContactBwdSmemLayout L(T, prog, P, M);
    float* s_q = smem + L.aba.q;
    float* s_qd = smem + L.aba.qd;
    float* s_f = smem + L.aba.f;
    float* s_qdd = smem + L.aba.qdd;
    float* s_tab = smem + L.aba.table;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, args.batch - tile_start);
    const bool vec_ok = args.aligned;

    coop_copy(s_q, args.q + tile_start * n, valid * n, vec_ok);
    coop_copy(s_qd, args.qd + tile_start * n, valid * n, vec_ok);
    if (!IMPULSE) coop_copy(s_f, args.f + tile_start * n, valid * n, vec_ok);
    else for (int i = tid; i < T * n; i += T) s_f[i] = 0.f;
    coop_copy(smem + L.lam, args.lam + tile_start * M, valid * M, vec_ok);
    if (args.g_out != nullptr) coop_copy(smem + L.g, args.g_out + tile_start * n, valid * n, vec_ok);
    else for (int i = tid; i < T * n; i += T) smem[L.g + i] = 0.f;
    if (args.g_lam != nullptr) coop_copy(smem + L.glam, args.g_lam + tile_start * M, valid * M, vec_ok);
    else for (int i = tid; i < T * M; i += T) smem[L.glam + i] = 0.f;
    stage_canonical_table(s_tab, args.table, prog, T);
    // J, velocity and bias start at zero: columns off a link's path
    for (int i = L.jac + tid; i < L.jscr; i += T) smem[i] = 0.f;
    for (int i = L.vel + tid; i < L.sdot; i += T) smem[i] = 0.f;
    __syncthreads();

    if (tid < valid) {
        const float* qrow = s_q + tid * n;
        const float* qdrow = s_qd + tid * n;
        float* frow = s_f + tid * n;
        float* xrow = s_qdd + tid * n;
        const float* lrow = smem + L.lam + tid * M;
        const float* grow = smem + L.g + tid * n;
        const float* glrow = smem + L.glam + tid * M;
        float* lk0 = smem + L.aba.link + tid;
        float* sl0 = smem + L.aba.slots + tid;
        float* J = smem + L.jac + tid;
        float* A = smem + L.a + tid;
        float* sdot = smem + L.sdot + tid;
        float* nu = smem + L.nu + tid;
        float* ghat = smem + L.ghat + tid;
        float* tauc = smem + L.tauc + tid;
        const int rs = n_u * T;
        osd_walk<T>(P, s_tab, qrow, qdrow, MR, J, smem + L.vel + tid, smem + L.bias + tid, smem + L.jscr + tid,
                    smem + L.state + tid);
        for (int c = 0; c < n; ++c) tauc[c * T] = IMPULSE ? 0.f : frow[c];
        // the forward's steps 2-4 on A: the same device code in the same order
        if (!IMPULSE) aba_body<T>(prog, s_tab, qrow, qdrow, frow, xrow, lk0, sl0, args.flags);
        else aba_body<T>(prog, s_tab, qrow, frow, frow, xrow, lk0, sl0, 0u);
        osd_inverse_inertia<T, true>(prog, P, s_tab, M, J, A, frow, xrow, lk0, sl0, grow, sdot);
        for (int k = 0; k < M; ++k) A[(k * M + k) * T] += args.mu;
        // the factorisation repeats the forward's, so its decision is the forward's; a row the forward left unsolved never
        // contributes, whatever the factorisation finds
        const bool ok = contact_factor<T>(A, smem + L.scale + tid, smem + L.piv + tid, M) && args.solved[tile_start + tid] != 0;
        if (ok) {
            for (int m = 0; m < M; ++m) nu[m * T] = glrow[m] + sdot[m * T];            // s = g_lambda + J G^T g
            contact_solve_transposed<T>(A, nu, smem + L.scale + tid, smem + L.piv + tid, M);
            for (int c = 0; c < n; ++c) ghat[c * T] = grow[c];
            for (int u = 0; u < n_u; ++u) {
                float jl = 0.f, jn = 0.f;
                for (int m = 0; m < M; ++m) {
                    jl = fmaf(J[m * rs + u * T], lrow[m], jl);
                    jn = fmaf(J[m * rs + u * T], nu[m * T], jn);
                }
                const int c = P.u_dof[u];
                tauc[c * T] += jl;
                ghat[c * T] -= jn;
            }
        } else {
            for (int m = 0; m < M; ++m) nu[m * T] = 0.f;
            for (int c = 0; c < n; ++c) { ghat[c * T] = 0.f; tauc[c * T] = 0.f; }
        }
        args.ok[tile_start + tid] = ok ? 1 : 0;
        smem[L.okf + tid] = ok ? 1.f : 0.f;
    }
    __syncthreads();
    store_transposed(args.nu + tile_start * M, smem + L.nu, M, valid, T);
    store_transposed(args.ghat + tile_start * n, smem + L.ghat, n, valid, T);
    store_transposed(args.tauc + tile_start * n, smem + L.tauc, n, valid, T);
    // the state the forward-dynamics adjoint runs at: an unsolved row (its q may not even be finite) at the zero state, so
    // that with g^ = 0 and tau_c = 0 it adds exactly zero to every gradient
    for (int i = tid; i < valid * n; i += T) {
        const bool row_ok = smem[L.okf + i / n] != 0.f;
        args.q_safe[tile_start * n + i] = row_ok ? s_q[i] : 0.f;
        args.qd_safe[tile_start * n + i] = (row_ok && !IMPULSE) ? s_qd[i] : 0.f;
    }
}

// =============================================================================================
// stage 3: dphi/dq, dphi/dqd, dphi/d(F, r)
// =============================================================================================
// The walk of osd_walk with the joint accelerations x (qdd, or qd_plus at zero velocity for the impulse) added to alpha, and
// a second velocity recursion (wt, vt) at the joint rates tau^:
//   d = R r;  v += w x d;  vt += wt x d;  a += alpha x d + w x (w x d);  R <- R F
//   movable joint c: z = R e_z;  alpha += qd_c (w x z) + x_c z;  w += qd_c z;  wt += tau^_c z;  R <- R Rz(q_c)
//   link e: phi += lambda_e . (vt, wt) - nu_e . (a, alpha)     (angular rows in pose mode only)
// phi depends on q and the table only through the rotations, and v, a, vt only carry adjoints down the tree, so each step
// keeps its parent's (R, w, alpha, wt) and (cos, sin) of its joint: STEP_FLOATS per step and row.  The reverse sweep hands
// adjoints down the tree as the walk handed states up: through registers to the previous step, or through a branch slot
// (BSLOT_FLOATS: the adjoints of R, w, alpha, wt, v, a, vt) that the children restored from their saved state add into.
constexpr int STEP_FLOATS = 20;
constexpr int FSLOT_FLOATS = 18;
constexpr int BSLOT_FLOATS = 27;

struct KinBwdArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;        // null for the impulse (zero velocity)
    const float* __restrict__ x;         // [B, n] qdd / qd_plus
    const float* __restrict__ lam;       // [B, M]
    const float* __restrict__ nu;        // [B, M]
    const float* __restrict__ taubar;    // [B, n]
    const uint8_t* __restrict__ ok;      // [B]
    float* __restrict__ q_grad;          // [B, n] added to, or null
    float* __restrict__ qd_grad;         // [B, n] added to, or null (the impulse: always null)
    float* __restrict__ partials;        // [gridDim.x, n_links * 28] or null
    int64_t batch;
    int32_t M;
    int32_t vec_ok;
};

struct KinBwdSmem {
    int table, acc, scratch, q, qd, x, tb, lam, nu, qg, qdg, step, fslot, bslot, total_floats;
    __host__ __device__ KinBwdSmem(int T, int NT, const TreeProgram& tp, const UnionProgram& P, int M) {
        const int n = tp.n_dofs;
        auto tile4 = [](int f) { return (f + 3) & ~3; };      // row-major tiles staged with float4 copies
        int o = 0;
        table = o;  o += tp.n_links * DRMB200_TABLE_STRIDE;
        acc = o;    o += tile4(tp.n_links * 12);
        scratch = o; o += tile4(block_accumulate_floats(12, NT));
        q = o;      o += tile4(T * n);
        qd = o;     o += tile4(T * n);
        x = o;      o += tile4(T * n);
        tb = o;     o += tile4(T * n);
        lam = o;    o += tile4(T * M);
        nu = o;     o += tile4(T * M);
        qg = o;     o += tile4(T * n);
        qdg = o;    o += tile4(T * n);
        step = o;   o += STEP_FLOATS * P.walk.n_steps * T;
        fslot = o;  o += FSLOT_FLOATS * P.walk.n_state_slots * T;
        bslot = o;  o += BSLOT_FLOATS * P.walk.n_state_slots * T;
        total_floats = o;
    }
};

template <int T, bool IMPULSE>
__global__ void __launch_bounds__(T < 32 ? 32 : T)
contact_kinematic_backward_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ UnionProgram P,
                                  const KinBwdArgs args) {
    // block_accumulate reduces whole warps: a CTA of T < 32 rows runs 32 threads, and threads T.. only join its reductions
    // (with zeros); they hold no row state
    constexpr int NT = T < 32 ? 32 : T;
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs;
    const int M = args.M;
    const int MR = M / P.walk.n_ee;
    const MultiProgram& W = P.walk;
    const KinBwdSmem L(T, NT, prog, P, M);
    float* s_tab = smem + L.table;
    float* s_acc = smem + L.acc;
    const int tid = threadIdx.x;
    const bool need_table = args.partials != nullptr;
    const bool vec_ok = args.vec_ok;

    stage_canonical_table(s_tab, args.table, prog, NT);
    for (int i = tid; i < prog.n_links * 12; i += NT) s_acc[i] = 0.f;

    const int64_t n_tiles = (args.batch + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t start = tile * T;
        const int valid = (int)min((int64_t)T, args.batch - start);
        __syncthreads();                                // previous tile fully consumed
        coop_copy(smem + L.q, args.q + start * n, valid * n, vec_ok);
        if (!IMPULSE) coop_copy(smem + L.qd, args.qd + start * n, valid * n, vec_ok);
        coop_copy(smem + L.x, args.x + start * n, valid * n, vec_ok);
        coop_copy(smem + L.tb, args.taubar + start * n, valid * n, vec_ok);
        coop_copy(smem + L.lam, args.lam + start * M, valid * M, vec_ok);
        coop_copy(smem + L.nu, args.nu + start * M, valid * M, vec_ok);
        for (int i = tid; i < T * n; i += NT) { smem[L.qg + i] = 0.f; smem[L.qdg + i] = 0.f; }
        for (int i = tid; i < BSLOT_FLOATS * W.n_state_slots * T; i += NT) smem[L.bslot + i] = 0.f;
        __syncthreads();

        const bool lane = tid < T;                      // a thread with row state
        const bool row = tid < valid;
        const bool active = row && args.ok[start + tid] != 0;
        const int r = row ? tid : 0;                    // rows past the batch walk row 0's data and contribute nothing
        const int ts = lane ? tid : 0;                  // (threads T.. never touch row state)
        const float* qrow = smem + L.q + r * n;
        const float* qdrow = smem + L.qd + r * n;
        const float* xrow = smem + L.x + r * n;
        const float* tbrow = smem + L.tb + r * n;
        const float* lrow = smem + L.lam + r * M;
        const float* nrow = smem + L.nu + r * M;
        float* qg = smem + L.qg + ts * n;
        float* qdg = smem + L.qdg + ts * n;
        float* stp = smem + L.step + ts;
        float* fsl = smem + L.fslot + ts;
        float* bsl = smem + L.bslot + ts;
        const V3 zero = v3(0.f, 0.f, 0.f);

        // ---- forward walk: every step's parent state ------------------------------------------------
        if (lane) {
            M3 R = identity3();
            V3 w = zero, al = zero, wt = zero;
            for (int k = 0; k < W.n_steps; ++k) {
                const int src = W.psrc[k];
                if (src < 0) {
                    R = identity3(); w = al = wt = zero;
                } else if (src > 0) {
                    const float* s = fsl + (src - 1) * FSLOT_FLOATS * T;
                    R = ldm(s, T); w = ldv(s + 9 * T, T); al = ldv(s + 12 * T, T); wt = ldv(s + 15 * T, T);
                }
                float* st = stp + k * STEP_FLOATS * T;
                stm(st, T, R); stv(st + 9 * T, T, w); stv(st + 12 * T, T, al); stv(st + 15 * T, T, wt);
                M3 F; V3 rr;
                load_Fr(s_tab + (int)W.link[k] * DRMB200_TABLE_STRIDE, F, rr);
                R = mul(R, F);
                const int c = W.dof[k];
                if (c >= 0) {
                    float sn, cs;
                    sincos_pi2(qrow[c], sn, cs);
                    st[18 * T] = cs; st[19 * T] = sn;
                    const V3 z = col2(R);
                    const float qdc = IMPULSE ? 0.f : qdrow[c];
                    al = al + qdc * cross(w, z) + xrow[c] * z;
                    w = w + qdc * z;
                    wt = wt + tbrow[c] * z;
                    rotate_z(R, cs, sn);
                }
                const int sv = W.save[k];
                if (sv >= 0) {
                    float* s = fsl + sv * FSLOT_FLOATS * T;
                    stm(s, T, R); stv(s + 9 * T, T, w); stv(s + 12 * T, T, al); stv(s + 15 * T, T, wt);
                }
            }
        }

        // ---- reverse sweep ----------------------------------------------------------------------------
        M3 Rb = zero3();
        V3 wb = zero, alb = zero, wtb = zero, vb = zero, ab = zero, vtb = zero;
        for (int k = W.n_steps - 1; k >= 0; --k) {
            float vals[12] = {};
            if (lane) {
            if (!(k + 1 < W.n_steps && W.psrc[k + 1] == 0)) {   // step k + 1 did not continue from step k's registers
                Rb = zero3(); wb = alb = wtb = vb = ab = vtb = zero;
            }
            const int sv = W.save[k];
            if (sv >= 0) {                                   // the adjoints its branch children handed back
                float* s = bsl + sv * BSLOT_FLOATS * T;
                M3 t = ldm(s, T);
                Rb.a00 += t.a00; Rb.a01 += t.a01; Rb.a02 += t.a02; Rb.a10 += t.a10; Rb.a11 += t.a11; Rb.a12 += t.a12;
                Rb.a20 += t.a20; Rb.a21 += t.a21; Rb.a22 += t.a22;
                wb = wb + ldv(s + 9 * T, T); alb = alb + ldv(s + 12 * T, T); wtb = wtb + ldv(s + 15 * T, T);
                vb = vb + ldv(s + 18 * T, T); ab = ab + ldv(s + 21 * T, T); vtb = vtb + ldv(s + 24 * T, T);
                for (int i = 0; i < BSLOT_FLOATS; ++i) s[i * T] = 0.f;
            }
            const int l = W.ee[k];
            if (l >= 0) {
                const float* lm = lrow + MR * l;
                const float* nm = nrow + MR * l;
                vtb = vtb + v3(lm[0], lm[1], lm[2]);
                ab = ab - v3(nm[0], nm[1], nm[2]);
                if (MR == 6) {
                    wtb = wtb + v3(lm[3], lm[4], lm[5]);
                    alb = alb - v3(nm[3], nm[4], nm[5]);
                }
            }
            const float* st = stp + k * STEP_FLOATS * T;
            const M3 R = ldm(st, T);
            const V3 w = ldv(st + 9 * T, T), al = ldv(st + 12 * T, T), wt = ldv(st + 15 * T, T);
            M3 F; V3 rr;
            load_Fr(s_tab + (int)W.link[k] * DRMB200_TABLE_STRIDE, F, rr);
            M3 Mk = F;
            const int c = W.dof[k];
            float cs = 1.f, sn = 0.f;
            if (c >= 0) {
                cs = st[18 * T]; sn = st[19 * T];
                const V3 z = col2(mul(R, F));
                const float qdc = IMPULSE ? 0.f : qdrow[c];
                const V3 zb = qdc * cross(alb, w) + xrow[c] * alb + qdc * wb + tbrow[c] * wtb;
                if (!IMPULSE) qdg[c] += dot(alb, cross(w, z)) + dot(wb, z);
                wb = wb + qdc * cross(z, alb);
                Rb.a02 += zb.x; Rb.a12 += zb.y; Rb.a22 += zb.z;
                rotate_z(Mk, cs, sn);
            }
            // R_out = R Mk
            const M3 Mbar = mulTN(R, Rb);
            if (c >= 0) qg[c] += theta_grad_z(Mbar, Mk);
            M3 Rb_in = mulNT(Rb, Mk);
            // d = R r feeds v, vt and a
            const V3 d = mul(R, rr);
            const V3 u = cross(w, d);
            const V3 ub = cross(ab, w);
            const V3 db = cross(ab, al) + cross(ub, w) + cross(vb, w) + cross(vtb, wt);
            alb = alb + cross(d, ab);
            wb = wb + cross(u, ab) + cross(d, ub) + cross(d, vb);
            wtb = wtb + cross(d, vtb);
            add_outer(Rb_in, db, rr);
            {
                M3 Fbar = Mbar;
                if (c >= 0) rotate_z(Fbar, cs, -sn);       // Mbar Rz^T
                const V3 rbar = mulT(R, db);
                m3_to_array(Fbar, vals);
                vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z;
            }
            Rb = Rb_in;
            const int src = W.psrc[k];
            if (src > 0) {                                   // hand the parent state's adjoint back to its branch slot
                float* s = bsl + (src - 1) * BSLOT_FLOATS * T;
                M3 t = ldm(s, T);
                t.a00 += Rb.a00; t.a01 += Rb.a01; t.a02 += Rb.a02; t.a10 += Rb.a10; t.a11 += Rb.a11; t.a12 += Rb.a12;
                t.a20 += Rb.a20; t.a21 += Rb.a21; t.a22 += Rb.a22;
                stm(s, T, t);
                stv(s + 9 * T, T, ldv(s + 9 * T, T) + wb); stv(s + 12 * T, T, ldv(s + 12 * T, T) + alb);
                stv(s + 15 * T, T, ldv(s + 15 * T, T) + wtb); stv(s + 18 * T, T, ldv(s + 18 * T, T) + vb);
                stv(s + 21 * T, T, ldv(s + 21 * T, T) + ab); stv(s + 24 * T, T, ldv(s + 24 * T, T) + vtb);
            }
            }   // lane
            if (need_table)
                block_accumulate<12, NT>(smem + L.scratch, s_acc + (int)W.link[k] * 12, vals, active && lane,
                                         [](int j) { return j; });
        }
        __syncthreads();
        // add this tile's rows (unsolved and idle rows add nothing)
        for (int i = tid; i < valid * n; i += NT) {
            const int rr = i / n;
            if (args.ok[start + rr] == 0) continue;
            if (args.q_grad != nullptr) args.q_grad[start * n + i] += smem[L.qg + i];
            if (!IMPULSE && args.qd_grad != nullptr) args.qd_grad[start * n + i] += smem[L.qdg + i];
        }
    }
    if (need_table) {
        __syncthreads();
        float* out = args.partials + (size_t)blockIdx.x * prog.n_links * DRMB200_TABLE_STRIDE;
        for (int i = tid; i < prog.n_links * DRMB200_TABLE_STRIDE; i += NT) out[i] = 0.f;
        __syncthreads();
        for (int i = tid; i < prog.n_links * 12; i += NT) {   // canonical -> natural entries (bijection per row)
            const int l = i / 12, e = i - l * 12;
            const int p = prog.parent[l];
            int src;
            const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
            out[l * DRMB200_TABLE_STRIDE + src] = sg * s_acc[i];
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static TileChoice contact_backward_tile(const TreeProgram& prog, const UnionProgram& P, int M) {
    return tile_ladder([&](int T) { return (size_t)ContactBwdSmemLayout(T, prog, P, M).total_floats * sizeof(float); }, 0);
}
static TileChoice kinematic_backward_tile(const TreeProgram& prog, const UnionProgram& P, int M) {
    return tile_ladder([&](int T) {
        return (size_t)KinBwdSmem(T, T < 32 ? 32 : T, prog, P, M).total_floats * sizeof(float);
    }, 0);
}

// the grid bound of the persistent kinematic kernel: at most one CTA per row and at most BWD_MAX_GRID
static int64_t kinematic_grid_bound(int64_t batch) { return batch < BWD_MAX_GRID ? (batch < 1 ? 1 : batch) : BWD_MAX_GRID; }

struct ContactBwdWorkspace {
    int64_t fd, partials, nu, ghat, tauc, taubar, q_safe, qd_safe, ok, total;
    ContactBwdWorkspace(const drmb200_topology_t* topo, int n, int M, int64_t batch) {
        int64_t o = 0;
        fd = o;       o += round256(forward_dynamics_backward_workspace_bytes(topo, batch));
        partials = o; o += round256(kinematic_grid_bound(batch) * topo->n_links * DRMB200_TABLE_STRIDE * (int64_t)sizeof(float));
        nu = o;       o += round256(batch * M * (int64_t)sizeof(float));
        ghat = o;     o += round256(batch * n * (int64_t)sizeof(float));
        tauc = o;     o += round256(batch * n * (int64_t)sizeof(float));
        taubar = o;   o += round256(batch * n * (int64_t)sizeof(float));
        q_safe = o;   o += round256(batch * n * (int64_t)sizeof(float));
        qd_safe = o;  o += round256(batch * n * (int64_t)sizeof(float));
        ok = o;       o += round256(batch);
        total = o;
    }
};

int64_t contact_backward_workspace_bytes(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links,
                                         int32_t position_only, int64_t batch) {
    if (topo == nullptr || topo->n_links < 1 || topo->n_links > DRMB200_MAX_LINKS || n_ee < 1 || n_ee > MT_MAX_EE ||
        ee_links == nullptr || batch < 0)
        return 0;
    const int M = (position_only ? 3 : 6) * n_ee;
    return ContactBwdWorkspace(topo, topo->n_dofs, M, batch).total;
}

template <bool IMPULSE>
static int contact_backward(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                            const float* q, const float* qd, const float* f, const float* ref, const float* out,
                            const float* lam, const uint8_t* solved, int64_t batch, uint32_t flags, int32_t position_only,
                            float regularization, const float* g_out, const float* g_lam, float* q_grad, float* qd_grad,
                            float* f_grad, float* ref_grad, float* table_grad, void* workspace, cudaStream_t stream) {
    (void)ref;      // accel_ref / velocity_ref enter only through the forward's outputs
    UnionProgram P;
    const TreeProgram* prog = nullptr;
    int rc = contact_programs(topo, n_ee, ee_links, regularization, batch, &P, &prog);
    if (rc != DRMB200_OK) return rc;
    const char* what = IMPULSE ? "contact impulse backward" : "contact dynamics backward";
    const int M = (position_only ? 3 : 6) * n_ee;
    const int n = prog->n_dofs;
    // every refusal before any launch
    const TileChoice c1 = contact_backward_tile(*prog, P, M);
    const TileChoice c3 = kinematic_backward_tile(*prog, P, M);
    if (c1.bytes > SMEM_CTA_MAX || c3.bytes > SMEM_CTA_MAX) {
        set_error("%s needs %zu B of shared memory per CTA (> 227 KB) for one row (%d joints, %d links, M = %d)", what,
                  c1.bytes > c3.bytes ? c1.bytes : c3.bytes, n, prog->n_links, M);
        return DRMB200_ELIMIT;
    }
    if (batch == 0) return DRMB200_OK;     // empty tensors may have null data pointers
    if (table == nullptr || q == nullptr || qd == nullptr || (!IMPULSE && f == nullptr) || out == nullptr ||
        lam == nullptr || solved == nullptr) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    if (workspace == nullptr) { set_error("%s needs its workspace (drmb200_contact_backward_workspace_bytes)", what); return DRMB200_EINVAL; }
    const bool want_kin = q_grad != nullptr || (!IMPULSE && qd_grad != nullptr) || table_grad != nullptr;
    const bool want_fd = want_kin || f_grad != nullptr;
    const bool want_any = want_fd || ref_grad != nullptr || (IMPULSE && qd_grad != nullptr);
    if (!want_any) return DRMB200_OK;

    const ContactBwdWorkspace ws(topo, n, M, batch);
    char* base = static_cast<char*>(workspace);
    float* nu = ref_grad != nullptr ? ref_grad : reinterpret_cast<float*>(base + ws.nu);
    float* ghat = (IMPULSE && qd_grad != nullptr) ? qd_grad : reinterpret_cast<float*>(base + ws.ghat);
    float* tauc = reinterpret_cast<float*>(base + ws.tauc);
    float* taubar = f_grad != nullptr ? f_grad : reinterpret_cast<float*>(base + ws.taubar);
    float* q_safe = reinterpret_cast<float*>(base + ws.q_safe);
    float* qd_safe = reinterpret_cast<float*>(base + ws.qd_safe);
    uint8_t* ok = reinterpret_cast<uint8_t*>(base + ws.ok);

    // stage 1
    ContactBwdArgs a1;
    a1.table = table; a1.q = q; a1.qd = qd; a1.f = IMPULSE ? nullptr : f; a1.lam = lam; a1.g_out = g_out; a1.g_lam = g_lam;
    a1.solved = solved;
    a1.nu = nu; a1.ghat = ghat; a1.tauc = tauc; a1.q_safe = q_safe; a1.qd_safe = qd_safe; a1.ok = ok;
    a1.batch = batch; a1.flags = IMPULSE ? 0u : (flags & (DRMB200_GRAVITY | DRMB200_DAMPING));
    a1.M = M; a1.mu = regularization;
    a1.aligned = aligned16(q, qd, IMPULSE ? nullptr : f, lam, g_out, g_lam);
    {
        const int64_t tiles = (batch + c1.tile - 1) / c1.tile;
#define DRM_LAUNCH_CB(TT) \
        rc = launch_kernel<contact_backward_kernel<TT, IMPULSE>>(tiles, TT, c1.bytes, stream, false, what, *prog, P, a1)
        switch (c1.tile) {
            case 64: DRM_LAUNCH_CB(64); break;
            case 32: DRM_LAUNCH_CB(32); break;
            case 16: DRM_LAUNCH_CB(16); break;
            case 8: DRM_LAUNCH_CB(8); break;
            case 4: DRM_LAUNCH_CB(4); break;
            case 2: DRM_LAUNCH_CB(2); break;
            default: DRM_LAUNCH_CB(1); break;
        }
#undef DRM_LAUNCH_CB
        if (rc != DRMB200_OK) return rc;
    }
    if (!want_fd) return DRMB200_OK;

    // stage 2: the forward-dynamics adjoint at (q, qd, tau_c) (the impulse: (q, 0, J^T Lambda), no flags), zero state on
    // unsolved rows
    rc = forward_dynamics_backward_device(topo, table, q_safe, qd_safe, tauc, batch, a1.flags, ghat, q_grad,
                                          IMPULSE ? nullptr : qd_grad, taubar, table_grad, base + ws.fd, stream);
    if (rc != DRMB200_OK) return rc;
    if (!want_kin) return DRMB200_OK;

    // stage 3
    KinBwdArgs a3;
    a3.table = table; a3.q = q; a3.qd = IMPULSE ? nullptr : qd; a3.x = out; a3.lam = lam; a3.nu = nu; a3.taubar = taubar;
    a3.ok = ok; a3.q_grad = q_grad; a3.qd_grad = IMPULSE ? nullptr : qd_grad;
    a3.partials = table_grad != nullptr ? reinterpret_cast<float*>(base + ws.partials) : nullptr;
    a3.batch = batch; a3.M = M;
    a3.vec_ok = aligned16(q, IMPULSE ? nullptr : qd, out, lam, nu, taubar);
    const int64_t tiles = (batch + c3.tile - 1) / c3.tile;
    int grid = 0;
#define DRM_LAUNCH_KB(TT) \
    rc = launch_persistent<contact_kinematic_backward_kernel<TT, IMPULSE>>(TT < 32 ? 32 : TT, c3.bytes, tiles, stream, what, \
                                                                            &grid, *prog, P, a3)
    switch (c3.tile) {
        case 64: DRM_LAUNCH_KB(64); break;
        case 32: DRM_LAUNCH_KB(32); break;
        case 16: DRM_LAUNCH_KB(16); break;
        case 8: DRM_LAUNCH_KB(8); break;
        case 4: DRM_LAUNCH_KB(4); break;
        case 2: DRM_LAUNCH_KB(2); break;
        default: DRM_LAUNCH_KB(1); break;
    }
#undef DRM_LAUNCH_KB
    if (rc != DRMB200_OK) return rc;
    return table_grad != nullptr ? launch_reduce(a3.partials, grid, topo, table_grad, stream) : DRMB200_OK;
}

int contact_dynamics_backward_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                     const float* q, const float* qd, const float* f, const float* accel_ref, const float* qdd,
                                     const float* force, const uint8_t* solved, int64_t batch, uint32_t flags,
                                     int32_t position_only, float regularization, const float* g_qdd, const float* g_force,
                                     float* q_grad, float* qd_grad, float* f_grad, float* accel_ref_grad, float* table_grad,
                                     void* workspace, cudaStream_t stream) {
    return contact_backward<false>(topo, n_ee, ee_links, table, q, qd, f, accel_ref, qdd, force, solved, batch, flags,
                                   position_only, regularization, g_qdd, g_force, q_grad, qd_grad, f_grad, accel_ref_grad,
                                   table_grad, workspace, stream);
}

int contact_impulse_backward_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                    const float* q, const float* qd, const float* velocity_ref, const float* qd_plus,
                                    const float* impulse, const uint8_t* solved, int64_t batch, int32_t position_only,
                                    float regularization, const float* g_qd_plus, const float* g_impulse, float* q_grad,
                                    float* qd_grad, float* velocity_ref_grad, float* table_grad, void* workspace,
                                    cudaStream_t stream) {
    return contact_backward<true>(topo, n_ee, ee_links, table, q, qd, nullptr, velocity_ref, qd_plus, impulse, solved, batch,
                                  0u, position_only, regularization, g_qd_plus, g_impulse, q_grad, qd_grad, nullptr,
                                  velocity_ref_grad, table_grad, workspace, stream);
}

}  // namespace drm
