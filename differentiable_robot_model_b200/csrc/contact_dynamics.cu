// contact_dynamics.cu -- batched contact dynamics and contact impulses of rigid contacts at several links (sm_90a).
//
// Per row (q, qd, f) and a list of E links held by bilateral rigid contacts, in ONE launch (spec in include/drm_b200.h and
// DESIGN.md §3), with J [M, n] the links' stacked Jacobians and G = dqdd_df exactly as operational_space.cu builds them:
//   A = J G J^T + mu I_M
//   contact dynamics:  A lambda = a_ref - (J qdd_free + Jdot qd),  qdd     = qdd_free + G J^T lambda,  force   = lambda
//   contact impulse:   A Lambda = v_ref - J qd,                    qd_plus = qd       + G J^T Lambda,  impulse = Lambda
// where qdd_free is the forward dynamics at (q, qd, f) with the call's flags.
//
// One thread per row, one kernel template for both modes (IMPULSE).  The row follows the operational-space kernel step by
// step, with its device code (osd_common.cuh); steps 1-5 are contact_row (contact_common.cuh), which the contact rollout
// (contact_rollout.cu) runs for every step:
//   1. osd_walk: J, J qd and Jdot qd;
//   2. aba_body: qdd_free, and the q-dependent U, d, cos, sin of every link (the impulse runs it at zero velocity, zero force
//      and without gravity -- f is not read -- and keeps only U, d, cos, sin);
//   3. osd_inverse_inertia: A in the smaller space (M sweeps of aba_unit_response when M <= n_u, else n_u rank-1 sweeps),
//      then mu on the diagonal;
//   4. contact_solve: Jacobi equilibration s_k = |A_kk|^-1/2, Gaussian elimination with partial pivoting on S A S (ties to
//      the lower row), back substitution; a row is unsolved when an A_kk is zero or not finite or a pivot is not finite or
//      has magnitude <= CONTACT_PIVOT_MIN;
//   5. tau = J^T lambda and ONE more aba_unit_response for G J^T lambda, added to qdd_free (or qd).
// An unsolved row gets solved = 0 and NaN in both outputs.
//
// Shared memory, per row and slot-major (element e of row t at base[e * T + t]) except the ABA's q / qd / f / qdd rows
// (AbaSmemLayout) and the staged reference rows: the ABA link and branch state, J [M][n_u], the walk's joint scratch and
// spilled branch state, J qd and Jdot qd [M], the right-hand side / solution [M], the scales [M], the dense A [M][M] (9.2 KB
// per row at M = 48) and the joint output [n].  Outputs leave through store_transposed.
#include <cmath>
#include "launch.cuh"
#include "contact_common.cuh"

namespace drm {

struct ContactArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ f;       // [B, n]; null for the impulse
    const float* __restrict__ ref;     // [B, M] a_ref / v_ref, or null (0)
    float* __restrict__ out;           // [B, n] qdd / qd_plus
    float* __restrict__ force;         // [B, M] lambda / Lambda, or null
    uint8_t* __restrict__ solved;      // [B]
    int64_t batch;
    uint32_t flags;
    int32_t M;                         // rows: 6 n_ee (pose) or 3 n_ee (position only)
    float mu;
    int32_t aligned;
};

struct ContactSmemLayout {
    AbaSmemLayout aba;
    int ref, jac, jscr, state, vel, bias, lam, scale, a, out, total_floats;
    __host__ __device__ ContactSmemLayout(int T, const TreeProgram& tp, const UnionProgram& P, int M)
        : aba(T, tp.n_dofs, tp.n_links, tp.n_slots) {
        int o = (aba.total_floats + 3) & ~3;   // 16-byte aligned: the reference rows are staged with float4 copies
        ref = o;   o += M * T;
        jac = o;   o += M * P.n_u * T;
        jscr = o;  o += 6 * P.walk.n_jslots * T;
        state = o; o += OSD_STATE * P.walk.n_state_slots * T;
        vel = o;   o += M * T;
        bias = o;  o += M * T;
        lam = o;   o += M * T;
        scale = o; o += M * T;
        a = o;     o += M * M * T;
        out = o;   o += tp.n_dofs * T;
        total_floats = o;
    }
};

template <int T, bool IMPULSE>
__global__ void __launch_bounds__(T)
contact_dynamics_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ UnionProgram P, const ContactArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = prog.n_dofs;
    const int M = args.M;
    const int MR = M / P.walk.n_ee;
    const int n_u = P.n_u;
    const ContactSmemLayout L(T, prog, P, M);
    float* s_q = smem + L.aba.q;
    float* s_qd = smem + L.aba.qd;
    float* s_f = smem + L.aba.f;
    float* s_qdd = smem + L.aba.qdd;
    float* s_tab = smem + L.aba.table;

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
            mbar_arrive_expect_tx(&mbar, (IMPULSE ? 2u : 3u) * bytes);
            bulk_g2s(s_q, args.q + tile_start * n, bytes, &mbar);
            bulk_g2s(s_qd, args.qd + tile_start * n, bytes, &mbar);
            if (!IMPULSE) bulk_g2s(s_f, args.f + tile_start * n, bytes, &mbar);
        }
    } else {
        coop_copy(s_q, args.q + tile_start * n, valid * n, vec_ok);
        coop_copy(s_qd, args.qd + tile_start * n, valid * n, vec_ok);
        if (!IMPULSE) coop_copy(s_f, args.f + tile_start * n, valid * n, vec_ok);
    }
    if (IMPULSE)            // the impulse's ABA runs at zero velocity and force: only its q-dependent U, d, cos, sin are used
        for (int i = tid; i < T * n; i += T) s_f[i] = 0.f;
    if (args.ref != nullptr) coop_copy(smem + L.ref, args.ref + tile_start * M, valid * M, vec_ok);
    else for (int i = L.ref + tid; i < L.ref + T * M; i += T) smem[i] = 0.f;
    stage_canonical_table(s_tab, args.table, prog, T);
    // J, velocity and bias start at zero: columns off a link's path
    for (int i = L.jac + tid; i < L.jscr; i += T) smem[i] = 0.f;
    for (int i = L.vel + tid; i < L.lam; i += T) smem[i] = 0.f;
    __syncthreads();
    if (bulk) mbar_wait(&mbar, 0);

    if (tid < valid) {
        bool ok;
        DRM_CONTACT_ROW(T, IMPULSE, false, nullptr, args.flags, args.mu, ok, false, 0.f, );
        args.solved[tile_start + tid] = ok ? 1 : 0;
    }
    __syncthreads();
    store_transposed(args.out + tile_start * n, smem + L.out, n, valid, T);
    if (args.force != nullptr) store_transposed(args.force + tile_start * M, smem + L.lam, M, valid, T);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// the largest power-of-two tile <= 64 rows while two CTAs still fit an SM, else down to one row per CTA
static TileChoice contact_tile(const TreeProgram& prog, const UnionProgram& P, int M, size_t static_bytes) {
    return tile_ladder([&](int T) { return (size_t)ContactSmemLayout(T, prog, P, M).total_floats * sizeof(float); }, static_bytes);
}

template <bool IMPULSE>
static int contact_launch(const TreeProgram& prog, const UnionProgram& P, const ContactArgs& args, cudaStream_t stream) {
    // every instantiation declares the same static shared memory (the mbarrier)
    size_t static_bytes;
    int rc = static_smem_bytes<contact_dynamics_kernel<64, IMPULSE>>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    const TileChoice c = contact_tile(prog, P, args.M, static_bytes);
    const char* what = IMPULSE ? "contact impulse" : "contact dynamics";
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("%s needs %zu B of shared memory per CTA (> 227 KB) for one row (%d joints, %d links, M = %d)", what,
                  c.bytes + static_bytes, prog.n_dofs, prog.n_links, args.M);
        return DRMB200_ELIMIT;
    }
    const int64_t tiles = (args.batch + c.tile - 1) / c.tile;
#define DRM_LAUNCH_CONTACT(TT) \
    launch_kernel<contact_dynamics_kernel<TT, IMPULSE>>(tiles, TT, c.bytes, stream, false, what, prog, P, args)
    switch (c.tile) {
        case 64: return DRM_LAUNCH_CONTACT(64);
        case 32: return DRM_LAUNCH_CONTACT(32);
        case 16: return DRM_LAUNCH_CONTACT(16);
        case 8: return DRM_LAUNCH_CONTACT(8);
        case 4: return DRM_LAUNCH_CONTACT(4);
        case 2: return DRM_LAUNCH_CONTACT(2);
        default: return DRM_LAUNCH_CONTACT(1);
    }
#undef DRM_LAUNCH_CONTACT
}

// The argument checks shared by both entry points and the contact rollout (contact_rollout.cu); on success P and *prog
// describe the walk and the (unfolded) tree.
int contact_programs(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, float regularization,
                            int64_t batch, UnionProgram* P, const TreeProgram** prog) {
    if (n_ee < 1 || n_ee > MT_MAX_EE) { set_error("n_ee=%d outside [1, %d]", n_ee, MT_MAX_EE); return DRMB200_EINVAL; }
    if (ee_links == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    int rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);  // first, so a tree the ABA refuses gets the ABA's message
    if (cp == nullptr) return rc;
    rc = build_union_program(topo, n_ee, ee_links, P);
    if (rc != DRMB200_OK) return rc;
    for (int l = 0; l < n_ee; ++l) {        // such a link has only zero rows: its constraint can never be solved
        int movable = 0;
        for (int c = 0; c < P->walk.n_dofs; ++c) movable += P->walk.cslot[l][c] >= 0;
        if (movable == 0) {
            set_error("ee_links[%d]=%d: no movable joint between the root and this link", l, ee_links[l]);
            return DRMB200_EINVAL;
        }
    }
    if (!(regularization >= 0.f) || !std::isfinite(regularization)) {
        set_error("regularization=%g: must be finite and >= 0", (double)regularization);
        return DRMB200_EINVAL;
    }
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    *prog = &cp->full;                      // unfolded: the walk and the ABA share one staged canonical table
    return DRMB200_OK;
}

int contact_dynamics_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                            const float* q, const float* qd, const float* f, const float* accel_ref, int64_t batch,
                            uint32_t flags, int32_t position_only, float regularization, float* qdd, float* force,
                            uint8_t* solved, cudaStream_t stream) {
    UnionProgram P;
    const TreeProgram* prog = nullptr;
    const int rc = contact_programs(topo, n_ee, ee_links, regularization, batch, &P, &prog);
    if (rc != DRMB200_OK) return rc;
    if (batch == 0) return DRMB200_OK;     // empty tensors may have null data pointers
    if (table == nullptr || q == nullptr || qd == nullptr || f == nullptr || qdd == nullptr || solved == nullptr) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    ContactArgs args;
    args.table = table; args.q = q; args.qd = qd; args.f = f; args.ref = accel_ref;
    args.out = qdd; args.force = force; args.solved = solved;
    args.batch = batch; args.flags = flags & (DRMB200_GRAVITY | DRMB200_DAMPING);
    args.M = (position_only ? 3 : 6) * n_ee;
    args.mu = regularization;
    args.aligned = aligned16(q, qd, f, accel_ref);
    return contact_launch<false>(*prog, P, args, stream);
}

int contact_impulse_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                           const float* q, const float* qd, const float* velocity_ref, int64_t batch, int32_t position_only,
                           float regularization, float* qd_plus, float* impulse, uint8_t* solved, cudaStream_t stream) {
    UnionProgram P;
    const TreeProgram* prog = nullptr;
    const int rc = contact_programs(topo, n_ee, ee_links, regularization, batch, &P, &prog);
    if (rc != DRMB200_OK) return rc;
    if (batch == 0) return DRMB200_OK;     // empty tensors may have null data pointers
    if (table == nullptr || q == nullptr || qd == nullptr || qd_plus == nullptr || solved == nullptr) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    ContactArgs args;
    args.table = table; args.q = q; args.qd = qd; args.f = nullptr; args.ref = velocity_ref;
    args.out = qd_plus; args.force = impulse; args.solved = solved;
    args.batch = batch; args.flags = 0;
    args.M = (position_only ? 3 : 6) * n_ee;
    args.mu = regularization;
    args.aligned = aligned16(q, qd, velocity_ref);
    return contact_launch<true>(*prog, P, args, stream);
}

}  // namespace drm
