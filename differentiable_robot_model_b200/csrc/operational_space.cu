// operational_space.cu -- batched operational-space dynamics of several links (sm_90a).
//
// Per row (q, qd, f) and a list of E links, in ONE launch (spec in include/drm_b200.h and DESIGN.md §3):
//   J               [M, n]  the links' geometric Jacobians stacked (6 rows per link: linear over angular; 3 for position only)
//   inv_inertia     [M, M]  J G J^T, G[:, j] = forward dynamics at (q, 0, e_j) without gravity or damping (dqdd_df)
//   velocity        [M]     J qd
//   bias            [M]     Jdot qd: the link origins' classical accelerations (and angular accelerations) at qdd = 0
//   acceleration    [M]     J qdd + Jdot qd, qdd = forward dynamics at (q, qd, f) with the call's flags
//
// One thread per row.  Three parts share the row's shared-memory state (their device code is in osd_common.cuh, which the
// contact-dynamics kernel shares):
//   * kinematics: one depth-first walk of the union of the root -> link paths (the MultiProgram of multi_program.cuh, in the
//     canonical +z frames, unfolded, so links behind fixed joints work).  Along the walk it propagates, besides (R, p), the
//     angular velocity omega, the origin velocity v, and at qdd = 0 the angular acceleration alpha and the origin's
//     classical acceleration a, all in the world frame:  with d = R_parent r_i,
//         v_i = v_p + omega_p x d,   a_i = a_p + alpha_p x d + omega_p x (omega_p x d),
//     then at a joint with world axis z and rate qd:  alpha += qd omega x z,  omega += qd z.
//     At link e, J qd = (v_e; omega_e) and Jdot qd = (a_e; alpha_e) -- the same quantities as
//     sum_j qd_j [(omega_j x z_j) x (p_e - p_j) + z_j x (v_e - v_j);  omega_j x z_j], but every term is a short local
//     vector, so nothing cancels when the links are far from the world origin.  The state is spilled at branch points.
//   * forward dynamics: aba_body.cuh on the whole (unfolded) tree gives qdd and leaves, per link, cos / sin of the joint angle,
//     U and d of the articulated inertia.  Those depend on q only, so every further right-hand side tau is two O(n) sweeps of
//     6-vectors at zero velocity and zero gravity, with the articulated-body arithmetic of aba_body (the tangent of its passes
//     2 and 3 in f):  leaves -> root  u = tau - p_z, pa = p + U u / (d + eps), p_parent += X^T pa;
//                     root -> leaves  a' = X a_parent, x = (u - U . a') / d, a = a' + e_z x.
//   * the product is formed in the smaller space (U = the movable joints on the union of the paths, n_u of them):
//         M <= n_u:  M sweeps with tau = J^T e_k give the columns of G J^T, then inv_inertia[:, k] = J (G J^T e_k);
//         M >  n_u:  n_u sweeps with tau = e_j give the columns G e_j, then inv_inertia += (J G e_j) J[:, j]^T.
//
// Shared memory, per row and slot-major (element e of row t at base[e * T + t]) except the ABA's q / qd / f / qdd rows
// (AbaSmemLayout): the ABA link and branch state, J [M][n_u], the walk's joint scratch (z, z x p per path depth) and spilled
// branch state (R, p, omega, v, alpha, a: 24 floats), and the output tiles inv_inertia [M][M], velocity, bias and acceleration
// [M].  The output tiles are written back with a cooperative transposing copy: consecutive threads store consecutive floats
// of the contiguous [T, M, M] block, so the stores coalesce without a second row-major copy of the tile in shared memory.
#include "launch.cuh"
#include "osd_common.cuh"

namespace drm {

struct OsdArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ f;
    float* __restrict__ inv_inertia;   // [B, M, M] or null
    float* __restrict__ acceleration;  // [B, M] or null
    float* __restrict__ velocity;      // [B, M] or null
    float* __restrict__ bias;          // [B, M] or null
    int64_t batch;
    uint32_t flags;
    int32_t M;                         // rows: 6 n_ee (pose) or 3 n_ee (position only)
    int32_t aligned;
};

struct OsdSmemLayout {
    AbaSmemLayout aba;
    int jac, jscr, state, vel, bias, acc, inv, total_floats;
    __host__ __device__ OsdSmemLayout(int T, const TreeProgram& tp, const UnionProgram& P, int M)
        : aba(T, tp.n_dofs, tp.n_links, tp.n_slots) {
        int o = aba.total_floats;
        jac = o;   o += M * P.n_u * T;
        jscr = o;  o += 6 * P.walk.n_jslots * T;
        state = o; o += OSD_STATE * P.walk.n_state_slots * T;
        vel = o;   o += M * T;
        bias = o;  o += M * T;
        acc = o;   o += M * T;
        inv = o;   o += M * M * T;
        total_floats = o;
    }
};

template <int T>
__global__ void __launch_bounds__(T)
operational_space_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ UnionProgram P, const OsdArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = prog.n_dofs;
    const int M = args.M;
    const int MR = M / P.walk.n_ee;
    const int n_u = P.n_u;
    const OsdSmemLayout L(T, prog, P, M);
    float* s_q = smem + L.aba.q;
    float* s_qd = smem + L.aba.qd;
    float* s_f = smem + L.aba.f;
    float* s_qdd = smem + L.aba.qdd;
    float* s_tab = smem + L.aba.table;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, args.batch - tile_start);
    const bool vec_ok = args.aligned;
    const bool bulk = args.aligned && n > 0 && ((valid & 3) == 0);

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
    stage_canonical_table(s_tab, args.table, prog, T);
    // J, velocity and bias start at zero: rows of links that are not walked (the root) and columns off a link's path
    for (int i = L.jac + tid; i < L.jscr; i += T) smem[i] = 0.f;
    for (int i = L.vel + tid; i < L.acc; i += T) smem[i] = 0.f;
    __syncthreads();
    if (bulk) mbar_wait(&mbar, 0);

    if (tid < valid) {
        const float* qrow = s_q + tid * n;
        const float* qdrow = s_qd + tid * n;
        float* frow = s_f + tid * n;
        float* qddrow = s_qdd + tid * n;
        float* lk0 = smem + L.aba.link + tid;
        float* sl0 = smem + L.aba.slots + tid;
        float* J = smem + L.jac + tid;
        float* vel = smem + L.vel + tid;
        float* bias = smem + L.bias + tid;
        float* acc = smem + L.acc + tid;
        float* inv = smem + L.inv + tid;
        const int rs = n_u * T;
        osd_walk<T>(P, s_tab, qrow, qdrow, MR, J, vel, bias, smem + L.jscr + tid, smem + L.state + tid);
        if (args.acceleration != nullptr || args.inv_inertia != nullptr) {
            aba_body<T>(prog, s_tab, qrow, qdrow, frow, qddrow, lk0, sl0, args.flags);
            for (int m = 0; m < M; ++m) {           // J qdd + Jdot qd
                float s = bias[m * T];
                for (int u = 0; u < n_u; ++u) s = fmaf(J[m * rs + u * T], qddrow[P.u_dof[u]], s);
                acc[m * T] = s;
            }
        }
        if (args.inv_inertia != nullptr) osd_inverse_inertia<T>(prog, P, s_tab, M, J, inv, frow, qddrow, lk0, sl0);
    }
    __syncthreads();
    if (args.inv_inertia != nullptr) store_transposed(args.inv_inertia + tile_start * M * M, smem + L.inv, M * M, valid, T);
    if (args.acceleration != nullptr) store_transposed(args.acceleration + tile_start * M, smem + L.acc, M, valid, T);
    if (args.velocity != nullptr) store_transposed(args.velocity + tile_start * M, smem + L.vel, M, valid, T);
    if (args.bias != nullptr) store_transposed(args.bias + tile_start * M, smem + L.bias, M, valid, T);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// the largest power-of-two tile <= 64 rows while two CTAs still fit an SM, else down to one row per CTA
static TileChoice osd_tile(const TreeProgram& prog, const UnionProgram& P, int M, size_t static_bytes) {
    return tile_ladder([&](int T) { return (size_t)OsdSmemLayout(T, prog, P, M).total_floats * sizeof(float); }, static_bytes);
}

int operational_space_dynamics_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                      const float* q, const float* qd, const float* f, int64_t batch, uint32_t flags,
                                      int32_t position_only, float* inv_inertia, float* acceleration, float* velocity,
                                      float* bias_acceleration, cudaStream_t stream) {
    if (n_ee < 1 || n_ee > MT_MAX_EE) { set_error("n_ee=%d outside [1, %d]", n_ee, MT_MAX_EE); return DRMB200_EINVAL; }
    if (ee_links == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    UnionProgram P;
    int rc = build_union_program(topo, n_ee, ee_links, &P);
    if (rc != DRMB200_OK) return rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);
    if (cp == nullptr) return rc;
    const TreeProgram& prog = cp->full;         // unfolded: the walk and the ABA share one staged canonical table
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (inv_inertia == nullptr && acceleration == nullptr && velocity == nullptr && bias_acceleration == nullptr) return DRMB200_OK;
    if (batch == 0) return DRMB200_OK;
    // q, qd, f may be null only for a model without movable joints (empty tensors): they are then never read
    if (table == nullptr || (prog.n_dofs > 0 && (q == nullptr || qd == nullptr || f == nullptr))) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }

    OsdArgs args;
    args.table = table; args.q = q; args.qd = qd; args.f = f;
    args.inv_inertia = inv_inertia; args.acceleration = acceleration; args.velocity = velocity; args.bias = bias_acceleration;
    args.batch = batch; args.flags = flags & (DRMB200_GRAVITY | DRMB200_DAMPING);
    args.M = (position_only ? 3 : 6) * n_ee;
    args.aligned = aligned16(q, qd, f);

    // every instantiation declares the same static shared memory (the mbarrier)
    size_t static_bytes;
    rc = static_smem_bytes<operational_space_kernel<64>>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    const TileChoice c = osd_tile(prog, P, args.M, static_bytes);
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("operational-space dynamics needs %zu B of shared memory per CTA (> 227 KB) for one row (%d joints, %d links, M = %d)",
                  c.bytes + static_bytes, prog.n_dofs, prog.n_links, args.M);
        return DRMB200_ELIMIT;
    }
    const int64_t tiles = (batch + c.tile - 1) / c.tile;
#define DRM_LAUNCH_OSD(TT) \
    launch_kernel<operational_space_kernel<TT>>(tiles, TT, c.bytes, stream, false, "operational-space dynamics", prog, P, args)
    switch (c.tile) {
        case 64: return DRM_LAUNCH_OSD(64);
        case 32: return DRM_LAUNCH_OSD(32);
        case 16: return DRM_LAUNCH_OSD(16);
        case 8: return DRM_LAUNCH_OSD(8);
        case 4: return DRM_LAUNCH_OSD(4);
        case 2: return DRM_LAUNCH_OSD(2);
        default: return DRM_LAUNCH_OSD(1);
    }
#undef DRM_LAUNCH_OSD
}

}  // namespace drm
