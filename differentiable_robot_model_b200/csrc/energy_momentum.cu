// energy_momentum.cu -- whole-body quantities of a batch of configurations in one launch (sm_90a): kinetic and potential
// energy, the generalized momentum p = H(q) qd, the centre of mass, its velocity and its Jacobian (definitions in
// include/drm_b200.h).
//
// With (R_i, p_i) link i's world pose, (w_i, v_i) its body-frame velocity and (f_lin, f_ang) = I_i V_i its body-frame
// spatial momentum (f_lin = m v + w x mc, f_ang = I_o w + mc x v), every link contributes, in the world frame,
//   mass m_i,  first moment h_i = m_i p_i + R_i mc_i,  linear momentum L_i = R_i f_lin,
//   angular momentum about the world origin A_i = R_i f_ang + p_i x L_i.
// Summed over the subtree sub(j) of a movable joint j (world axis z_j, origin p_j) they give
//   momentum[dof(j)] = z_j . (A_sub - p_j x L_sub),     J_com[:, dof(j)] = z_j x (h_sub - m_sub p_j) / M,
// and summed over the whole tree the energies, the CoM (h / M) and its velocity (L / M).
//
// Mapping: one THREAD per configuration, on the unfolded tree.
//   * root -> leaves: the walk of kinematic_state.cu (TreeProgram in document order, canonical +z joint frames, branch
//     state (R, p, w, v) spilled to slots).  Kinetic energy, M, h and L accumulate in registers; each link leaves
//     (m, h, L, A, z, p) -- 16 floats -- in its slot-major shared-memory record.
//   * leaves -> root, in reverse document order (parent[i] < i): a link's record already holds its descendants' sums when
//     it is reached; a movable link writes its momentum and J_com column, then every link adds (m, h, L, A) into its
//     parent's record.
// The outputs are staged slot-major in shared memory and leave with a cooperative transposing copy (consecutive threads
// store consecutive floats).  T (rows per CTA) is the largest of 64, 32, ..., 1 with which two CTAs fit an SM.
// Everything the position-only outputs (potential, com, com_jacobian) depend on is computed by the same instructions
// with or without qd, so they are bit-identical either way.
//
// Algorithmic HBM bytes per configuration: 8n in (4n without qd), 4 (8 + 4n) out.
#include "launch.cuh"

namespace drm {

constexpr int EM_REC = 16;           // per-link record: m, h (3), L (3), A (3), z (3), p (3)
constexpr int EM_STATE = 18;         // spilled branch state: R (9), p, w, v

struct EmArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;     // null: zero velocity (no velocity-dependent output is requested)
    float* __restrict__ kinetic;      // [B] or null
    float* __restrict__ potential;    // [B] or null
    float* __restrict__ momentum;     // [B, n] or null
    float* __restrict__ com;          // [B, 3] or null
    float* __restrict__ com_velocity; // [B, 3] or null
    float* __restrict__ com_jacobian; // [B, 3, n] or null
    int64_t batch;
    int32_t aligned;
};

struct EmSmemLayout {
    int q, qd, table, slots, rec, kin, pot, mom, com, comv, jcom, total_floats;
    __host__ __device__ static int up4(int x) { return (x + 3) & ~3; }       // 16-byte aligned regions
    __host__ __device__ EmSmemLayout(int T, int n, int n_links, int n_slots) {
        int o = 0;
        q = o;     o += up4(T * n);
        qd = o;    o += up4(T * n);
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        slots = o; o += n_slots * EM_STATE * T;
        rec = o;   o += n_links * EM_REC * T;
        kin = o;   o += T;
        pot = o;   o += T;
        mom = o;   o += n * T;
        com = o;   o += 3 * T;
        comv = o;  o += 3 * T;
        jcom = o;  o += 3 * n * T;
        total_floats = o;
    }
};

__global__ void __launch_bounds__(64)
energy_momentum_kernel(const __grid_constant__ TreeProgram prog, const EmArgs args) {
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs, N = prog.n_links;
    const int T = blockDim.x;
    const EmSmemLayout L(T, n, N, prog.n_slots);
    const bool with_vel = args.qd != nullptr;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, args.batch - tile_start);
    const bool vec_in = args.aligned && ((tile_start * n) & 3) == 0;     // each tile checks its own global range
    coop_copy(smem + L.q, args.q + tile_start * n, valid * n, vec_in);
    if (with_vel) coop_copy(smem + L.qd, args.qd + tile_start * n, valid * n, vec_in);
    stage_canonical_table(smem + L.table, args.table, prog, T);
    __syncthreads();

    if (tid < valid) {
        const float* qrow = smem + L.q + tid * n;
        const float* qdrow = smem + L.qd + tid * n;
        const float* s_tab = smem + L.table;
        float* slot0 = smem + L.slots + tid;
        float* rec0 = smem + L.rec + tid;

        // ---- root -> leaves ----
        const V3 zero = v3(0.f, 0.f, 0.f);
        const LinkRow root = load_row(s_tab);          // the root's frame is the world frame, at rest
        float mass = root.m, kin2 = 0.f;               // kin2 = 2 x kinetic energy
        V3 h = root.mc, lin_sum = zero;
        M3 R = identity3();
        V3 p = zero, w = zero, v = zero;
        for (int i = 1; i < N; ++i) {
            const LinkRow row = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
            const int src = prog.psrc[i];
            M3 Rp; V3 pp, wp, vp;
            if (src == 0) { Rp = R; pp = p; wp = w; vp = v; }
            else if (src < 0) { Rp = identity3(); pp = wp = vp = zero; }
            else {
                const float* sl = slot0 + (src - 1) * EM_STATE * T;
                Rp = ldm(sl, T); pp = ldv(sl + 9 * T, T); wp = ldv(sl + 12 * T, T); vp = ldv(sl + 15 * T, T);
            }
            p = mul_add(Rp, row.r, pp);
            M3 M = row.F;
            const int c = prog.dof[i];
            float qd_k = 0.f;
            if (c >= 0) {
                float sn, cs;
                sincos_pi2(qrow[c], sn, cs);
                rotate_z(M, cs, sn);
                if (with_vel) qd_k = qdrow[c];
            }
            R = mul(Rp, M);
            v = mulT(M, cross_add(wp, row.r, vp));      // v_i = E (v_p + w_p x r)
            w = mulT(M, wp); w.z += qd_k;               // w_i = E w_p + (0, 0, qd)
            const int sv = prog.save[i];
            if (sv >= 0) {
                float* sl = slot0 + sv * EM_STATE * T;
                stm(sl, T, R); stv(sl + 9 * T, T, p); stv(sl + 12 * T, T, w); stv(sl + 15 * T, T, v);
            }

            const V3 f_lin = cross_add(w, row.mc, row.m * v);             // m v + w x mc
            const V3 f_ang = cross_add(row.mc, v, mul(row.Io, w));        // I_o w + mc x v
            kin2 += dot(v, f_lin) + dot(w, f_ang);
            const V3 cw = mul(R, row.mc);
            const V3 hi = v3(fmaf(row.m, p.x, cw.x), fmaf(row.m, p.y, cw.y), fmaf(row.m, p.z, cw.z));
            const V3 Li = mul(R, f_lin);
            const V3 Ai = cross_add(p, Li, mul(R, f_ang));
            mass += row.m;
            h = h + hi;
            lin_sum = lin_sum + Li;
            float* rc = rec0 + i * EM_REC * T;
            rc[0] = row.m;
            stv(rc + T, T, hi); stv(rc + 4 * T, T, Li); stv(rc + 7 * T, T, Ai);
            stv(rc + 10 * T, T, col2(R)); stv(rc + 13 * T, T, p);
        }

        const bool massive = mass != 0.f;
        const float inv_mass = massive ? 1.f / mass : 0.f;
        smem[L.kin + tid] = 0.5f * kin2;
        smem[L.pot + tid] = 9.81f * h.z;
        stv(smem + L.com + tid, T, massive ? inv_mass * h : zero);
        stv(smem + L.comv + tid, T, massive ? inv_mass * lin_sum : zero);

        // ---- leaves -> root ----
        float* mom = smem + L.mom + tid;
        float* jcom = smem + L.jcom + tid;
        for (int k = 0; k < n; ++k) { mom[k * T] = 0.f; jcom[k * T] = 0.f; jcom[(n + k) * T] = 0.f; jcom[(2 * n + k) * T] = 0.f; }
        for (int i = N - 1; i >= 1; --i) {
            const float* rc = rec0 + i * EM_REC * T;
            const float ms = rc[0];
            const V3 hs = ldv(rc + T, T), Ls = ldv(rc + 4 * T, T), As = ldv(rc + 7 * T, T);
            const int c = prog.dof[i];
            if (c >= 0) {
                const V3 z = ldv(rc + 10 * T, T), pj = ldv(rc + 13 * T, T);
                mom[c * T] = dot(z, As - cross(pj, Ls));
                const V3 jc = cross(z, hs - ms * pj);
                if (massive) stv(jcom + c * T, n * T, inv_mass * jc);
            }
            const int par = prog.parent[i];
            if (par > 0) {
                float* pr = rec0 + par * EM_REC * T;
                pr[0] += ms;
                stv(pr + T, T, ldv(pr + T, T) + hs);
                stv(pr + 4 * T, T, ldv(pr + 4 * T, T) + Ls);
                stv(pr + 7 * T, T, ldv(pr + 7 * T, T) + As);
            }
        }
    }
    __syncthreads();
    if (args.kinetic != nullptr) store_transposed(args.kinetic + tile_start, smem + L.kin, 1, valid, T);
    if (args.potential != nullptr) store_transposed(args.potential + tile_start, smem + L.pot, 1, valid, T);
    if (args.momentum != nullptr) store_transposed(args.momentum + tile_start * n, smem + L.mom, n, valid, T);
    if (args.com != nullptr) store_transposed(args.com + tile_start * 3, smem + L.com, 3, valid, T);
    if (args.com_velocity != nullptr) store_transposed(args.com_velocity + tile_start * 3, smem + L.comv, 3, valid, T);
    if (args.com_jacobian != nullptr) store_transposed(args.com_jacobian + tile_start * 3 * n, smem + L.jcom, 3 * n, valid, T);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// the largest power-of-two tile <= 64 rows while two CTAs still fit an SM, else down to one row per CTA
static TileChoice energy_momentum_tile(const TreeProgram& prog, size_t static_bytes) {
    return tile_ladder([&](int T) {
        return (size_t)EmSmemLayout(T, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float);
    }, static_bytes);
}

int energy_momentum_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd, int64_t batch,
                           float* kinetic, float* potential, float* momentum, float* com, float* com_velocity,
                           float* com_jacobian, cudaStream_t stream) {
    int rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);
    if (cp == nullptr) return rc;
    const TreeProgram& prog = cp->full;          // every link's own pose and inertia: never folded
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (kinetic == nullptr && potential == nullptr && momentum == nullptr && com == nullptr && com_velocity == nullptr &&
        com_jacobian == nullptr)
        return DRMB200_OK;
    if (batch == 0) return DRMB200_OK;
    // q and qd may be null only for a model without movable joints (empty tensors): they are then never read
    if (table == nullptr || (prog.n_dofs > 0 && q == nullptr)) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    const bool need_qd = kinetic != nullptr || momentum != nullptr || com_velocity != nullptr;
    if (need_qd && prog.n_dofs > 0 && qd == nullptr) {
        set_error("kinetic energy, momentum or CoM velocity requested without qd");
        return DRMB200_EINVAL;
    }

    EmArgs args;
    args.table = table; args.q = q; args.qd = need_qd && prog.n_dofs > 0 ? qd : nullptr;
    args.kinetic = kinetic; args.potential = potential; args.momentum = momentum; args.com = com;
    args.com_velocity = com_velocity; args.com_jacobian = com_jacobian;
    args.batch = batch;
    args.aligned = aligned16(q, args.qd);

    constexpr auto kern = energy_momentum_kernel;
    size_t static_bytes;
    rc = static_smem_bytes<kern>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    const TileChoice c = energy_momentum_tile(prog, static_bytes);
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("energy and momentum need %zu B of shared memory per CTA (> 227 KB) for one row (%d joints, %d links)",
                  c.bytes + static_bytes, prog.n_dofs, prog.n_links);
        return DRMB200_ELIMIT;
    }
    return launch_kernel<kern>((batch + c.tile - 1) / c.tile, c.tile, c.bytes, stream, false, "energy and momentum", prog, args);
}

}  // namespace drm
