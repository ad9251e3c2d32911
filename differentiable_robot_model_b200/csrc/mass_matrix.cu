// mass_matrix.cu -- batched joint-space inertia matrix H(q) [B, n, n] in ONE launch (sm_90a).
//
// Replaces DifferentiableRobotModel.compute_lagrangian_inertia_matrix (robot_model.py:403-450), which evaluates
// compute_inverse_dynamics n + 1 times (column j = ID(q, 0, e_j) - ID(q, 0, 0), every evaluation a full walk of the
// per-link op graph).  The difference cancels gravity (and damping acts on qd = 0), so column j is exactly the RNEA
// torque for zero velocity, zero gravity and unit acceleration of joint j; the kernel evaluates those n columns
// inside one launch, one thread per configuration, in the canonical joint frames of drm_common.cuh:
//     (cos, sin) of every joint once                                   (n sincos instead of n (n + 1))
//     column j:  al_i = E al_p + e_z [i = j],  a_i = E (a_p + al_p x r)          (zero above the subtree of j)
//                f_i = m a_i - mc x al_i,  n_i = Io al_i + mc x a_i             (no velocity terms)
//                leaves -> root:  f_p += M f_i,  n_p += r x (M f_i) + M n_i,  H[dof(i), j] = n_i.z
// The (al | a) pair goes through E = Rz^T F~^T as f32x2 pair (drm_common.cuh).  H is staged in shared memory in
// its global row-major layout and leaves as one TMA bulk store per tile.
//
// Algorithmic HBM bytes per configuration: 4n in + 4n^2 out (224 B at n = 7); about 1 k instructions per column and
// 7-DoF configuration, FP32-issue-bound like RNEA.
#include "launch.cuh"

namespace drm {

struct MmArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    float* __restrict__ H;
    int64_t batch;
    int32_t aligned;
};

struct MmSmemLayout {
    int q, H, table, link, slots, total_floats;
    __host__ __device__ MmSmemLayout(int T, int n, int n_links, int n_slots) {
        int o = 0;
        H = o;  o += T * n * n;                    // 16-byte aligned rows first (T multiple of 4)
        q = o;  o += T * n;
        o = (o + 3) & ~3;
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o;  o += n_links * 8 * T;           // per link: f(3) n(3) cos sin, slot-major
        slots = o; o += n_slots * 6 * T;           // branch-point acceleration states
        total_floats = o;
    }
};

template <int T>
__global__ void __launch_bounds__(T)
mass_matrix_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const MmArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = prog.n_dofs;
    const int N = prog.n_links;
    const MmSmemLayout L(T, n, N, prog.n_slots);
    float* s_q = smem + L.q;
    float* s_H = smem + L.H;
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
            mbar_arrive_expect_tx(&mbar, bytes);
            bulk_g2s(s_q, args.q + tile_start * n, bytes, &mbar);
        }
    } else {
        coop_copy(s_q, args.q + tile_start * n, valid * n, vec_ok);
    }
    // fold.n_red > 0: fixed links folded into their movable ancestors, prog is the reduced tree (drm_common.cuh)
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
        float* hrow = s_H + tid * n * n;
        float* lk0 = s_link + tid;
        float* sl0 = s_slot + tid;
        const V3 zero = v3(0.f, 0.f, 0.f);

        // joint rotations, once
        for (int i = 1; i < N; ++i) {
            const int c = prog.dof[i];
            float cs = 1.f, sn = 0.f;
            if (c >= 0) sincos_pi2(qrow[c], sn, cs);
            lk0[(i * 8 + 6) * T] = cs; lk0[(i * 8 + 7) * T] = sn;
        }

        for (int j = 1; j < N; ++j) {
            const int cj = prog.dof[j];
            if (cj < 0) continue;

            // ---- root -> leaves: accelerations for a unit acceleration of joint j, body wrenches ----------
            for (int i = 1; i < j; ++i) {                       // nothing above / beside the subtree of j moves
                float* lk = lk0 + i * 8 * T;
                stv(lk, T, zero); stv(lk + 3 * T, T, zero);
            }
            V3P X = pk3(zero, zero);                            // (al | a) of the previously processed link
            for (int i = j; i < N; ++i) {
                const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
                float* lk = lk0 + i * 8 * T;
                const int P = prog.parent[i];
                const int src = prog.psrc[i];
                V3 alp = zero, ap = zero;
                if (P >= j) {                                    // parents outside the subtree carry no acceleration
                    if (src == 0) upk3(X, alp, ap);
                    else if (src > 0) { const float* sl = sl0 + (src - 1) * 6 * T; alp = ldv(sl, T); ap = ldv(sl + 3 * T, T); }
                }
                X = rotzT_p(mulT_p(C.F, pk3(alp, cross_add(alp, C.r, ap))), lk[6 * T], lk[7 * T]);
                V3 al, a;
                upk3(X, al, a);
                if (i == j) { al.z += 1.f; X = pk3(al, a); }
                stv(lk, T, C.m * a - cross(C.mc, al));                             // f_i
                stv(lk + 3 * T, T, mul_add(C.Io, al, cross(C.mc, a)));             // n_i
                const int sv = prog.save[i];
                if (sv >= 0) { float* sl = sl0 + sv * 6 * T; stv(sl, T, al); stv(sl + 3 * T, T, a); }
            }

            // ---- leaves -> root: wrench propagation, column j of H ------------------------------------------
            for (int i = N - 1; i >= 1; --i) {
                float* lk = lk0 + i * 8 * T;
                const V3 f = ldv(lk, T), nn = ldv(lk + 3 * T, T);
                const int c = prog.dof[i];
                if (c >= 0) hrow[c * n + cj] = nn.z;
                const int P = prog.parent[i];
                if (P > 0) {
                    M3 F; V3 r;
                    load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, F, r);
                    V3 fp, np;
                    upk3(mul_pv(F, rotz_p(pk3(f, nn), lk[6 * T], lk[7 * T])), fp, np);
                    np = cross_add(r, fp, np);
                    float* pk = lk0 + P * 8 * T;
                    stv(pk, T, ldv(pk, T) + fp);
                    stv(pk + 3 * T, T, ldv(pk + 3 * T, T) + np);
                }
            }
        }
    }

    if (bulk) {
        fence_proxy_async();
        __syncthreads();
        if (tid == 0) {
            bulk_s2g(args.H + tile_start * n * n, s_H, (uint32_t)valid * n * n * 4u);
            bulk_commit();
            bulk_wait_read<0>();
        }
    } else {
        __syncthreads();
        coop_copy(args.H + tile_start * n * n, s_H, valid * n * n, vec_ok);
    }
}

// prefolded: `table` holds the rows of drmb200_fold_link_table (constant models fold once instead of once per CTA)
int mass_matrix_device_impl(const drmb200_topology_t* topo, const float* table, const float* q, int64_t batch, float* H,
                            cudaStream_t stream, bool prefolded) {
    FoldChoice fc;
    const int rc = select_fold(topo, prefolded, &fc);
    if (rc != DRMB200_OK) return rc;
    const TreeProgram& prog = *fc.prog;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr || H == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    MmArgs args;
    args.table = table; args.q = q; args.H = H; args.batch = batch;
    args.aligned = aligned16(q, H);
    const TileChoice c = tile_64_or_32([&](int T) {
        return (size_t)MmSmemLayout(T, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float);
    });
    if (c.bytes > SMEM_CTA_MAX) { set_error("model needs %zu B of shared memory per CTA (> 227 KB)", c.bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (batch + c.tile - 1) / c.tile;
    return c.tile == 64 ? launch_kernel<mass_matrix_kernel<64>>(tiles, 64, c.bytes, stream, false, "mass matrix", prog, fc.fold, args)
                        : launch_kernel<mass_matrix_kernel<32>>(tiles, 32, c.bytes, stream, false, "mass matrix", prog, fc.fold, args);
}

int mass_matrix_device(const drmb200_topology_t* topo, const float* table, const float* q, int64_t batch, float* H, cudaStream_t stream) {
    return mass_matrix_device_impl(topo, table, q, batch, H, stream, false);
}
int mass_matrix_prefolded_device(const drmb200_topology_t* topo, const float* folded, const float* q, int64_t batch, float* H,
                                 cudaStream_t stream) {
    return mass_matrix_device_impl(topo, folded, q, batch, H, stream, true);
}

}  // namespace drm
