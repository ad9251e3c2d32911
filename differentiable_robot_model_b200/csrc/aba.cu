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
#include "aba_body.cuh"
#include "launch.cuh"

namespace drm {

struct AbaArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ f;
    float* __restrict__ qdd;
    int64_t batch;
    uint32_t flags;
    int32_t aligned;
    float h;                        // IMPLICIT: the step of the implicit damping
};

// The kernel's body, instantiated by aba_kernel and aba_implicit_kernel (IMPLICIT: implicit damping of step args.h)
template <int T, bool IMPLICIT>
__device__ __forceinline__ void aba_run(const TreeProgram& prog, const FoldProgram& fold, const AbaArgs args) {
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

    if (tid < valid)
        aba_body<T, IMPLICIT>(prog, s_tab, s_q + tid * n, s_qd + tid * n, s_f + tid * n, s_qdd + tid * n, s_link + tid,
                              s_slot + tid, args.flags, args.h);

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

template <int T>
__global__ void __launch_bounds__(T)
aba_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const AbaArgs args) {
    aba_run<T, false>(prog, fold, args);
}

template <int T>
__global__ void __launch_bounds__(T)
aba_implicit_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const AbaArgs args) {
    aba_run<T, true>(prog, fold, args);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int forward_dynamics_device_impl(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                       const float* f, int64_t batch, uint32_t flags, float* qdd, cudaStream_t stream,
                                       bool prefolded, float dt) {
    FoldChoice fc;
    const int rc = select_fold(topo, prefolded, &fc);
    if (rc != DRMB200_OK) return rc;
    const TreeProgram& prog = *fc.prog;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || f == nullptr || qdd == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }

    AbaArgs args;
    args.table = table; args.q = q; args.qd = qd; args.f = f; args.qdd = qdd; args.batch = batch; args.flags = flags;
    args.h = dt;
    args.aligned = aligned16(q, qd, f, qdd);

    // 64 configurations per CTA unless the model's per-link state would leave a single CTA per SM
    const TileChoice c = tile_64_or_32([&](int T) {
        return (size_t)AbaSmemLayout(T, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float);
    });
    if (c.bytes > SMEM_CTA_MAX) { set_error("model needs %zu B of shared memory per CTA (> 227 KB)", c.bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (batch + c.tile - 1) / c.tile;
    if (flags & DRMB200_IMPLICIT_DAMPING)
        return c.tile == 64 ? launch_kernel<aba_implicit_kernel<64>>(tiles, 64, c.bytes, stream, false, "aba", prog, fc.fold, args)
                            : launch_kernel<aba_implicit_kernel<32>>(tiles, 32, c.bytes, stream, false, "aba", prog, fc.fold, args);
    return c.tile == 64 ? launch_kernel<aba_kernel<64>>(tiles, 64, c.bytes, stream, false, "aba", prog, fc.fold, args)
                        : launch_kernel<aba_kernel<32>>(tiles, 32, c.bytes, stream, false, "aba", prog, fc.fold, args);
}

int forward_dynamics_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                            const float* f, int64_t batch, uint32_t flags, float* qdd, cudaStream_t stream) {
    return forward_dynamics_device_impl(topo, table, q, qd, f, batch, flags & ~DRMB200_IMPLICIT_DAMPING, qdd, stream, false,
                                        0.f);
}
int forward_dynamics_prefolded_device(const drmb200_topology_t* topo, const float* folded, const float* q, const float* qd,
                                      const float* f, int64_t batch, uint32_t flags, float* qdd, cudaStream_t stream) {
    return forward_dynamics_device_impl(topo, folded, q, qd, f, batch, flags & ~DRMB200_IMPLICIT_DAMPING, qdd, stream, true,
                                        0.f);
}
int forward_dynamics_implicit_damping_device(const drmb200_topology_t* topo, const float* table, const float* q,
                                             const float* qd, const float* f, int64_t batch, uint32_t flags, float dt,
                                             float* qdd, cudaStream_t stream) {
    flags |= DRMB200_IMPLICIT_DAMPING;
    const int rc = check_implicit_damping(flags, dt);
    if (rc != DRMB200_OK) return rc;
    return forward_dynamics_device_impl(topo, table, q, qd, f, batch, flags, qdd, stream, false, dt);
}

}  // namespace drm
