// backward.cu -- analytic reverse-mode kernels for FK/Jacobian and RNEA (sm_90a).
//
// The reference differentiates its per-link op graph with torch autograd (about 7 k graph nodes for one
// Kuka RNEA).  Here each backward is ONE launch that re-walks the chain / tree per configuration and
// evaluates the adjoint recursions of SURVEY.md Appendix B; the exact recursions (same order, same
// intermediate quantities) are stated in executable form in oracle/adjoint_proto.py and verified there
// against autograd of the fp64 oracle.  Like the forward kernels they work in the canonical joint
// frames of drm_common.cuh (every joint a +z rotation), and map the table gradient back through the
// inverse signed permutation when it is written out.
//
// Outputs:
//   * gradients w.r.t. the per-configuration inputs (q, qd, qdd): one row per configuration, staged in
//     shared memory and streamed out exactly like the forward outputs;
//   * the gradient of the link table [n_links, 28]: a SUM OVER THE BATCH.  Per link, every thread of a
//     CTA drops its partial values into a padded shared-memory scratch matrix, the warps reduce its rows
//     with shuffles into a per-CTA accumulator (deterministic order), CTAs are persistent over tiles, and
//     each CTA writes one [n_links, 28] partial to a workspace that a second tiny kernel sums in fixed
//     order -- no atomics, bitwise reproducible.
//
// Nothing per-link is saved by the forward kernels (that would add >= 15 floats per link per
// configuration of HBM traffic); everything is recomputed here from q, qd, qdd.
#include "backward_common.cuh"

namespace drm {

// =============================================================================================
// FK + Jacobian backward
// =============================================================================================
struct FkBwdArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ g_pos;
    const float* __restrict__ g_quat;
    const float* __restrict__ g_jl;
    const float* __restrict__ g_ja;
    float* __restrict__ q_grad;
    float* __restrict__ partials;        // [gridDim.x, n_links * 28] or null
    int64_t batch;
    int32_t n_links;
    int32_t vec_ok;
};

struct FkBwdSmem {
    int q, qg, gpos, gquat, gjl, gja, table, link, scratch, acc, total_floats;
    __host__ __device__ FkBwdSmem(int tile, int n, int len) {
        int o = 0;
        gquat = o; o += tile * 4;
        q = o; o += tile * n;
        qg = o; o += tile * n;
        gpos = o; o += tile * 3;
        gjl = o; o += tile * 3 * n;
        gja = o; o += tile * 3 * n;
        table = o; o += len * 12;
        link = o; o += len * 2 * tile;                   // per path link: cos, sin -- slot-major (R~, p are re-derived)
        scratch = o; o += block_accumulate_floats(12, tile);
        acc = o; o += len * 12;                          // canonical (F~, r~) gradient per path link
        total_floats = o;
    }
};

template <bool NEED_TABLE, int T>
__global__ void __launch_bounds__(T)
fk_jacobian_backward_kernel(const __grid_constant__ PathProgram prog, const FkBwdArgs args) {
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs, len = prog.len;
    const FkBwdSmem L(T, n, len);
    float* s_q = smem + L.q;
    float* s_qg = smem + L.qg;
    float* s_gpos = smem + L.gpos;
    float* s_gquat = smem + L.gquat;
    float* s_gjl = smem + L.gjl;
    float* s_gja = smem + L.gja;
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_scr = smem + L.scratch;
    float* s_acc = smem + L.acc;
    const int tid = threadIdx.x;
    const bool vec_ok = args.vec_ok;

    for (int i = tid; i < len * 12; i += T) {
        const int k = i / 12, e = i - k * 12;
        int src;
        const float sg = canon_map(e, prog.paxis[k], prog.axis[k], src);
        s_tab[i] = sg * __ldg(args.table + (int)prog.link[k] * DRMB200_TABLE_STRIDE + src);
        if (NEED_TABLE) s_acc[i] = 0.f;
    }

    const int64_t n_tiles = (args.batch + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t start = tile * T;
        const int valid = (int)min((int64_t)T, args.batch - start);
        __syncthreads();                                    // previous tile fully consumed
        coop_copy(s_q, args.q + start * n, valid * n, vec_ok);
        tile_load_or_zero(s_gpos, args.g_pos ? args.g_pos + start * 3 : nullptr, valid * 3, T * 3, vec_ok);
        tile_load_or_zero(s_gquat, args.g_quat ? args.g_quat + start * 4 : nullptr, valid * 4, T * 4, vec_ok);
        tile_load_or_zero(s_gjl, args.g_jl ? args.g_jl + start * 3 * n : nullptr, valid * 3 * n, T * 3 * n, vec_ok);
        tile_load_or_zero(s_gja, args.g_ja ? args.g_ja + start * 3 * n : nullptr, valid * 3 * n, T * 3 * n, vec_ok);
        for (int i = tid; i < T * n; i += T) s_qg[i] = 0.f;
        __syncthreads();

        const bool active = tid < valid;
        const float* qrow = s_q + tid * n;
        const float* gl = s_gjl + tid * 3 * n;
        const float* ga = s_gja + tid * 3 * n;
        float* lk = s_link + tid;

        // ---- forward recompute along the path; keep R~_k, p_k, (cos, sin) in smem ----------------
        M3 R = identity3();
        V3 p = v3(0.f, 0.f, 0.f);
        V3 pbar = v3(s_gpos[tid * 3], s_gpos[tid * 3 + 1], s_gpos[tid * 3 + 2]);
        for (int k = 0; k < len; ++k) {
            M3 F; V3 r;
            load_Fr(s_tab + k * 12, F, r);
            p = mul_add(R, r, p);
            R = mul(R, F);
            const int c = prog.dof[k];
            float cs = 1.f, sn = 0.f;
            if (c >= 0) {
                sincos_pi2(qrow[c], sn, cs);
                const V3 g = v3(gl[c], gl[n + c], gl[2 * n + c]);
                pbar = cross_add(g, col2(R), pbar);         // adjoint of p_ee: J_lin = z x (p_ee - p_i)
                rotate_z(R, cs, sn);
            }
            float* s = lk + k * 2 * T;
            s[0] = cs; s[T] = sn;
        }
        const V3 p_ee = p;
        const float4 gq = reinterpret_cast<const float4*>(s_gquat)[tid];
        M3 Rbar = permute_cols_adjoint(quat_backward(unpermute_cols(R, prog.ee_axis), gq), prog.ee_axis);

        // ---- reverse sweep ee -> root ------------------------------------------------------------
        // The chain is walked back DOWN in registers: R~_{k-1} = R~_k M_k^T and p_{k-1} = p_k - R~_{k-1} r_k (M_k is
        // orthogonal), so only (cos, sin) per link live in shared memory -- 2 floats instead of 14 per link, which
        // is what bounds the occupancy of this kernel.  The re-derived poses differ from the forward ones by rounding.
        M3 Rk = R;                                          // R~_k of the link being processed
        V3 pk = p;
        for (int k = len - 1; k >= 0; --k) {
            const float* s = lk + k * 2 * T;
            const float cs = s[0], sn = s[T];
            M3 F; V3 r;
            load_Fr(s_tab + k * 12, F, r);
            const int c = prog.dof[k];
            M3 M = F;
            if (c >= 0) rotate_z(M, cs, sn);
            const M3 RP = (k > 0) ? mulNT(Rk, M) : identity3();
            const V3 pP = (k > 0) ? pk - mul(RP, r) : v3(0.f, 0.f, 0.f);
            if (c >= 0) {
                const V3 z = col2(Rk);
                const V3 g = v3(gl[c], gl[n + c], gl[2 * n + c]);
                const V3 h = v3(ga[c], ga[n + c], ga[2 * n + c]);
                const V3 zbar = cross_add(p_ee - pk, g, h);   // d x G_l + G_a
                Rbar.a02 += zbar.x; Rbar.a12 += zbar.y; Rbar.a22 += zbar.z;    // z = R~_k e_z
                pbar = pbar - cross(g, z);                    // adjoint of p_k
            }
            const M3 Mbar = mulTN(RP, Rbar);
            const V3 rbar = mulT(RP, pbar);
            M3 Rbar_P = mulNT(Rbar, M);
            add_outer(Rbar_P, pbar, r);
            if (c >= 0) s_qg[tid * n + c] = theta_grad_z(Mbar, M);
            if (NEED_TABLE) {
                M3 Fbar = Mbar;
                if (c >= 0) rotate_z(Fbar, cs, -sn);          // Mbar Rz^T
                float vals[12];
                m3_to_array(Fbar, vals);
                vals[9] = rbar.x; vals[10] = rbar.y; vals[11] = rbar.z;
                block_accumulate<12, T>(s_scr, s_acc + k * 12, vals, active, [](int j) { return j; });
            }
            Rbar = Rbar_P;
            Rk = RP;
            pk = pP;
        }
        if (args.q_grad != nullptr) {
            __syncthreads();
            coop_copy(args.q_grad + start * n, s_qg, valid * n, vec_ok);
        }
    }
    if (NEED_TABLE) {
        __syncthreads();
        float* out = args.partials + (size_t)blockIdx.x * args.n_links * DRMB200_TABLE_STRIDE;
        for (int i = tid; i < args.n_links * DRMB200_TABLE_STRIDE; i += T) out[i] = 0.f;
        __syncthreads();
        for (int i = tid; i < len * 12; i += T) {            // canonical -> natural entries (bijection per row)
            const int k = i / 12, e = i - k * 12;
            int src;
            const float sg = canon_map(e, prog.paxis[k], prog.axis[k], src);
            out[(int)prog.link[k] * DRMB200_TABLE_STRIDE + src] = sg * s_acc[i];
        }
    }
}

// sums the per-CTA partial tables in fixed order and ADDS them to table_grad
__global__ void reduce_partials_kernel(const float* __restrict__ partials, int n_blocks, int n_entries,
                                       float* __restrict__ table_grad) {
    // one warp per table entry: lanes stride over the CTA partials (fixed assignment -> fixed summation order),
    // then a shuffle tree.  (One thread per entry looping over ~1000 partials took longer than the
    // single-sweep backward kernel it follows.)
    // launched as a programmatic dependent of the adjoint kernel before it on the stream (launch_reduce): its set-up
    // overlaps that kernel's tail, and this wait returns when that grid has completed and its partials are visible
    // (a no-op after an ordinary launch)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (e >= n_entries) return;
    float s = 0.f;
    for (int b = lane; b < n_blocks; b += 32) s += partials[(size_t)b * n_entries + e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) table_grad[e] += s;
}

int64_t table_grad_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    if (topo == nullptr || topo->n_links < 1 || topo->n_links > DRMB200_MAX_LINKS) return 0;
    int64_t tiles = (batch + 15) / 16;            // smallest tile the launchers may pick (backward_aba.cu)
    if (tiles < 1) tiles = 1;
    const int64_t grid = tiles < BWD_MAX_GRID ? tiles : BWD_MAX_GRID;
    return grid * topo->n_links * DRMB200_TABLE_STRIDE * (int64_t)sizeof(float);
}

int launch_reduce(const float* partials, int grid, const drmb200_topology_t* topo, float* table_grad,
                         cudaStream_t stream) {
    const int entries = topo->n_links * DRMB200_TABLE_STRIDE;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((entries * 32 + 255) / 256);
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, reduce_partials_kernel, partials, grid, entries, table_grad);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("reduce launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}


int fk_jacobian_backward_device(const drmb200_topology_t* topo, int32_t ee_link, const float* table, const float* q,
                                int64_t batch, const float* g_pos, const float* g_quat, const float* g_jl,
                                const float* g_ja, float* q_grad, float* table_grad, void* workspace,
                                cudaStream_t stream) {
    PathProgram prog;
    int rc = build_path_program(topo, ee_link, &prog);
    if (rc != DRMB200_OK) return rc;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || (q_grad == nullptr && table_grad == nullptr)) return DRMB200_OK;
    if (table == nullptr || q == nullptr) { set_error("table / q is null"); return DRMB200_EINVAL; }
    if (table_grad != nullptr && workspace == nullptr) { set_error("table_grad requested without workspace"); return DRMB200_EINVAL; }

    FkBwdArgs args;
    args.table = table; args.q = q; args.g_pos = g_pos; args.g_quat = g_quat; args.g_jl = g_jl; args.g_ja = g_ja;
    args.q_grad = q_grad; args.partials = static_cast<float*>(workspace); args.batch = batch;
    args.n_links = topo->n_links;
    auto al16 = [](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    args.vec_ok = (al16(q) && al16(g_pos) && al16(g_quat) && al16(g_jl) && al16(g_ja) && al16(q_grad)) ? 1 : 0;

    int tile = 32, best_warps = 0;           // the tile that keeps the most warps resident per SM
    for (int t = 128; t >= 32; t >>= 1) {
        const size_t b = (size_t)FkBwdSmem(t, prog.n_dofs, prog.len).total_floats * sizeof(float) + 1024;
        const int warps = b > 227 * 1024 ? 0 : (int)((227 * 1024) / b) * (t / 32);
        if (warps > best_warps) { best_warps = warps; tile = t; }
    }
    const size_t smem_bytes = (size_t)FkBwdSmem(tile, prog.n_dofs, prog.len).total_floats * sizeof(float);
    if (smem_bytes > 227 * 1024) { set_error("fk backward needs %zu B of shared memory per CTA (> 227 KB)", smem_bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (batch + tile - 1) / tile;
    int grid = 0;
    const bool need_table = table_grad != nullptr;
#define DRM_LAUNCH_FKB(NT, TT)                                                                                  \
    do {                                                                                                        \
        rc = persistent_grid(fk_jacobian_backward_kernel<NT, TT>, TT, smem_bytes, tiles, &grid, "fk backward"); \
        if (rc != DRMB200_OK) return rc;                                                                        \
        fk_jacobian_backward_kernel<NT, TT><<<grid, TT, smem_bytes, stream>>>(prog, args);                      \
    } while (0)
    if (need_table) { if (tile == 128) DRM_LAUNCH_FKB(true, 128); else if (tile == 64) DRM_LAUNCH_FKB(true, 64); else DRM_LAUNCH_FKB(true, 32); }
    else            { if (tile == 128) DRM_LAUNCH_FKB(false, 128); else if (tile == 64) DRM_LAUNCH_FKB(false, 64); else DRM_LAUNCH_FKB(false, 32); }
#undef DRM_LAUNCH_FKB
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("fk backward launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return need_table ? launch_reduce(args.partials, grid, topo, table_grad, stream) : DRMB200_OK;
}

}  // namespace drm
