// dynamics_regressor.cu -- the batched joint-torque regressor of the inertial parameters (sm_90a):
//   Y [B, n, n_links, 14],  Y[b, i, l, k] = d tau_i / d table[l, 12 + k]
// for exactly what drmb200_inverse_dynamics evaluates (same table, flags, inputs).  tau is linear in every link's
// (I_o, mc, m) and in its damping, so  tau_i = sum_{l,k} Y[b, i, l, k] table[l, 12 + k]  for any table.
//
// Link l's body wrench in its canonical frame (rnea.cu),
//   f = w x (m v - mc x w) + (m a - mc x al),   n = w x (I_o w + mc x v) + v x (m v - mc x w) + I_o al + mc x a,
// reaches joint i (an ancestor-or-self of l, axis z_i and origin p_i in the world frame) as
//   tau_i += u . n + s . f,   u = R_l^T z_i,  s = R_l^T (z_i x (p_l - p_i))              (R_l, p_l: pose of link l)
// and u . n + s . f, written out per parameter, is
//   I_o[r][c] : (u x w)_r w_c + u_r al_c
//   mc        : v x (u x w) - w x (u x v) + a x u - w x (s x w) - al x s
//   m         : s . (a + w x v)
// Damping adds qd_i to column 13 of the link that owns joint i.  All other entries -- the root, links outside the subtree
// of joint i, fixed links' damping -- are exact zeros.
//
// Mapping: one THREAD per (configuration, link l).  The thread walks root -> l (the links of l's root path, document
// order), carrying the motion state (w, v, al, a) of rnea.cu pass 1 and the world pose (R, p) in the canonical +z joint
// frames of drm_common.cuh; every movable ancestor leaves (z_i, p_i) in the thread's own output slots of row i, which the
// emission pass reads back before it overwrites them.  The 13 canonical columns map back to the caller's table columns
// through canon_map (canonical entry e = sign * natural[src], so column src receives sign * column e).
// A CTA owns TC configurations x all n_links links (TC * n_links threads); its output is one contiguous [TC, n, L, 14]
// range, staged in shared memory and stored with one TMA bulk copy (cooperative copies for ragged or unaligned tiles).
// TC is the largest count (<= 128 / n_links) whose footprint stays under ~113 KB (two CTAs per SM); a model that needs
// more than 227 KB at TC = 1 is refused with DRMB200_ELIMIT.
//
// The regressor needs one column per table row, so it always walks the full (unfolded) tree.
//
// Algorithmic HBM bytes per configuration: 12n in, 56 n L out (84 B and 3528 B for the 7-DoF, 9-link Kuka).
#include "launch.cuh"

namespace drm {

constexpr int REG_COLS = 14;          // I_o 9 | mc 3 | m | damping

struct RegArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ qdd;
    float* __restrict__ Y;
    int64_t batch;
    uint32_t flags;
    int32_t aligned;
    int32_t tc;                          // configurations per CTA
};

struct RegSmemLayout {
    int in[3], out, table, total_floats;
    __host__ __device__ static int up4(int x) { return (x + 3) & ~3; }       // 16-byte aligned regions
    __host__ __device__ RegSmemLayout(int tc, int n, int n_links) {
        int o = 0;
        for (int k = 0; k < 3; ++k) { in[k] = o; o += up4(tc * n); }
        out = o; o += up4(tc * n * n_links * REG_COLS);
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        total_floats = o;
    }
};

// one thread: configuration rows qrow / qdrow / qddrow, link l; o points at Y[c, 0, l, 0] in the staged tile, rows of
// dof k at o + k * rs
__device__ __forceinline__ void regressor_body(const TreeProgram& prog, const float* s_tab, const float* qrow, const float* qdrow,
                                               const float* qddrow, int l, int n, float* o, int rs, uint32_t flags) {
    if (l == 0) {                                                         // the root's columns
        for (int k = 0; k < n; ++k)
            for (int e = 0; e < REG_COLS; ++e) o[k * rs + e] = 0.f;
        return;
    }
    uint64_t path = 0;                                                    // ancestors-or-self of l, root excluded
    for (int k = l; k > 0; k = prog.parent[k]) path |= 1ull << k;

    const float g = (flags & DRMB200_GRAVITY) ? 9.81f : 0.f;             // robot_model.py:347
    const V3 zero = v3(0.f, 0.f, 0.f);
    V3 w = zero, v = zero, al = zero, a = v3(0.f, 0.f, g), p = zero;
    M3 R = identity3();
    uint64_t dofs = 0;                                                    // dofs of the movable links on the path
    for (int i = 1; i <= l; ++i) {                                        // uniform loop, per-thread predicate
        if (!((path >> i) & 1ull)) continue;
        M3 M;
        V3 r;
        load_Fr(s_tab + i * DRMB200_TABLE_STRIDE, M, r);
        p = mul_add(R, r, p);                                             // p_i = p_p + R_p r~
        const int c = prog.dof[i];
        float qd_k = 0.f, qdd_k = 0.f;
        if (c >= 0) {
            float cs, sn;
            sincos_pi2(qrow[c], sn, cs);
            rotate_z(M, cs, sn);
            qd_k = qdrow[c];
            qdd_k = qddrow[c];
        }
        // rnea.cu pass 1: w = E w_p + qd e_z, v = E (v_p + w_p x r), al = E al_p + qdd e_z + w x qd e_z,
        // a = E (a_p + al_p x r) + v x qd e_z
        const V3 vn = mulT(M, cross_add(w, r, v)), an = mulT(M, cross_add(al, r, a));
        w = mulT(M, w); w.z += qd_k;
        al = mulT(M, al) + cross_z(w, qd_k); al.z += qdd_k;
        v = vn;
        a = an + cross_z(v, qd_k);
        R = mul(R, M);
        if (c >= 0) {                                                     // (z_i, p_i) wait in row c's slots
            float* rec = o + c * rs;
            rec[0] = R.a02; rec[1] = R.a12; rec[2] = R.a22; rec[3] = p.x; rec[4] = p.y; rec[5] = p.z;
            dofs |= 1ull << c;
        }
    }

    const int ci = prog.axis[l];
    const int own = prog.dof[l];
    const bool damp = (flags & DRMB200_DAMPING) != 0;
    const V3 awv = cross_add(w, v, a);                                    // a + w x v
    for (int k = 0; k < n; ++k) {
        float* ok = o + k * rs;
        if (!((dofs >> k) & 1ull)) {
            for (int e = 0; e < REG_COLS; ++e) ok[e] = 0.f;
            continue;
        }
        const V3 z = v3(ok[0], ok[1], ok[2]), pi = v3(ok[3], ok[4], ok[5]);
        const V3 u = mulT(R, z), s = mulT(R, cross(z, p - pi));
        const V3 uw = cross(u, w), uv = cross(u, v), sw = cross(s, w);
        const V3 gmc = cross(v, uw) - cross(w, uv) + cross(a, u) - cross(w, sw) - cross(al, s);
        float y[13];
        const float uwa[3] = {uw.x, uw.y, uw.z}, ua[3] = {u.x, u.y, u.z}, wa[3] = {w.x, w.y, w.z}, ala[3] = {al.x, al.y, al.z};
#pragma unroll
        for (int rr = 0; rr < 3; ++rr)
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) y[3 * rr + cc] = fmaf(uwa[rr], wa[cc], ua[rr] * ala[cc]);
        y[9] = gmc.x; y[10] = gmc.y; y[11] = gmc.z;
        y[12] = dot(s, awv);
#pragma unroll
        for (int e = 0; e < 12; ++e) {                                    // canonical I_o~, mc~ -> the caller's columns
            int src;
            const float sg = canon_map(12 + e, 0, ci, src);
            ok[src - 12] = sg * y[e];
        }
        ok[12] = y[12];
        ok[13] = (damp && k == own) ? qdrow[k] : 0.f;
    }
}

__global__ void dynamics_regressor_kernel(const __grid_constant__ TreeProgram prog, const RegArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = prog.n_dofs;
    const int N = prog.n_links;
    const int TC = args.tc;
    const RegSmemLayout L(TC, n, N);
    float* s_in0 = smem + L.in[0];
    float* s_in1 = smem + L.in[1];
    float* s_in2 = smem + L.in[2];
    float* s_out = smem + L.out;
    float* s_tab = smem + L.table;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * TC;
    const int valid = (int)min((int64_t)TC, args.batch - tile_start);
    // each tile checks the 16-byte alignment of its own global ranges
    const bool vec_in = args.aligned && ((tile_start * n) & 3) == 0;
    const bool bulk_in = vec_in && ((valid * n) & 3) == 0;
    const int per_row = n * N * REG_COLS;
    const int64_t out_off = tile_start * per_row;
    const int out_floats = valid * per_row;
    const bool vec_out = args.aligned && (out_off & 3) == 0;
    const bool bulk_out = vec_out && (out_floats & 3) == 0;

    if (bulk_in) {
        if (tid == 0) {
            mbar_init(&mbar, 1);
            fence_mbar_init();
            const uint32_t bytes = (uint32_t)valid * n * 4u;
            mbar_arrive_expect_tx(&mbar, 3u * bytes);
            bulk_g2s(s_in0, args.q + tile_start * n, bytes, &mbar);
            bulk_g2s(s_in1, args.qd + tile_start * n, bytes, &mbar);
            bulk_g2s(s_in2, args.qdd + tile_start * n, bytes, &mbar);
        }
    } else {
        coop_copy(s_in0, args.q + tile_start * n, valid * n, vec_in);
        coop_copy(s_in1, args.qd + tile_start * n, valid * n, vec_in);
        coop_copy(s_in2, args.qdd + tile_start * n, valid * n, vec_in);
    }
    stage_canonical_table(s_tab, args.table, prog, blockDim.x);
    __syncthreads();
    if (bulk_in) mbar_wait(&mbar, 0);

    const int lc = tid / N, l = tid - lc * N;
    if (lc < valid) {
        const int row = lc * n;
        regressor_body(prog, s_tab, s_in0 + row, s_in1 + row, s_in2 + row, l, n, s_out + lc * per_row + l * REG_COLS, N * REG_COLS,
                       args.flags);
    }

    if (bulk_out) {
        fence_proxy_async();
        __syncthreads();
        if (tid == 0) {
            bulk_s2g(args.Y + out_off, s_out, (uint32_t)out_floats * 4u);
            bulk_commit();
            bulk_wait_read<0>();
        }
    } else {
        __syncthreads();
        coop_copy(args.Y + out_off, s_out, out_floats, vec_out);
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// ~128 threads per CTA: TC = 128 / n_links configurations, fewer while the footprint would leave a single CTA per SM
static TileChoice regressor_tile(const TreeProgram& prog, size_t static_bytes) {
    const int N = prog.n_links;
    return tile_count_down(N >= 128 ? 1 : 128 / N, [&](int tc) {
        return (size_t)RegSmemLayout(tc, prog.n_dofs, N).total_floats * sizeof(float);
    }, static_bytes);
}

int dynamics_regressor_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd, const float* qdd,
                              int64_t batch, uint32_t flags, float* Y, cudaStream_t stream) {
    int rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);
    if (cp == nullptr) return rc;
    const TreeProgram& prog = cp->full;          // one column per table row: never folded
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || qdd == nullptr || Y == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    RegArgs args;
    args.table = table; args.q = q; args.qd = qd; args.qdd = qdd; args.Y = Y;
    args.batch = batch; args.flags = flags & (DRMB200_GRAVITY | DRMB200_DAMPING);
    args.aligned = aligned16(q, qd, qdd, Y);

    constexpr auto kern = dynamics_regressor_kernel;
    size_t static_bytes;
    rc = static_smem_bytes<kern>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    const TileChoice c = regressor_tile(prog, static_bytes);
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("model needs %zu B of shared memory per CTA (> 227 KB) for its dynamics regressor", c.bytes + static_bytes);
        return DRMB200_ELIMIT;
    }
    args.tc = c.tile;
    return launch_kernel<kern>((batch + c.tile - 1) / c.tile, c.tile * prog.n_links, c.bytes, stream, false, "dynamics regressor",
                               prog, args);
}

}  // namespace drm
