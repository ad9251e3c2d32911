// inverse_kinematics.cu -- batched damped least-squares (Levenberg-Marquardt) inverse kinematics (sm_90a).
//
// One thread per row (a start configuration and a pose target), all iterations inside ONE launch.  The reference has no
// IK; users otherwise loop FK + Jacobian + an optimiser step in Python.  Every row runs, in fp32 (spec in DESIGN.md §3):
//
//   q <- clamp(q0, lower, upper); lambda <- damping_in[b] or damping_init; evaluate (p, R, J) at q
//   repeat max_iters times while the row is not done:
//       A = J J^T + lambda I (6x6 pose / 3x3 position); Cholesky; a pivot <= 0 or not finite rejects the step
//       q' = clamp(q + J^T A^-1 e); evaluate at q'
//       E' < E: accept (q, J, e, E <- trial), lambda <- max(lambda / 2, IK_LAMBDA_MIN)
//       else:   reject, lambda <- min(4 lambda, IK_LAMBDA_MAX)
//
// "evaluate" walks the root -> ee path in the canonical +z frames of drm_common.cuh (the path program and signed table
// gather of fk_jacobian.cu) and returns the error e = (p* - p, rotvec(quat* (x) conj(quat(R)))), E = |e|^2.  It has ONE
// call site (the initial evaluation is iteration "-1" of the same loop), so the arithmetic of an evaluation does not
// depend on where it happens: K iterations in one call are bit-identical to K chained calls of max_iters = 1.
//
// Shared memory, slot-major (element e of row t at base[e * TILE + t]: conflict-free for any n):
//   per row  q[2][n], J[2][6][n] (current / trial, swapped by an index on accept), target (p*, quat*) 7 floats
//   per CTA  the canonical path rows (12 floats per path link) and the joint limits 2n
// A, its Cholesky factor, e and y stay in registers.  HBM traffic per row is 4n + 28 B in and 4n + 13 B out, independent
// of max_iters: the kernel is arithmetic-bound.
#include <cmath>
#include "ik_common.cuh"
#include "launch.cuh"

namespace drm {

struct IkArgs {
    const float* __restrict__ table;       // [n_links, 28]
    const float* __restrict__ q0;          // [B, n]
    const float* __restrict__ tpos;        // [B, 3]
    const float* __restrict__ tquat;       // [B, 4] xyzw, or null (position only)
    const float* __restrict__ lower;       // [n] or null
    const float* __restrict__ upper;       // [n] or null
    const float* __restrict__ damping_in;  // [B] or null
    float* __restrict__ q;                 // [B, n]
    float* __restrict__ pos_err;           // [B]
    float* __restrict__ rot_err;           // [B]
    uint8_t* __restrict__ converged;       // [B]
    float* __restrict__ damping_out;       // [B]
    int64_t batch;
    int32_t max_iters;
    float damping_init, pos_tol, rot_tol;
};

// shared-memory carve-up (floats); T rows per CTA
struct IkSmemLayout {
    int q, jac, tgt, tab, lim, total_floats;
    __host__ __device__ IkSmemLayout(int T, int n, int path_len) {
        int o = 0;
        tab = o; o += path_len * 12;           // 16-byte aligned: load_Fr reads float4
        lim = o; o += 2 * n;
        q = o;   o += 2 * n * T;
        jac = o; o += 2 * 6 * n * T;
        tgt = o; o += 7 * T;
        total_floats = o;
    }
};

// Pose and error of one configuration.  qx: this row's q slots (stride T); J: this row's Jacobian slots, rows 0..2 J_lin,
// 3..5 J_ang (only path columns are written; the others stay zero).  Returns E; e[0..M) and the two error norms.
template <bool POSE>
__device__ __forceinline__ float evaluate(const PathProgram& prog, const float* s_tab, const float* qx, float* J, int T, int n,
                                          const float* tgt, float* e, float& perr, float& rerr) {
    M3 R = identity3();
    V3 p = v3(0.f, 0.f, 0.f);
    const int nT = n * T;
    for (int k = 0; k < prog.len; ++k) {
        M3 F; V3 r;
        load_Fr(s_tab + k * 12, F, r);
        p = mul_add(R, r, p);                    // p_i = R_parent r_i + p_parent
        R = mul(R, F);                           // R_parent F~_i
        const int c = prog.dof[k];
        if (c >= 0) {
            float sn, cs;
            sincos_pi2(qx[c * T], sn, cs);
            const V3 z = col2(R);                // joint axis in the world frame (unchanged by Rz)
            const V3 m = cross(z, p);
            float* col = J + c * T;
            col[0] = m.x; col[nT] = m.y; col[2 * nT] = m.z;
            col[3 * nT] = z.x; col[4 * nT] = z.y; col[5 * nT] = z.z;
            rotate_z(R, cs, sn);
        }
    }
    // J_lin[:, c] = z x (p_ee - p_i) = z x p_ee - z x p_i
    for (int k = 0; k < prog.len; ++k) {
        const int c = prog.dof[k];
        if (c < 0) continue;
        float* col = J + c * T;
        const V3 z = v3(col[3 * nT], col[4 * nT], col[5 * nT]);
        const V3 j = cross_add(z, p, v3(-col[0], -col[nT], -col[2 * nT]));
        col[0] = j.x; col[nT] = j.y; col[2 * nT] = j.z;
    }
    e[0] = tgt[0] - p.x; e[1] = tgt[T] - p.y; e[2] = tgt[2 * T] - p.z;
    float E = fmaf(e[0], e[0], fmaf(e[1], e[1], e[2] * e[2]));
    perr = sqrtf(E);
    rerr = 0.f;
    if (POSE) {
        const float E_rot = rotvec_error(R, prog.ee_axis, tgt + 3 * T, T, e[3], e[4], e[5]);
        rerr = sqrtf(E_rot);
        E += E_rot;
    }
    return E;
}

template <bool POSE>
__global__ void __launch_bounds__(64)
inverse_kinematics_kernel(const __grid_constant__ PathProgram prog, const IkArgs args) {
    constexpr int M = POSE ? 6 : 3;              // rows of e and J that enter the system
    extern __shared__ __align__(128) float smem[];
    const int T = blockDim.x;
    const int n = prog.n_dofs;
    const IkSmemLayout L(T, n, prog.len);
    float* s_tab = smem + L.tab;
    float* s_lim = smem + L.lim;
    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, args.batch - tile_start);
    const bool limits = args.lower != nullptr;

    // ---- stage: path rows (signed gather), limits, clamped q0 and the targets, all slot-major -------------------------
    stage_walked_rows(s_tab, args.table, prog.tab_map, prog.len * 12, T);
    if (limits)
        for (int c = tid; c < n; c += T) { s_lim[c] = __ldg(args.lower + c); s_lim[n + c] = __ldg(args.upper + c); }
    if (!prog.full_cover)                        // Jacobian columns of joints off the path stay zero in both buffers
        for (int i = tid; i < 12 * n * T; i += T) smem[L.jac + i] = 0.f;
    __syncthreads();
    float* s_q = smem + L.q;
    for (int i = tid; i < valid * n; i += T) {   // coalesced global reads; q0 row-major -> slot-major
        const int r = i / n, c = i - r * n;
        s_q[c * T + r] = clamp_joint(__ldg(args.q0 + tile_start * n + i), s_lim, n, c, limits);
    }
    float* s_tgt = smem + L.tgt;
    for (int i = tid; i < valid * 3; i += T) {
        const int r = i / 3;
        s_tgt[(i - 3 * r) * T + r] = __ldg(args.tpos + tile_start * 3 + i);
    }
    if (POSE)
        for (int i = tid; i < valid * 4; i += T) {
            const int r = i >> 2;
            s_tgt[(3 + (i & 3)) * T + r] = __ldg(args.tquat + tile_start * 4 + i);
        }
    __syncthreads();

    if (tid < valid) {
        const int64_t row = tile_start + tid;
        const float* tgt = s_tgt + tid;
        if (POSE) normalize_target_quat(s_tgt + 3 * T + tid, T);      // the target quaternion, normalised once
        const int nT = n * T;
        float* const q_rows = smem + L.q + tid;             // buffer b of this row: q_rows + b nT, j_rows + 6 b nT
        float* const j_rows = smem + L.jac + tid;
        float lam = args.damping_in != nullptr ? __ldg(args.damping_in + row) : args.damping_init;
        float e[6], E = 0.f, perr = 0.f, rerr = 0.f;
        bool done = false;
        int cur = 0;
        // it = -1: the evaluation at the clamped start; it >= 0: trial steps.  ONE evaluate() call site.
        for (int it = -1;;) {
            int dst = cur;
            if (it >= 0) {
                if (done || it >= args.max_iters) break;
                dst = cur ^ 1;
                const float* J = j_rows + 6 * cur * nT;
                // A = J J^T + lambda I, lower triangle, over the path columns (the others are zero)
                float A[M][M];
#pragma unroll
                for (int i = 0; i < M; ++i)
#pragma unroll
                    for (int j = 0; j <= i; ++j) A[i][j] = 0.f;
                for (int k = 0; k < prog.len; ++k) {
                    const int c = prog.dof[k];
                    if (c < 0) continue;
                    float jc[M];
#pragma unroll
                    for (int i = 0; i < M; ++i) jc[i] = J[i * nT + c * T];
#pragma unroll
                    for (int i = 0; i < M; ++i)
#pragma unroll
                        for (int j = 0; j <= i; ++j) A[i][j] = fmaf(jc[i], jc[j], A[i][j]);
                }
                // Cholesky A = L L^T in place (L_ii stored as its reciprocal)
                bool ok = true;
#pragma unroll
                for (int j = 0; j < M; ++j) {
                    float d = A[j][j] + lam;
#pragma unroll
                    for (int k = 0; k < j; ++k) d = fmaf(-A[j][k], A[j][k], d);
                    ok = ok && d > 0.f && d < INFINITY;
                    const float inv = 1.f / sqrtf(d);
                    A[j][j] = inv;
#pragma unroll
                    for (int i = j + 1; i < M; ++i) {
                        float s = A[i][j];
#pragma unroll
                        for (int k = 0; k < j; ++k) s = fmaf(-A[i][k], A[j][k], s);
                        A[i][j] = s * inv;
                    }
                }
                ++it;
                if (!ok) { lam = fminf(4.f * lam, IK_LAMBDA_MAX); continue; }
                // y = A^-1 e: L w = e, L^T y = w
                float y[M];
#pragma unroll
                for (int i = 0; i < M; ++i) {
                    float s = e[i];
#pragma unroll
                    for (int k = 0; k < i; ++k) s = fmaf(-A[i][k], y[k], s);
                    y[i] = s * A[i][i];
                }
#pragma unroll
                for (int i = M - 1; i >= 0; --i) {
                    float s = y[i];
#pragma unroll
                    for (int k = i + 1; k < M; ++k) s = fmaf(-A[k][i], y[k], s);
                    y[i] = s * A[i][i];
                }
                // q' = clamp(q + J^T y); joints off the path keep their (already clamped) value
                const float* qc = q_rows + cur * nT;
                float* qt = q_rows + dst * nT;
                if (!prog.full_cover)
                    for (int c = 0; c < n; ++c) qt[c * T] = qc[c * T];
                for (int k = 0; k < prog.len; ++k) {
                    const int c = prog.dof[k];
                    if (c < 0) continue;
                    float s = 0.f;
#pragma unroll
                    for (int i = 0; i < M; ++i) s = fmaf(J[i * nT + c * T], y[i], s);
                    qt[c * T] = clamp_joint(qc[c * T] + s, s_lim, n, c, limits);
                }
            }
            float et[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, pt, rt;
            const float Et = evaluate<POSE>(prog, s_tab, q_rows + dst * nT, j_rows + 6 * dst * nT, T, n, tgt, et, pt, rt);
            if (it < 0 || Et < E) {
                if (it >= 0) lam = fmaxf(0.5f * lam, IK_LAMBDA_MIN);
                cur = dst;
                E = Et; perr = pt; rerr = rt;
#pragma unroll
                for (int i = 0; i < 6; ++i) e[i] = et[i];
                done = perr <= args.pos_tol && rerr <= args.rot_tol;
            } else {
                lam = fminf(4.f * lam, IK_LAMBDA_MAX);
            }
            if (it < 0) it = 0;
        }
        if (cur != 0)
            for (int c = 0; c < n; ++c) q_rows[c * T] = q_rows[nT + c * T];
        args.pos_err[row] = perr;
        args.rot_err[row] = rerr;
        args.converged[row] = done ? 1 : 0;
        args.damping_out[row] = lam;
    }
    __syncthreads();
    for (int i = tid; i < valid * n; i += T) {   // slot-major -> row-major, coalesced global writes
        const int r = i / n, c = i - r * n;
        args.q[tile_start * n + i] = s_q[c * T + r];
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// 64 rows while two CTAs still fit an SM, else 32 (a 63-DoF chain: ~117 KB at 32 rows)
static TileChoice ik_tile(const PathProgram& prog, size_t static_bytes) {
    return tile_64_or_32([&](int T) { return (size_t)IkSmemLayout(T, prog.n_dofs, prog.len).total_floats * sizeof(float); },
                         static_bytes);
}

template <bool POSE>
static int launch_ik(const PathProgram& prog, const IkArgs& args, cudaStream_t stream) {
    constexpr auto kern = inverse_kinematics_kernel<POSE>;
    size_t static_bytes;
    const int rc = static_smem_bytes<kern>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    const TileChoice c = ik_tile(prog, static_bytes);
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("inverse kinematics needs %zu B of shared memory per CTA (> 227 KB) for %d joints", c.bytes + static_bytes,
                  prog.n_dofs);
        return DRMB200_ELIMIT;
    }
    return launch_kernel<kern>((args.batch + c.tile - 1) / c.tile, c.tile, c.bytes, stream, false, "inverse kinematics", prog, args);
}

int inverse_kinematics_device(const drmb200_topology_t* topo, int32_t ee_link, const float* table, const float* q0,
                              const float* target_pos, const float* target_quat, const float* lower, const float* upper,
                              const float* damping_in, int64_t batch, int32_t max_iters, float damping_init, float pos_tol,
                              float rot_tol, float* q, float* pos_err, float* rot_err, uint8_t* converged, float* damping_out,
                              cudaStream_t stream) {
    PathProgram prog;
    const int rc = build_path_program(topo, ee_link, &prog);
    if (rc != DRMB200_OK) return rc;
    if (prog.n_dofs == 0) { set_error("inverse kinematics of a model without movable joints"); return DRMB200_EINVAL; }
    int movable = 0;
    for (int k = 0; k < prog.len; ++k) movable += prog.dof[k] >= 0;
    if (movable == 0) { set_error("ee_link=%d: no movable joint between the root and this link", ee_link); return DRMB200_EINVAL; }
    const int arg_rc = check_ik_arguments(table, q0, target_pos, lower, upper, batch, max_iters, damping_init, pos_tol, rot_tol, q,
                                          pos_err, rot_err, converged, damping_out);
    if (arg_rc != DRMB200_OK || batch == 0) return arg_rc;
    IkArgs args;
    args.table = table; args.q0 = q0; args.tpos = target_pos; args.tquat = target_quat;
    args.lower = lower; args.upper = upper; args.damping_in = damping_in;
    args.q = q; args.pos_err = pos_err; args.rot_err = rot_err; args.converged = converged; args.damping_out = damping_out;
    args.batch = batch; args.max_iters = max_iters;
    args.damping_init = damping_init; args.pos_tol = pos_tol; args.rot_tol = rot_tol;
    return target_quat != nullptr ? launch_ik<true>(prog, args, stream) : launch_ik<false>(prog, args, stream);
}

}  // namespace drm
