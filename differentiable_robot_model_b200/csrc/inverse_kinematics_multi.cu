// inverse_kinematics_multi.cu -- batched Levenberg-Marquardt inverse kinematics of SEVERAL links at once (sm_90a).
//
// The multi-link counterpart of inverse_kinematics.cu: one thread per row (a start configuration and one target per link),
// all iterations inside ONE launch.  The links share the joints on the common part of their root paths (an arm carrying a
// hand), so one damped least-squares solve over the stacked errors of every link moves them together; no combination of
// single-link solves does that.  Per row, in fp32 (spec in include/drm_b200.h and DESIGN.md §3):
//
//   U = the movable joints on the union of the root -> link paths (n_u of them), M = 3 n_ee (position) or 6 n_ee (pose)
//   q <- clamp(q0); lambda <- damping_in[b] or damping_init; evaluate at q
//   repeat max_iters times while the row is not done:
//       M <= n_u (task space):   A = J_U J_U^T + lambda I_M,   dq_U = J_U^T A^-1 e
//       M >  n_u (joint space):  A = J_U^T J_U + lambda I_nu,  dq_U = A^-1 J_U^T e      (the same step, smaller system)
//       Cholesky of A (a pivot <= 0 or not finite rejects the step); q' = clamp(q + dq) on U; evaluate at q'
//       E' < E: accept, lambda <- max(lambda / 2, IK_LAMBDA_MIN);  else reject, lambda <- min(4 lambda, IK_LAMBDA_MAX)
//
// "evaluate" walks the union of the paths once with the MultiProgram of fk_tree.cu (same depth-first order, same signed
// table gather) and, as it passes each requested link, writes that link's rows of the stacked Jacobian and error with the
// arithmetic of inverse_kinematics.cu's evaluate(): with one link and M <= n_u every operation is the same in the same
// order, so the result is bit-identical to drmb200_inverse_kinematics.  Like there, evaluate() has ONE call site, so K
// iterations in one call are bit-identical to K chained calls of max_iters = 1.
//
// Shared memory, slot-major (element e of row t at base[e * T + t]):
//   per row  q[2][n]; J[2][M][n_u] (current / trial, swapped by an index on accept; entries of joints off a link's path
//            stay zero); e[2][M]; the targets; the lower triangle of A (m = min(M, n_u): up to 48 x 48); the solve vector
//            y[m]; the joint scratch z_i, z_i x p_i of the walk (6 per path depth) and the spilled (R, p) of branch points
//   per CTA  the canonical rows of the walked links (12 floats each) and the joint limits 2n
// A no longer fits in registers (the single-link kernel keeps its 6 x 6 there).  HBM traffic per row is independent of
// max_iters: the kernel is arithmetic-bound.
#include <cmath>
#include "ik_common.cuh"
#include "launch.cuh"
#include "multi_program.cuh"

namespace drm {

struct IkmArgs {
    const float* __restrict__ table;       // [n_links, 28]
    const float* __restrict__ q0;          // [B, n]
    const float* __restrict__ tpos;        // [n_ee, B, 3]
    const float* __restrict__ tquat;       // [n_ee, B, 4] xyzw, or null (position only)
    const float* __restrict__ lower;       // [n] or null
    const float* __restrict__ upper;       // [n] or null
    const float* __restrict__ damping_in;  // [B] or null
    float* __restrict__ q;                 // [B, n]
    float* __restrict__ pos_err;           // [n_ee, B]
    float* __restrict__ rot_err;           // [n_ee, B]
    uint8_t* __restrict__ converged;       // [B]
    float* __restrict__ damping_out;       // [B]
    int64_t batch;
    int32_t max_iters;
    float damping_init, pos_tol, rot_tol;
};

// shared-memory carve-up (floats); T rows per CTA
struct IkmSmemLayout {
    int M, m, tw, q, jac, err, tgt, a, y, jscr, state, tab, lim, total_floats;
    __host__ __device__ IkmSmemLayout(int T, int n, int n_u, int n_ee, bool pose, int n_steps, int n_jslots, int n_state_slots) {
        M = (pose ? 6 : 3) * n_ee;
        m = M <= n_u ? M : n_u;
        tw = pose ? 7 : 3;
        int o = 0;
        tab = o;   o += n_steps * 12;          // 16-byte aligned: load_Fr reads float4
        lim = o;   o += 2 * n;
        q = o;     o += 2 * n * T;
        jac = o;   o += 2 * M * n_u * T;
        err = o;   o += 2 * M * T;
        tgt = o;   o += tw * n_ee * T;
        a = o;     o += m * (m + 1) / 2 * T;
        y = o;     o += m * T;
        jscr = o;  o += 6 * n_jslots * T;
        state = o; o += 12 * n_state_slots * T;
        total_floats = o;
    }
};

__device__ __forceinline__ int tri(int i, int j) { return i * (i + 1) / 2 + j; }

// Pose errors and stacked Jacobian of one configuration.  qx: this row's q slots; J: this row's J[M][n_u] slots; e: its
// e[M] slots; jscr / st: its joint scratch and branch-state slots; tgt: its targets (tw slots per link).  Returns E and
// whether every link is within tolerance.
template <bool POSE>
__device__ __forceinline__ float evaluate_multi(const UnionProgram& P, const float* s_tab, const float* qx, float* J, float* e,
                                                float* jscr, float* st, const float* tgt, int T, float pos_tol, float rot_tol,
                                                bool& within) {
    constexpr int MR = POSE ? 6 : 3;             // rows per link
    constexpr int TW = POSE ? 7 : 3;
    const MultiProgram& W = P.walk;
    M3 R = identity3();
    V3 p = v3(0.f, 0.f, 0.f);
    float E = 0.f;
    within = true;
    for (int k = 0; k < W.n_steps; ++k) {
        M3 F; V3 r;
        load_Fr(s_tab + k * 12, F, r);
        const int src = W.psrc[k];
        if (src < 0) {
            R = identity3(); p = v3(0.f, 0.f, 0.f);
        } else if (src > 0) {
            const float* s = st + (src - 1) * 12 * T;
            R = ldm(s, T); p = ldv(s + 9 * T, T);
        }
        p = mul_add(R, r, p);                    // p_i = R_parent r_i + p_parent
        R = mul(R, F);                           // R_parent F~_i
        const int c = W.dof[k];
        if (c >= 0) {
            float sn, cs;
            sincos_pi2(qx[c * T], sn, cs);
            const V3 z = col2(R);                // joint axis in the world frame (unchanged by Rz)
            float* js = jscr + W.jslot[k] * 6 * T;
            stv(js, T, z);
            stv(js + 3 * T, T, cross(z, p));
            rotate_z(R, cs, sn);
        }
        const int sv = W.save[k];
        if (sv >= 0) {
            float* s = st + sv * 12 * T;
            stm(s, T, R); stv(s + 9 * T, T, p);
        }
        const int l = W.ee[k];
        if (l < 0) continue;
        // link l: its rows of J and of e
        link_jacobian(P, l, MR, p, jscr, J, T);
        const float* tl = tgt + TW * l * T;
        float* el = e + MR * l * T;
        const float ex = tl[0] - p.x, ey = tl[T] - p.y, ez = tl[2 * T] - p.z;
        el[0] = ex; el[T] = ey; el[2 * T] = ez;
        float El = fmaf(ex, ex, fmaf(ey, ey, ez * ez));
        const float perr = sqrtf(El);
        float rerr = 0.f;
        if (POSE) {
            float rx, ry, rz;
            const float E_rot = rotvec_error(R, W.axis[k], tl + 3 * T, T, rx, ry, rz);
            el[3 * T] = rx; el[4 * T] = ry; el[5 * T] = rz;
            rerr = sqrtf(E_rot);
            El += E_rot;
        }
        within = within && perr <= pos_tol && rerr <= rot_tol;
        E += El;
    }
    return E;
}

template <bool POSE>
__global__ void __launch_bounds__(64)
inverse_kinematics_multi_kernel(const __grid_constant__ UnionProgram P, const IkmArgs args) {
    constexpr int MR = POSE ? 6 : 3;
    extern __shared__ __align__(128) float smem[];
    const MultiProgram& W = P.walk;
    const int T = blockDim.x;
    const int n = W.n_dofs, n_u = P.n_u, n_ee = W.n_ee;
    const IkmSmemLayout L(T, n, n_u, n_ee, POSE, W.n_steps, W.n_jslots, W.n_state_slots);
    const int M = L.M, m = L.m, TW = L.tw;
    float* s_tab = smem + L.tab;
    float* s_lim = smem + L.lim;
    const int tid = threadIdx.x;
    const int64_t B = args.batch;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, B - tile_start);
    const bool limits = args.lower != nullptr;

    // ---- stage: walked rows (signed gather), limits, zeroed Jacobians, clamped q0 and the targets, slot-major ----------
    stage_walked_rows(s_tab, args.table, W.tab_map, W.n_steps * 12, T);
    if (limits)
        for (int c = tid; c < n; c += T) { s_lim[c] = __ldg(args.lower + c); s_lim[n + c] = __ldg(args.upper + c); }
    for (int i = tid; i < 2 * M * n_u * T; i += T) smem[L.jac + i] = 0.f;
    __syncthreads();
    float* s_q = smem + L.q;
    for (int i = tid; i < valid * n; i += T) {   // coalesced global reads; q0 row-major -> slot-major
        const int r = i / n, c = i - r * n;
        s_q[c * T + r] = clamp_joint(__ldg(args.q0 + tile_start * n + i), s_lim, n, c, limits);
    }
    float* s_tgt = smem + L.tgt;
    for (int l = 0; l < n_ee; ++l) {
        for (int i = tid; i < valid * 3; i += T) {
            const int r = i / 3;
            s_tgt[(TW * l + i - 3 * r) * T + r] = __ldg(args.tpos + ((int64_t)l * B + tile_start) * 3 + i);
        }
        if (POSE)
            for (int i = tid; i < valid * 4; i += T) {
                const int r = i >> 2;
                s_tgt[(TW * l + 3 + (i & 3)) * T + r] = __ldg(args.tquat + ((int64_t)l * B + tile_start) * 4 + i);
            }
    }
    __syncthreads();

    if (tid < valid) {
        const int64_t row = tile_start + tid;
        const float* tgt = s_tgt + tid;
        if (POSE)                                // the target quaternions, normalised once
            for (int l = 0; l < n_ee; ++l) normalize_target_quat(s_tgt + (TW * l + 3) * T + tid, T);
        const int nT = n * T, JT = M * n_u * T, rs = n_u * T;
        float* const q_rows = smem + L.q + tid;              // buffer b of this row: q_rows + b nT, j_rows + b JT, e_rows + b M T
        float* const j_rows = smem + L.jac + tid;
        float* const e_rows = smem + L.err + tid;
        float* const A = smem + L.a + tid;
        float* const y = smem + L.y + tid;
        float* const jscr = smem + L.jscr + tid;
        float* const st = smem + L.state + tid;
        const bool task = M <= n_u;
        float lam = args.damping_in != nullptr ? __ldg(args.damping_in + row) : args.damping_init;
        float E = 0.f;
        bool done = false;
        int cur = 0;
        // it = -1: the evaluation at the clamped start; it >= 0: trial steps.  ONE evaluate_multi() call site.
        for (int it = -1;;) {
            int dst = cur;
            if (it >= 0) {
                if (done || it >= args.max_iters) break;
                dst = cur ^ 1;
                const float* J = j_rows + cur * JT;
                const float* e = e_rows + cur * M * T;
                // A = J J^T (M x M) or J^T J (n_u x n_u), lower triangle; the Jacobian-weighted error J^T e -> y (joint space)
                if (task) {
                    for (int i = 0; i < M; ++i)
                        for (int j = 0; j <= i; ++j) {
                            float s = 0.f;
                            for (int u = 0; u < n_u; ++u) s = fmaf(J[i * rs + u * T], J[j * rs + u * T], s);
                            A[tri(i, j) * T] = s;
                        }
                } else {
                    for (int a = 0; a < n_u; ++a) {
                        for (int b = 0; b <= a; ++b) {
                            float s = 0.f;
                            for (int i = 0; i < M; ++i) s = fmaf(J[i * rs + a * T], J[i * rs + b * T], s);
                            A[tri(a, b) * T] = s;
                        }
                        float g = 0.f;
                        for (int i = 0; i < M; ++i) g = fmaf(J[i * rs + a * T], e[i * T], g);
                        y[a * T] = g;
                    }
                }
                // Cholesky A + lambda I = L L^T in place (L_ii stored as its reciprocal)
                bool ok = true;
                for (int j = 0; j < m && ok; ++j) {
                    float d = A[tri(j, j) * T] + lam;
                    for (int k = 0; k < j; ++k) d = fmaf(-A[tri(j, k) * T], A[tri(j, k) * T], d);
                    ok = d > 0.f && d < INFINITY;
                    const float inv = 1.f / sqrtf(d);
                    A[tri(j, j) * T] = inv;
                    for (int i = j + 1; i < m; ++i) {
                        float s = A[tri(i, j) * T];
                        for (int k = 0; k < j; ++k) s = fmaf(-A[tri(i, k) * T], A[tri(j, k) * T], s);
                        A[tri(i, j) * T] = s * inv;
                    }
                }
                ++it;
                if (!ok) { lam = fminf(4.f * lam, IK_LAMBDA_MAX); continue; }
                // y = A^-1 (e or J^T e): L w = ., L^T y = w
                for (int i = 0; i < m; ++i) {
                    float s = task ? e[i * T] : y[i * T];
                    for (int k = 0; k < i; ++k) s = fmaf(-A[tri(i, k) * T], y[k * T], s);
                    y[i * T] = s * A[tri(i, i) * T];
                }
                for (int i = m - 1; i >= 0; --i) {
                    float s = y[i * T];
                    for (int k = i + 1; k < m; ++k) s = fmaf(-A[tri(k, i) * T], y[k * T], s);
                    y[i * T] = s * A[tri(i, i) * T];
                }
                // q' = clamp(q + dq) on U, dq = J^T y (task space) or y (joint space); joints outside U keep their value
                const float* qc = q_rows + cur * nT;
                float* qt = q_rows + dst * nT;
                if (n_u < n)
                    for (int c = 0; c < n; ++c) qt[c * T] = qc[c * T];
                for (int u = 0; u < n_u; ++u) {
                    const int c = P.u_dof[u];
                    float s;
                    if (task) {
                        s = 0.f;
                        for (int i = 0; i < M; ++i) s = fmaf(J[i * rs + u * T], y[i * T], s);
                    } else {
                        s = y[u * T];
                    }
                    qt[c * T] = clamp_joint(qc[c * T] + s, s_lim, n, c, limits);
                }
            }
            bool within;
            const float Et = evaluate_multi<POSE>(P, s_tab, q_rows + dst * nT, j_rows + dst * JT, e_rows + dst * M * T, jscr, st,
                                                  tgt, T, args.pos_tol, args.rot_tol, within);
            if (it < 0 || Et < E) {
                if (it >= 0) lam = fmaxf(0.5f * lam, IK_LAMBDA_MIN);
                cur = dst;
                E = Et;
                done = within;
            } else {
                lam = fminf(4.f * lam, IK_LAMBDA_MAX);
            }
            if (it < 0) it = 0;
        }
        if (cur != 0)
            for (int c = 0; c < n; ++c) q_rows[c * T] = q_rows[nT + c * T];
        const float* e = e_rows + cur * M * T;
        for (int l = 0; l < n_ee; ++l) {         // |e_pos|, |e_rot| of each link, as evaluate_multi() computed them
            const float* el = e + MR * l * T;
            args.pos_err[l * B + row] = sqrtf(fmaf(el[0], el[0], fmaf(el[T], el[T], el[2 * T] * el[2 * T])));
            args.rot_err[l * B + row] =
                POSE ? sqrtf(fmaf(el[3 * T], el[3 * T], fmaf(el[4 * T], el[4 * T], el[5 * T] * el[5 * T]))) : 0.f;
        }
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
// the largest power-of-two tile <= 64 rows while two CTAs still fit an SM, else down to one row per CTA
static TileChoice ikm_tile(const UnionProgram& P, bool pose, size_t static_bytes) {
    const MultiProgram& W = P.walk;
    return tile_ladder([&](int T) {
        return (size_t)IkmSmemLayout(T, W.n_dofs, P.n_u, W.n_ee, pose, W.n_steps, W.n_jslots, W.n_state_slots).total_floats *
               sizeof(float);
    }, static_bytes);
}

template <bool POSE>
static int launch_ikm(const UnionProgram& P, const IkmArgs& args, cudaStream_t stream) {
    constexpr auto kern = inverse_kinematics_multi_kernel<POSE>;
    size_t static_bytes;
    const int rc = static_smem_bytes<kern>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    const TileChoice c = ikm_tile(P, POSE, static_bytes);
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("multi-link inverse kinematics needs %zu B of shared memory per CTA (> 227 KB) for one row (%d joints, %d links)",
                  c.bytes + static_bytes, P.walk.n_dofs, P.walk.n_ee);
        return DRMB200_ELIMIT;
    }
    return launch_kernel<kern>((args.batch + c.tile - 1) / c.tile, c.tile, c.bytes, stream, false, "multi-link inverse kinematics", P,
                               args);
}

int inverse_kinematics_multi_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                    const float* q0, const float* target_pos, const float* target_quat, const float* lower,
                                    const float* upper, const float* damping_in, int64_t batch, int32_t max_iters,
                                    float damping_init, float pos_tol, float rot_tol, float* q, float* pos_err, float* rot_err,
                                    uint8_t* converged, float* damping_out, cudaStream_t stream) {
    UnionProgram P;
    const int rc = build_union_program(topo, n_ee, ee_links, &P);
    if (rc != DRMB200_OK) return rc;
    const MultiProgram& W = P.walk;
    if (W.n_dofs == 0) { set_error("inverse kinematics of a model without movable joints"); return DRMB200_EINVAL; }
    for (int l = 0; l < n_ee; ++l) {
        int movable = 0;
        for (int c = 0; c < W.n_dofs; ++c) movable += W.cslot[l][c] >= 0;
        if (movable == 0) {
            set_error("ee_links[%d]=%d: no movable joint between the root and this link", l, ee_links[l]);
            return DRMB200_EINVAL;
        }
    }
    const int arg_rc = check_ik_arguments(table, q0, target_pos, lower, upper, batch, max_iters, damping_init, pos_tol, rot_tol, q,
                                          pos_err, rot_err, converged, damping_out);
    if (arg_rc != DRMB200_OK || batch == 0) return arg_rc;
    IkmArgs args;
    args.table = table; args.q0 = q0; args.tpos = target_pos; args.tquat = target_quat;
    args.lower = lower; args.upper = upper; args.damping_in = damping_in;
    args.q = q; args.pos_err = pos_err; args.rot_err = rot_err; args.converged = converged; args.damping_out = damping_out;
    args.batch = batch; args.max_iters = max_iters;
    args.damping_init = damping_init; args.pos_tol = pos_tol; args.rot_tol = rot_tol;
    return target_quat != nullptr ? launch_ikm<true>(P, args, stream) : launch_ikm<false>(P, args, stream);
}

}  // namespace drm
