// contact_rollout.cu -- batched contact-constrained rollouts (sm_90a): T steps of semi-implicit Euler over the contact
// dynamics of bilateral rigid contacts at several links, with Baumgarte stabilisation, in ONE launch.
//
// Step t, fp32, in exactly this order (spec in include/drm_b200.h and DESIGN.md §3):
//   1. the walk at (q_t, qd_t): J, v = J qd, Jdot qd and every held link's world pose (p_l, R_l);
//   2. e [M]: per link p_l - p*_l and, in pose mode, the world-frame rotation vector of R_l R*_l^T, the shorter way round
//      (minus ik_common.cuh's rotvec_error, so that de/dt ~ the angular rows of J qd);
//   3. a_ref = -(2 omega) v - (omega^2) e, each product and the difference rounded once; omega = 0 forms no term: a_ref = 0;
//   4. (qdd_t, lambda_t, ok_t) = the contact dynamics at (q_t, qd_t, f_t, a_ref): DRM_CONTACT_ROW (contact_common.cuh), the
//      contact kernel's own statements;
//   5. qd_{t+1} = qd_t + dt * qdd_t;  q_{t+1} = q_t + dt * qd_{t+1}, each "+ dt *" one rounded multiply and one rounded add.
// With omega = 0 the trajectory is bit-identical to a loop of drmb200_contact_dynamics(accel_ref = NULL) calls followed by
// `qd = qd + dt * qdd; q = q + dt * qd`.  The targets are staged once (quaternions normalised as the IK kernels do) or, when
// none are given, taken from the step-0 walk: p*_l = p_l(q0) and quat*_l = the quaternion of R_l(q0), un-permuted as
// drmb200_fk_jacobian returns it, so both kinds go through rotvec_error.  DRMB200_IMPLICIT_DAMPING: step 4's ABA takes the
// pivots d + dt damping (contact_rollout_implicit_kernel), which its unit-response sweeps read back, so qdd_free, G and A
// are those of the implicit step.
//
// Mapping: the contact kernel's (one thread per row, T rows per CTA, the same slot-major row state) with the rollouts' time
// loop (rollout_pipeline.cuh: state staging, f double buffer, integrate and q / qd / qdd stores).  Once per CTA the
// canonical (unfolded) table, the (q0, qd0) tile and the targets are staged; the state then lives in shared memory for all
// steps.  Per step the f_t tile is copied into the ABA's f row, which the unit-response sweeps overwrite; the integrate
// reads qdd from the slot-major output, which is also copied into a row-major double buffer for the pipeline's qdd store.
// lambda (slot-major) leaves through store_transposed and a_ref (row-major, the layout the contact row reads) through a
// linear cooperative copy, after the pipeline's stores.  The solved flag is the AND of every step's, kept in a register
// and written once.
//
// Algorithmic HBM bytes per configuration-step: f in 4n, q / qd / qdd out 12n, force out 4M (a_ref 4M more when asked for).
#include <cmath>
#include "contact_common.cuh"
#include "ik_common.cuh"
#include "launch.cuh"
#include "rollout_pipeline.cuh"

namespace drm {

int contact_programs(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, float regularization,
                     int64_t batch, UnionProgram* P, const TreeProgram** prog);

struct ContactRolloutArgs {
    const float* __restrict__ table;
    const float* __restrict__ q0;
    const float* __restrict__ qd0;
    const float* __restrict__ f;            // [T, B, n]
    const float* __restrict__ target_pos;   // [n_ee, B, 3] or null (the step-0 poses)
    const float* __restrict__ target_quat;  // [n_ee, B, 4] or null
    float* __restrict__ q;                  // [T, B, n]
    float* __restrict__ qd;
    float* __restrict__ qdd;                // may be null
    float* __restrict__ force;              // [T, B, M] or null
    float* __restrict__ accel_ref;          // [T, B, M] or null
    uint8_t* __restrict__ solved;           // [B]
    int64_t batch;
    int32_t n_steps;
    float dt;
    uint32_t flags;
    int32_t M;
    float mu;
    float two_omega;                        // 2 omega and omega^2, each rounded once; omega = 0: no a_ref term at all
    float omega_sq;
    int32_t stabilize;
    int32_t aligned;                        // q0, qd0, f, q, qd, qdd 16-byte aligned and batch * n % 4 == 0
    int8_t axis[MT_MAX_EE];                 // axis code of every held link (un-permutation before the quaternion)
};

struct ContactRolloutSmem {
    AbaSmemLayout aba;
    int fbuf, qddbuf, ref, jac, jscr, state, vel, bias, lam, scale, a, out, pose, tpos, tquat, total_floats;
    __host__ __device__ ContactRolloutSmem(int T, const TreeProgram& tp, const UnionProgram& P, int M)
        : aba(T, tp.n_dofs, tp.n_links, tp.n_slots) {
        const int n = tp.n_dofs, E = P.walk.n_ee;
        int o = (aba.total_floats + 3) & ~3;    // 16-byte aligned: TMA targets and sources
        fbuf = o;   o += 2 * T * n;             // double buffers
        qddbuf = o; o += 2 * T * n;
        ref = o;   o += M * T;
        jac = o;   o += M * P.n_u * T;
        jscr = o;  o += 6 * P.walk.n_jslots * T;
        state = o; o += OSD_STATE * P.walk.n_state_slots * T;
        vel = o;   o += M * T;
        bias = o;  o += M * T;
        lam = o;   o += M * T;
        scale = o; o += M * T;
        a = o;     o += M * M * T;
        out = o;   o += n * T;
        pose = o;  o += 12 * E * T;
        tpos = o;  o += 3 * E * T;
        tquat = o; o += (M == 6 * E ? 4 * E : 0) * T;
        total_floats = o;
    }
};

// The kernel's body, instantiated by contact_rollout_kernel (explicit damping) and contact_rollout_implicit_kernel
// (IMPLICIT: implicit damping of step h = dt, DRMB200_IMPLICIT_DAMPING): two kernel names rather than a template flag on
// one, so that the explicit kernel keeps its symbol.
template <int T, bool IMPLICIT>
__device__ __forceinline__ void contact_rollout_run(const TreeProgram& prog, const UnionProgram& P,
                                                    const ContactRolloutArgs& args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar[2];

    const int n = prog.n_dofs;
    const int M = args.M;
    const int E = P.walk.n_ee;
    const int MR = M / E;
    const int n_u = P.n_u;
    const ContactRolloutSmem L(T, prog, P, M);
    float* s_q = smem + L.aba.q;
    float* s_qd = smem + L.aba.qd;
    float* s_f = smem + L.aba.f;
    float* s_qdd = smem + L.aba.qdd;
    float* s_tab = smem + L.aba.table;
    float* s_qddb = smem + L.qddbuf;
    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;

    const RolloutPipeline<T> pipe(mbar, s_q, s_qd, smem + L.fbuf, args.f, nullptr, nullptr, args.q, args.qd, n, args.batch,
                                  args.n_steps, args.dt, args.aligned);
    const int valid = pipe.valid;
    pipe.begin(args.q0, args.qd0);
    stage_canonical_table(s_tab, args.table, prog, T);
    // J, velocity and bias start at zero (columns off a link's path); a_ref stays zero without stabilisation
    for (int i = L.ref + tid; i < L.jscr; i += T) smem[i] = 0.f;
    for (int i = L.vel + tid; i < L.lam; i += T) smem[i] = 0.f;
    const bool given = args.target_pos != nullptr;
    if (given) {                                          // [n_ee, B, 3] / [n_ee, B, 4] -> slot-major, element (l, k) at (K l + k) T
        for (int i = tid; i < E * valid * 3; i += T) {
            const int l = i / (valid * 3), rem = i - l * valid * 3, r = rem / 3, k = rem - r * 3;
            smem[L.tpos + (3 * l + k) * T + r] = args.target_pos[((int64_t)l * args.batch + tile_start + r) * 3 + k];
        }
        if (MR == 6)
            for (int i = tid; i < E * valid * 4; i += T) {
                const int l = i / (valid * 4), rem = i - l * valid * 4, r = rem / 4, k = rem - r * 4;
                smem[L.tquat + (4 * l + k) * T + r] = args.target_quat[((int64_t)l * args.batch + tile_start + r) * 4 + k];
            }
    }
    __syncthreads();
    if (given && MR == 6 && tid < valid)
        for (int l = 0; l < E; ++l) normalize_target_quat(smem + L.tquat + 4 * l * T + tid, T);

    uint8_t solved = 1;
    for (int t = 0; t < args.n_steps; ++t) {
        const float* s_ft = pipe.fetch(t);
        float* s_qddt = s_qddb + (t & 1) * T * n;
        if (tid < valid) {
            for (int c = 0; c < n; ++c) s_f[tid * n + c] = s_ft[tid * n + c];
            // steps 2-3, between the walk and the contact dynamics: the targets (step 0, when not given) and a_ref
            auto baumgarte = [&]() {
                const float* ps = smem + L.pose + tid;
                float* tp = smem + L.tpos + tid;
                float* tq = smem + L.tquat + tid;
                if (t == 0 && !given)
                    for (int l = 0; l < E; ++l) {
                        stv(tp + 3 * l * T, T, ldv(ps + 12 * l * T, T));
                        if (MR == 6) {
                            M3 R = ldm(ps + (12 * l + 3) * T, T);
                            if (args.axis[l] != 0) R = unpermute_cols(R, args.axis[l]);
                            const float4 c = quat_xyzw(R);
                            tq[4 * l * T] = c.x; tq[(4 * l + 1) * T] = c.y; tq[(4 * l + 2) * T] = c.z; tq[(4 * l + 3) * T] = c.w;
                        }
                    }
                if (!args.stabilize) return;
                const float* v = smem + L.vel + tid;
                float* ref = smem + L.ref + tid * M;
                for (int l = 0; l < E; ++l) {
                    const V3 p = ldv(ps + 12 * l * T, T), pt = ldv(tp + 3 * l * T, T);
                    const float e[3] = {p.x - pt.x, p.y - pt.y, p.z - pt.z};
                    for (int k = 0; k < 3; ++k)
                        ref[MR * l + k] = __fsub_rn(__fmul_rn(-args.two_omega, v[(MR * l + k) * T]), __fmul_rn(args.omega_sq, e[k]));
                    if (MR == 6) {
                        float rx, ry, rz;
                        rotvec_error(ldm(ps + (12 * l + 3) * T, T), args.axis[l], tq + 4 * l * T, T, rx, ry, rz);
                        const float er[3] = {-rx, -ry, -rz};      // rotvec(R R*^T) = -rotvec(R* R^T)
                        for (int k = 0; k < 3; ++k)
                            ref[MR * l + 3 + k] = __fsub_rn(__fmul_rn(-args.two_omega, v[(MR * l + 3 + k) * T]),
                                                            __fmul_rn(args.omega_sq, er[k]));
                    }
                }
            };
            bool ok;
            DRM_CONTACT_ROW(T, false, true, smem + L.pose + tid, args.flags, args.mu, ok, IMPLICIT, args.dt, baumgarte(););
            solved &= ok ? 1 : 0;
            if (args.qdd != nullptr)
                for (int c = 0; c < n; ++c) s_qddt[tid * n + c] = smem[L.out + c * T + tid];
        }

        pipe.integrate_and_store(t, smem + L.out + tid, T, args.qdd, s_qddt);     // q̈ from the slot-major output
        const int64_t mrow = ((int64_t)t * args.batch + tile_start) * M;
        if (args.force != nullptr) store_transposed(args.force + mrow, smem + L.lam, M, valid, T);
        if (args.accel_ref != nullptr) {
            float* dst = args.accel_ref + mrow;
            coop_copy(dst, smem + L.ref, valid * M, (reinterpret_cast<uintptr_t>(dst) & 15u) == 0);
        }
        if (args.force != nullptr || args.accel_ref != nullptr) __syncthreads();    // before the next step rewrites them
    }
    pipe.finish();
    if (tid < valid) args.solved[tile_start + tid] = solved;
}

template <int T>
__global__ void __launch_bounds__(T)
contact_rollout_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ UnionProgram P,
                       const __grid_constant__ ContactRolloutArgs args) {
    contact_rollout_run<T, false>(prog, P, args);
}

template <int T>
__global__ void __launch_bounds__(T)
contact_rollout_implicit_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ UnionProgram P,
                                const __grid_constant__ ContactRolloutArgs args) {
    contact_rollout_run<T, true>(prog, P, args);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
int contact_rollout_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                           const float* q0, const float* qd0, const float* f, const float* target_pos,
                           const float* target_quat, int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                           int32_t position_only, float regularization, float stabilization, float* q, float* qd, float* qdd,
                           float* force, float* accel_ref, uint8_t* solved, cudaStream_t stream) {
    UnionProgram P;
    const TreeProgram* prog = nullptr;
    int rc = contact_programs(topo, n_ee, ee_links, regularization, batch, &P, &prog);
    if (rc != DRMB200_OK) return rc;
    if (n_steps < 0) { set_error("n_steps=%d < 0", (int)n_steps); return DRMB200_EINVAL; }
    if (!(stabilization >= 0.f) || !std::isfinite(stabilization)) {
        set_error("stabilization=%g: must be finite and >= 0", (double)stabilization);
        return DRMB200_EINVAL;
    }
    rc = check_implicit_damping(flags, dt);
    if (rc == DRMB200_OK) rc = check_implicit_gains(flags, dt, false);
    if (rc != DRMB200_OK) return rc;
    if (position_only && target_quat != nullptr) {
        set_error("target_quat must be null for position-only contacts");
        return DRMB200_EINVAL;
    }
    if (!position_only && (target_pos == nullptr) != (target_quat == nullptr)) {
        set_error("pose contacts need target_pos and target_quat both given or both null");
        return DRMB200_EINVAL;
    }
    if (batch == 0 || n_steps == 0) return DRMB200_OK;     // empty tensors may have null data pointers
    if (table == nullptr || q0 == nullptr || qd0 == nullptr || f == nullptr || q == nullptr || qd == nullptr || solved == nullptr) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    ContactRolloutArgs args;
    args.table = table; args.q0 = q0; args.qd0 = qd0; args.f = f; args.target_pos = target_pos; args.target_quat = target_quat;
    args.q = q; args.qd = qd; args.qdd = qdd; args.force = force; args.accel_ref = accel_ref; args.solved = solved;
    args.batch = batch; args.n_steps = n_steps; args.dt = dt; args.flags = flags & (DRMB200_GRAVITY | DRMB200_DAMPING);
    args.M = (position_only ? 3 : 6) * n_ee;
    args.mu = regularization;
    args.two_omega = 2.0f * stabilization;
    args.omega_sq = stabilization * stabilization;
    args.stabilize = stabilization > 0.f;
    args.aligned = aligned16(q0, qd0, f, q, qd, qdd) && ((batch * prog->n_dofs) & 3) == 0;
    for (int l = 0; l < MT_MAX_EE; ++l) args.axis[l] = l < n_ee ? topo->axis[ee_links[l]] : 0;

    size_t static_bytes;
    rc = static_smem_bytes<contact_rollout_kernel<64>>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    // the largest power-of-two tile <= 64 rows while two CTAs still fit an SM, else down to one row per CTA
    const TileChoice c = tile_ladder([&](int T) {
        return (size_t)ContactRolloutSmem(T, *prog, P, args.M).total_floats * sizeof(float);
    }, static_bytes);
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("contact rollout needs %zu B of shared memory per CTA (> 227 KB) for one row (%d joints, %d links, M = %d)",
                  c.bytes + static_bytes, prog->n_dofs, prog->n_links, args.M);
        return DRMB200_ELIMIT;
    }
    const int64_t tiles = (batch + c.tile - 1) / c.tile;
    if (flags & DRMB200_IMPLICIT_DAMPING) {
#define DRM_LAUNCH_CONTACT_ROLLOUT(TT) \
    launch_kernel<contact_rollout_implicit_kernel<TT>>(tiles, TT, c.bytes, stream, false, "contact rollout", *prog, P, args)
        switch (c.tile) {
            case 64: return DRM_LAUNCH_CONTACT_ROLLOUT(64);
            case 32: return DRM_LAUNCH_CONTACT_ROLLOUT(32);
            case 16: return DRM_LAUNCH_CONTACT_ROLLOUT(16);
            case 8: return DRM_LAUNCH_CONTACT_ROLLOUT(8);
            case 4: return DRM_LAUNCH_CONTACT_ROLLOUT(4);
            case 2: return DRM_LAUNCH_CONTACT_ROLLOUT(2);
            default: return DRM_LAUNCH_CONTACT_ROLLOUT(1);
        }
#undef DRM_LAUNCH_CONTACT_ROLLOUT
    }
#define DRM_LAUNCH_CONTACT_ROLLOUT(TT) \
    launch_kernel<contact_rollout_kernel<TT>>(tiles, TT, c.bytes, stream, false, "contact rollout", *prog, P, args)
    switch (c.tile) {
        case 64: return DRM_LAUNCH_CONTACT_ROLLOUT(64);
        case 32: return DRM_LAUNCH_CONTACT_ROLLOUT(32);
        case 16: return DRM_LAUNCH_CONTACT_ROLLOUT(16);
        case 8: return DRM_LAUNCH_CONTACT_ROLLOUT(8);
        case 4: return DRM_LAUNCH_CONTACT_ROLLOUT(4);
        case 2: return DRM_LAUNCH_CONTACT_ROLLOUT(2);
        default: return DRM_LAUNCH_CONTACT_ROLLOUT(1);
    }
#undef DRM_LAUNCH_CONTACT_ROLLOUT
}

}  // namespace drm
