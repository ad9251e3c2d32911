// rollout.cu -- batched forward-dynamics rollouts (sm_90a): T steps of semi-implicit Euler over the articulated-body
// algorithm in ONE launch, open loop or with a diagonal joint-space PD law closing the loop, and the reverse-time adjoint
// of both.
//
// Open-loop step t, fp32, in exactly this order (qdd_t is what drmb200_forward_dynamics returns for (q_t, qd_t, f_t)):
//   qdd_t = FD(q_t, qd_t, f_t);   qd_{t+1} = qd_t + dt * qdd_t;   q_{t+1} = q_t + dt * qd_{t+1}
// PD step t, every operation rounded separately (the definition is stated in include/drm_b200.h):
//   e_t = q_ref[t] - q_t;  ed_t = qd_ref[t] - qd_t;  u_t = (f[t] + kp e_t) + kd ed_t;  tau_t = clamp(u_t, -lim, lim)
//   qdd_t = FD(q_t, qd_t, tau_t), then the same integrate.  (qd_ref / f absent: 0 - qd_t / 0 + kp e_t; lim absent: no
//   clamp.)
// each "+ dt *" one rounded multiply and one rounded add, so that the trajectory is bit-identical to the stepwise torch loop.
// DRMB200_IMPLICIT_DAMPING: FD is the forward dynamics with implicit damping of step h = dt (rollout_implicit_kernel,
// pd_rollout_implicit_kernel; aba_body.cuh), and each step of the adjoint runs the implicit ABA adjoint; the integrate and the element-wise step are
// unchanged.
// DRMB200_IMPLICIT_GAINS (PD only, stable PD): u-hat on the predicted position q + dt qd, the per-row pivot addends
// c = dt (kd + dt kp) of the unsaturated joints in the ABA, tau_t = u - c qdd_t (pd_rollout_implicit_gains_kernel; the
// definition is stated in include/drm_b200.h).  Its adjoint recomputes u_t and c_t in the element-wise step, runs the ABA
// adjoint with the addends (backward_aba.cu) and adds the feedback terms of the header.
//
// Forward mapping: the articulated-body kernel's (aba.cu) -- one thread per configuration, T per CTA, the same per-thread
// body (aba_body.cuh) -- with the time loop of rollout_pipeline.cuh inside (rollout_kernel: its own copy).  Once per CTA the table is staged (and folded,
// "rnea_fold") and the (q0, qd0) tile loaded; the state then lives in shared memory for all steps.  Per step the input
// tiles (f, or q_ref | qd_ref | f) arrive by TMA into a double buffer and q / qd / qdd (and tau) leave by bulk store; qdd
// and tau are double-buffered.  rollout_kernel's ABA reads f straight from the input buffer.  pd_rollout_kernel stages
// per-row gains once per CTA, shared gains and limits once as [n] rows, and each thread forms its tau_t row from the live
// s_q / s_qd into the tau tile, which aba_body reads as its f.
// Algorithmic HBM bytes per configuration-step: open loop f in 4n, q / qd / qdd out 12n = 16n (112 B at n = 7; 12n without
// qdd); PD q_ref 4n (+ qd_ref 4n, + f 4n) in, q / qd / qdd / tau 16n out: up to 28n.
//
// Adjoint (drmb200_forward_dynamics_rollout_backward): a host loop t = T-1 ... 0 over the analytic ABA adjoint
// (backward_aba.cu), with running adjoints a_q, a_qd of the state (start at zero):
//   a_q += g_q[t];  a_qd += g_qd[t];  a_qd' = a_qd + dt a_q;  g_qdd_t = dt a_qd' + g_qdd[t]
//   (gq, gqd, gf) = ABA adjoint at (q_t, qd_t, f_t) with g_qdd_t;  f_grad[t] = gf;  a_q += gq;  a_qd = a_qd' + gqd
// and q0_grad = a_q, qd0_grad = a_qd at the end.  One element-wise launch per step fuses the post-update of step t+1 with
// the pre-update of step t; the table gradient of all steps is summed in the adjoint's per-CTA partial tables and reduced
// once, so a backward is 2T + 2 launches.
// drmb200_pd_rollout_backward folds the feedback into the same element-wise step.  With gu_t = mask_t (gf_t + g_tau[t]),
// mask_t = (-lim <= u_t <= lim) (1 without a limit; u_t recomputed bit-exactly), the post-update of step t becomes
//   a_q = (a_q + gq) - kp gu_t;  a_qd = (a_qd' + gqd) - kd gu_t;  f_grad[t] = gu_t;  q_ref_grad[t] = kp gu_t;
//   qd_ref_grad[t] = kd gu_t;  kp_grad += gu_t e_t;  kd_grad += gu_t ed_t      (kp_grad / kd_grad per row, [B, n])
// still 2T + 2 launches, no atomics.
#include "aba_body.cuh"
#include "launch.cuh"
#include "rollout_pipeline.cuh"

namespace drm {

int forward_dynamics_backward_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t,
                                     uint32_t, const float*, float*, float*, float*, float*, void*, cudaStream_t, bool, bool, float,
                                     const float*, float*, float*);
int64_t forward_dynamics_backward_workspace_bytes(const drmb200_topology_t*, int64_t);

// u = (f + kp e) + kd ed with e = q_ref - q, ed = qd_ref - qd: the rounding of the torch expression
// `f + kp * (q_ref - q) + kd * (qd_ref - qd)`; pass 0.f for an absent f / qd_ref (a zero tensor, -0 included)
__device__ __forceinline__ float pd_command(float q_ref, float q, float qd_ref, float qd, float f, float kp, float kd,
                                            float& e, float& ed) {
    e = __fsub_rn(q_ref, q);
    ed = __fsub_rn(qd_ref, qd);
    return __fadd_rn(__fadd_rn(f, __fmul_rn(kp, e)), __fmul_rn(kd, ed));
}

// torch.clamp(u, -lim, lim): NaN propagates
__device__ __forceinline__ float pd_clamp(float u, float lim) {
    return isnan(u) ? u : fminf(fmaxf(u, -lim), lim);
}

struct RolloutArgs {
    const float* __restrict__ table;
    const float* __restrict__ q0;
    const float* __restrict__ qd0;
    const float* __restrict__ f;
    float* __restrict__ q;
    float* __restrict__ qd;
    float* __restrict__ qdd;        // may be null
    int64_t batch;
    int32_t n_steps;
    float dt;
    uint32_t flags;
    int32_t aligned;                // every base 16-byte aligned and batch * n_dofs % 4 == 0: every step's tiles are too
};

struct RolloutSmem {
    int q, qd, f, qdd, table, link, slots, total_floats;
    __host__ __device__ RolloutSmem(int T, int n, int n_links, int n_slots) {
        int o = 0;
        q = o;   o += T * n;
        qd = o;  o += T * n;
        f = o;   o += 2 * T * n;         // double buffer
        qdd = o; o += 2 * T * n;         // double buffer
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o;  o += n_links * ABA_LINK * T;
        slots = o; o += n_slots * ABA_SLOT * T;
        total_floats = o;
    }
};

// The open-loop kernel keeps its own copy of rollout_pipeline.cuh's time loop: built on RolloutPipeline it compiled to a
// different schedule of the ABA body (same registers and stack) that measured 1.5-2.5 % slower on an H100 80GB HBM3 at
// 700 W (DESIGN.md §5), while the PD and contact kernels ran as fast as before.  Its ordering is the pipeline's.
// Its body is instantiated by rollout_kernel and rollout_implicit_kernel (IMPLICIT: the forward dynamics with implicit
// damping of step h = dt, aba_body.cuh), two kernel names rather than a template flag, as for the PD kernel below.
template <int T, bool IMPLICIT>
__device__ __forceinline__ void rollout_run(const TreeProgram& prog, const FoldProgram& fold, const RolloutArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar[2];

    const int n = prog.n_dofs;
    const int N = prog.n_links;
    const RolloutSmem L(T, n, N, prog.n_slots);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_f = smem + L.f;
    float* s_qdd = smem + L.qdd;
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_slot = smem + L.slots;

    const int tid = threadIdx.x;
    const int64_t tile_off = (int64_t)blockIdx.x * T * n;
    const int valid = (int)min((int64_t)T, args.batch - (int64_t)blockIdx.x * T);
    const int tile_floats = valid * n;
    const int64_t step = args.batch * n;                 // floats between the [B, n] slices of consecutive steps
    const bool vec_ok = args.aligned;
    const bool bulk = args.aligned && ((tile_floats & 3) == 0);
    const uint32_t bytes = (uint32_t)tile_floats * 4u;

    if (bulk) {
        if (tid == 0) {
            mbar_init(&mbar[0], 1);
            mbar_init(&mbar[1], 1);
            fence_mbar_init();
            mbar_arrive_expect_tx(&mbar[0], 3u * bytes);
            bulk_g2s(s_q, args.q0 + tile_off, bytes, &mbar[0]);
            bulk_g2s(s_qd, args.qd0 + tile_off, bytes, &mbar[0]);
            bulk_g2s(s_f, args.f + tile_off, bytes, &mbar[0]);
        }
    } else {
        coop_copy(s_q, args.q0 + tile_off, tile_floats, vec_ok);
        coop_copy(s_qd, args.qd0 + tile_off, tile_floats, vec_ok);
    }
    if (fold.n_red > 0) stage_folded_table(s_tab, s_link, args.table, fold, prog, T);
    else stage_canonical_table(s_tab, args.table, prog, T);
    __syncthreads();

    const float dt = args.dt;
    for (int t = 0; t < args.n_steps; ++t) {
        const int b = t & 1;
        float* s_ft = s_f + b * T * n;
        float* s_qddt = s_qdd + b * T * n;
        if (bulk) {
            // buffer b ^ 1 was last read by the passes of step t - 1, which every thread finished (and fenced against the
            // async proxy) before the barrier that ended step t - 1
            if (tid == 0 && t + 1 < args.n_steps) {
                mbar_arrive_expect_tx(&mbar[b ^ 1], bytes);
                bulk_g2s(s_f + (b ^ 1) * T * n, args.f + (t + 1) * step + tile_off, bytes, &mbar[b ^ 1]);
            }
            mbar_wait(&mbar[b], (uint32_t)(t >> 1) & 1u);
        } else {
            coop_copy(s_ft, args.f + t * step + tile_off, tile_floats, vec_ok);
            __syncthreads();
        }

        if (tid < valid)
            aba_body<T, IMPLICIT>(prog, s_tab, s_q + tid * n, s_qd + tid * n, s_ft + tid * n, s_qddt + tid * n, s_link + tid,
                                  s_slot + tid, args.flags, dt);

        if (bulk) {
            if (tid == 0) bulk_wait_read<0>();           // the stores of step t - 1 have read s_q / s_qd
            __syncthreads();
        }
        if (tid < valid) {
            float* qr = s_q + tid * n;
            float* qdr = s_qd + tid * n;
            const float* ar = s_qddt + tid * n;
            for (int k = 0; k < n; ++k) {
                const float v = __fadd_rn(qdr[k], __fmul_rn(dt, ar[k]));
                qdr[k] = v;
                qr[k] = __fadd_rn(qr[k], __fmul_rn(dt, v));
            }
        }
        if (bulk) {
            fence_proxy_async();
            __syncthreads();
            if (tid == 0) {
                bulk_s2g(args.q + t * step + tile_off, s_q, bytes);
                bulk_s2g(args.qd + t * step + tile_off, s_qd, bytes);
                if (args.qdd != nullptr) bulk_s2g(args.qdd + t * step + tile_off, s_qddt, bytes);
                bulk_commit();
            }
        } else {
            __syncthreads();
            coop_copy(args.q + t * step + tile_off, s_q, tile_floats, vec_ok);
            coop_copy(args.qd + t * step + tile_off, s_qd, tile_floats, vec_ok);
            if (args.qdd != nullptr) coop_copy(args.qdd + t * step + tile_off, s_qddt, tile_floats, vec_ok);
            // the next step's integrate rewrites s_q / s_qd only after the barrier that follows its f copy
        }
    }
    if (bulk && tid == 0) bulk_wait_read<0>();
}

template <int T>
__global__ void __launch_bounds__(T)
rollout_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const RolloutArgs args) {
    rollout_run<T, false>(prog, fold, args);
}

template <int T>
__global__ void __launch_bounds__(T)
rollout_implicit_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold,
                        const RolloutArgs args) {
    rollout_run<T, true>(prog, fold, args);
}

struct PDRolloutArgs {
    const float* __restrict__ table;
    const float* __restrict__ q0;
    const float* __restrict__ qd0;
    const float* __restrict__ q_ref;
    const float* __restrict__ qd_ref;   // may be null
    const float* __restrict__ f;        // may be null
    const float* __restrict__ kp;       // [n] or [B, n]
    const float* __restrict__ kd;
    const float* __restrict__ lim;      // [n], may be null
    float* __restrict__ q;
    float* __restrict__ qd;
    float* __restrict__ qdd;            // may be null
    float* __restrict__ tau;
    int64_t batch;
    int32_t n_steps;
    float dt;
    uint32_t flags;
    int32_t per_row;                    // kp / kd are [B, n]
    int32_t aligned;                    // as RolloutArgs, over every tile pointer (and kp / kd when per row)
};

struct PDRolloutSmem {
    int q, qd, in, tau, qdd, kp, kd, lim, table, link, slots, piv, total_floats;
    // n_in input tiles per step (q_ref, then qd_ref and f when given); every region starts 16-byte aligned.  gains: the
    // implicit gains' per-row pivot addends c of the current step, [T, n] after every other region (empty without)
    __host__ __device__ PDRolloutSmem(int T, int n, int n_links, int n_slots, int n_in, bool per_row, bool gains = false) {
        const int gain = ((per_row ? T : 1) * n + 3) & ~3;
        int o = 0;
        q = o;   o += T * n;
        qd = o;  o += T * n;
        in = o;  o += 2 * n_in * T * n;  // double buffer
        tau = o; o += 2 * T * n;         // double buffer
        qdd = o; o += 2 * T * n;         // double buffer
        kp = o;  o += gain;
        kd = o;  o += gain;
        lim = o; o += (n + 3) & ~3;
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o;  o += n_links * ABA_LINK * T;
        slots = o; o += n_slots * ABA_SLOT * T;
        piv = o;   o += gains ? T * n : 0;
        total_floats = o;
    }
};

// The PD kernel's body, instantiated by pd_rollout_kernel (explicit damping), pd_rollout_implicit_kernel and
// pd_rollout_implicit_gains_kernel: kernel names rather than a template flag on one, so that the explicit kernel keeps its
// symbol.  GAINS (DRMB200_IMPLICIT_GAINS): each thread forms u_t into its tau row and c_t into its row of the addend tile,
// the ABA runs with the pivot addends c_t, and the tau row then becomes u_t - c_t qdd_t on the unsaturated joints.
template <int T, bool IMPLICIT, bool GAINS = false>
__device__ __forceinline__ void pd_rollout_run(const TreeProgram& prog, const FoldProgram& fold, const PDRolloutArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar[2];

    const int n = prog.n_dofs;
    const bool has_qdr = args.qd_ref != nullptr, has_f = args.f != nullptr, has_lim = args.lim != nullptr;
    const int n_in = 1 + (int)has_qdr + (int)has_f;
    const PDRolloutSmem L(T, n, prog.n_links, prog.n_slots, n_in, args.per_row != 0, GAINS);
    float* s_tau = smem + L.tau;
    float* s_qdd = smem + L.qdd;
    float* s_kp = smem + L.kp;
    float* s_kd = smem + L.kd;
    float* s_lim = smem + L.lim;
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_slot = smem + L.slots;
    const int tid = threadIdx.x;
    const int o_f = (has_qdr ? 2 : 1) * T * n;          // tiles of one input buffer: q_ref | qd_ref | f

    const RolloutPipeline<T> pipe(mbar, smem + L.q, smem + L.qd, smem + L.in, args.q_ref, args.qd_ref, args.f, args.q, args.qd,
                                  n, args.batch, args.n_steps, args.dt, args.aligned);
    pipe.begin(args.q0, args.qd0);
    if (args.per_row) {
        coop_copy(s_kp, args.kp + pipe.tile_off, pipe.tile_floats, pipe.vec_ok);
        coop_copy(s_kd, args.kd + pipe.tile_off, pipe.tile_floats, pipe.vec_ok);
    } else {
        coop_copy(s_kp, args.kp, n, false);
        coop_copy(s_kd, args.kd, n, false);
    }
    if (has_lim) coop_copy(s_lim, args.lim, n, false);
    if (fold.n_red > 0) stage_folded_table(s_tab, s_link, args.table, fold, prog, T);
    else stage_canonical_table(s_tab, args.table, prog, T);
    __syncthreads();

    const int gain_row = args.per_row ? tid * n : 0;
    for (int t = 0; t < args.n_steps; ++t) {
        const float* s_it = pipe.fetch(t);
        float* s_taut = s_tau + (t & 1) * T * n;
        float* s_qddt = s_qdd + (t & 1) * T * n;
        if (tid < pipe.valid) {
            const float* qr = pipe.s_q + tid * n;
            const float* qdr = pipe.s_qd + tid * n;
            const float* ref = s_it + tid * n;
            float* taur = s_taut + tid * n;
            if constexpr (GAINS) {
                const float h = args.dt;
                float* cr = smem + L.piv + tid * n;
                float* ar = s_qddt + tid * n;
                uint64_t sat = 0;                                // n <= 63
                for (int k = 0; k < n; ++k) {
                    const float kp = s_kp[gain_row + k], kd = s_kd[gain_row + k];
                    const float qp = __fadd_rn(qr[k], __fmul_rn(h, qdr[k]));      // the position the step predicts
                    float e, ed;
                    const float u = pd_command(ref[k], qp, has_qdr ? ref[T * n + k] : 0.f, qdr[k], has_f ? ref[o_f + k] : 0.f,
                                               kp, kd, e, ed);
                    const bool s = has_lim && !(u >= -s_lim[k] && u <= s_lim[k]);   // torch.clamp's rule, NaN saturated
                    sat |= (uint64_t)s << k;
                    taur[k] = s ? pd_clamp(u, s_lim[k]) : u;
                    cr[k] = s ? 0.f : __fmul_rn(h, __fadd_rn(kd, __fmul_rn(h, kp)));
                }
                aba_body<T, IMPLICIT, true>(prog, s_tab, qr, qdr, taur, ar, s_link + tid, s_slot + tid, args.flags, h, cr);
                for (int k = 0; k < n; ++k)
                    if (!((sat >> k) & 1)) taur[k] = __fsub_rn(taur[k], __fmul_rn(cr[k], ar[k]));
            } else {
                for (int k = 0; k < n; ++k) {
                    float e, ed;
                    const float u = pd_command(ref[k], qr[k], has_qdr ? ref[T * n + k] : 0.f, qdr[k], has_f ? ref[o_f + k] : 0.f,
                                               s_kp[gain_row + k], s_kd[gain_row + k], e, ed);
                    taur[k] = has_lim ? pd_clamp(u, s_lim[k]) : u;
                }
                aba_body<T, IMPLICIT>(prog, s_tab, qr, qdr, taur, s_qddt + tid * n, s_link + tid, s_slot + tid, args.flags,
                                      args.dt);
            }
        }
        pipe.integrate_and_store(t, s_qddt + tid * n, 1, args.tau, s_taut, args.qdd, s_qddt);
    }
    pipe.finish();
}

template <int T>
__global__ void __launch_bounds__(T)
pd_rollout_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const PDRolloutArgs args) {
    pd_rollout_run<T, false>(prog, fold, args);
}

template <int T>
__global__ void __launch_bounds__(T)
pd_rollout_implicit_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold,
                           const PDRolloutArgs args) {
    pd_rollout_run<T, true>(prog, fold, args);
}

// DRMB200_IMPLICIT_GAINS, with explicit (IMPLICIT = false) or implicit joint damping
template <int T, bool IMPLICIT>
__global__ void __launch_bounds__(T)
pd_rollout_implicit_gains_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold,
                                 const PDRolloutArgs args) {
    pd_rollout_run<T, IMPLICIT, true>(prog, fold, args);
}

// ---------------------------------------------------------------------------------------------
// adjoint: the element-wise update between two ABA adjoint launches, the post-update of step s = t + 1 fused with the
// pre-update of step t.  Feedback adds the PD terms to the post-update; without it the fields of the feedback block are
// unused.
// ---------------------------------------------------------------------------------------------
struct AdjStepArgs {
    float* a_q;                 // running adjoints of q_t / qd_t  [B, n]
    float* a_qd;
    float* g_step;              // g_qdd_t handed to the ABA adjoint
    const float* gq;            // ABA adjoint of step s (post-update; unused when first)
    const float* gqd;
    // feedback: step s of the post-update -- its state, inputs, upstream g_tau (NULL = zero) and outputs (NULL = not wanted)
    const float* gf;
    const float* qs;
    const float* qds;
    const float* q_ref;
    const float* qd_ref;
    const float* f;
    const float* g_tau;
    float* f_grad;
    float* q_ref_grad;
    float* qd_ref_grad;
    float* kp_grad;             // [B, n] running sums over the steps (NULL = not wanted)
    float* kd_grad;
    const float* kp;
    const float* kd;
    const float* lim;
    int32_t n;
    int32_t per_row;
    int32_t last_post;          // s = T - 1: kp_grad / kd_grad are written rather than accumulated
    // step t of the pre-update
    const float* g_q;           // upstream gradients of step t, NULL = zero
    const float* g_qd;
    const float* g_qdd;
    float* out_q;               // final: q0_grad / qd0_grad (NULL = not wanted)
    float* out_qd;
    int64_t count;
    float dt;
    int32_t first;              // t = T - 1: the running adjoints start at zero
    int32_t final;              // after step 0: post-update only, written to out_q / out_qd
    // implicit gains: the pivot adjoint c-bar and the accelerations of step s (the ABA adjoint's outputs); step t's state,
    // inputs and upstream g_tau, and its u_t / c_t for the ABA adjoint (written)
    const float* c_bar;
    const float* qdd_s;
    const float* qt;
    const float* qdt;
    const float* q_ref_t;
    const float* qd_ref_t;
    const float* f_t;
    const float* g_tau_t;
    float* u_step;
    float* c_step;
};

// The implicit gains' command of a step (drmb200_pd_rollout, DRMB200_IMPLICIT_GAINS) at element i: u-hat on the predicted
// position q + h qd, whether it saturates (torch.clamp's rule, NaN saturated) and its e, ed.  q_ref / qd_ref / f / lim are
// the step's (qd_ref / f / lim may be NULL).
__device__ __forceinline__ float pd_gains_command(const AdjStepArgs& a, int64_t i, const float* q, const float* qd,
                                                  const float* q_ref, const float* qd_ref, const float* f, float kp, float kd,
                                                  float& e, float& ed, bool& sat) {
    const int k = (int)(i % a.n);
    const float qp = __fadd_rn(q[i], __fmul_rn(a.dt, qd[i]));
    const float u = pd_command(q_ref[i], qp, qd_ref ? qd_ref[i] : 0.f, qd[i], f ? f[i] : 0.f, kp, kd, e, ed);
    sat = a.lim != nullptr && !(u >= -a.lim[k] && u <= a.lim[k]);
    return u;
}

// Gains (only with Feedback): the adjoint of the implicit gains.  The pre-update of step t also recomputes u_t, c_t (for
// the ABA adjoint) and adds -c_t g_tau[t] to g_qdd_t; the post-update of step s takes, with gu = mask (gf + g_tau) and
// gc = mask (c-bar - qdd_s g_tau), a_q -= kp gu, a_qd -= (kd + h kp) gu, f_grad = gu, q_ref_grad = kp gu,
// qd_ref_grad = kd gu, kp_grad += gu e + h^2 gc, kd_grad += gu ed + h gc.
template <bool Feedback, bool Gains>
__device__ __forceinline__ void rollout_adjoint_step(const AdjStepArgs& a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.count; i += (int64_t)gridDim.x * blockDim.x) {
        float aq = 0.f, aqd = 0.f;
        if (!a.first) {                                        // post-update of step s
            if constexpr (Gains) {
                const int64_t gi = a.per_row ? i : (int)(i % a.n);
                const float kp = a.kp[gi], kd = a.kd[gi], h = a.dt;
                float e, ed;
                bool sat;
                pd_gains_command(a, i, a.qs, a.qds, a.q_ref, a.qd_ref, a.f, kp, kd, e, ed, sat);
                float gu = a.gf[i], gc = a.c_bar[i];
                if (a.g_tau != nullptr) {
                    gu = __fadd_rn(gu, a.g_tau[i]);
                    gc = __fsub_rn(gc, __fmul_rn(a.qdd_s[i], a.g_tau[i]));
                }
                if (sat) gu = gc = 0.f;
                aq = __fsub_rn(__fadd_rn(a.a_q[i], a.gq[i]), __fmul_rn(kp, gu));
                aqd = __fsub_rn(__fadd_rn(a.a_qd[i], a.gqd[i]), __fmul_rn(__fadd_rn(kd, __fmul_rn(h, kp)), gu));
                if (a.f_grad != nullptr) a.f_grad[i] = gu;
                if (a.q_ref_grad != nullptr) a.q_ref_grad[i] = __fmul_rn(kp, gu);
                if (a.qd_ref_grad != nullptr) a.qd_ref_grad[i] = __fmul_rn(kd, gu);
                const float gkp = __fadd_rn(__fmul_rn(gu, e), __fmul_rn(__fmul_rn(h, h), gc));
                const float gkd = __fadd_rn(__fmul_rn(gu, ed), __fmul_rn(h, gc));
                if (a.kp_grad != nullptr) a.kp_grad[i] = a.last_post ? gkp : __fadd_rn(a.kp_grad[i], gkp);
                if (a.kd_grad != nullptr) a.kd_grad[i] = a.last_post ? gkd : __fadd_rn(a.kd_grad[i], gkd);
            } else if constexpr (Feedback) {
                const int k = (int)(i % a.n);
                const int64_t gi = a.per_row ? i : k;
                const float kp = a.kp[gi], kd = a.kd[gi];
                float e, ed;
                const float u = pd_command(a.q_ref[i], a.qs[i], a.qd_ref ? a.qd_ref[i] : 0.f, a.qds[i], a.f ? a.f[i] : 0.f, kp,
                                           kd, e, ed);
                float gu = a.gf[i];
                if (a.g_tau != nullptr) gu = __fadd_rn(gu, a.g_tau[i]);
                if (a.lim != nullptr && !(u >= -a.lim[k] && u <= a.lim[k])) gu = 0.f;   // torch.clamp's rule: equality passes
                aq = __fsub_rn(__fadd_rn(a.a_q[i], a.gq[i]), __fmul_rn(kp, gu));
                aqd = __fsub_rn(__fadd_rn(a.a_qd[i], a.gqd[i]), __fmul_rn(kd, gu));
                if (a.f_grad != nullptr) a.f_grad[i] = gu;
                if (a.q_ref_grad != nullptr) a.q_ref_grad[i] = __fmul_rn(kp, gu);
                if (a.qd_ref_grad != nullptr) a.qd_ref_grad[i] = __fmul_rn(kd, gu);
                if (a.kp_grad != nullptr) a.kp_grad[i] = a.last_post ? __fmul_rn(gu, e) : __fadd_rn(a.kp_grad[i], __fmul_rn(gu, e));
                if (a.kd_grad != nullptr) a.kd_grad[i] = a.last_post ? __fmul_rn(gu, ed) : __fadd_rn(a.kd_grad[i], __fmul_rn(gu, ed));
            } else {
                aq = __fadd_rn(a.a_q[i], a.gq[i]);
                aqd = __fadd_rn(a.a_qd[i], a.gqd[i]);
            }
        }
        if (a.final) {
            if (a.out_q != nullptr) a.out_q[i] = aq;
            if (a.out_qd != nullptr) a.out_qd[i] = aqd;
            continue;
        }
        if (a.g_q != nullptr) aq = __fadd_rn(aq, a.g_q[i]);    // pre-update of step t
        if (a.g_qd != nullptr) aqd = __fadd_rn(aqd, a.g_qd[i]);
        aqd = __fadd_rn(aqd, __fmul_rn(a.dt, aq));             // a_qd' = a_qd + dt a_q
        float g = __fmul_rn(a.dt, aqd);
        if (a.g_qdd != nullptr) g = __fadd_rn(g, a.g_qdd[i]);
        if constexpr (Gains) {                                 // u_t, c_t as the forward formed them
            const int k = (int)(i % a.n);
            const int64_t gi = a.per_row ? i : k;
            const float kp = a.kp[gi], kd = a.kd[gi], h = a.dt;
            float e, ed;
            bool sat;
            const float u = pd_gains_command(a, i, a.qt, a.qdt, a.q_ref_t, a.qd_ref_t, a.f_t, kp, kd, e, ed, sat);
            const float c = sat ? 0.f : __fmul_rn(h, __fadd_rn(kd, __fmul_rn(h, kp)));
            a.u_step[i] = sat ? pd_clamp(u, a.lim[k]) : u;
            a.c_step[i] = c;
            if (a.g_tau_t != nullptr) g = __fsub_rn(g, __fmul_rn(c, a.g_tau_t[i]));
        }
        a.a_q[i] = aq;
        a.a_qd[i] = aqd;
        a.g_step[i] = g;
    }
}

template <bool Feedback>
__global__ void __launch_bounds__(256) rollout_adjoint_step_kernel(const AdjStepArgs a) {
    rollout_adjoint_step<Feedback, false>(a);
}

__global__ void __launch_bounds__(256) pd_rollout_implicit_gains_adjoint_step_kernel(const AdjStepArgs a) {
    rollout_adjoint_step<true, true>(a);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// "rnea_fold", as drmb200_forward_dynamics, and the checks both forward rollouts start with (pd: the PD rollout's)
static int rollout_program(const drmb200_topology_t* topo, int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                           bool pd, FoldChoice* fc) {
    const int rc = select_fold(topo, false, fc);
    if (rc != DRMB200_OK) return rc;
    if (batch < 0 || n_steps < 0) { set_error("batch=%lld, n_steps=%d: must be >= 0", (long long)batch, (int)n_steps); return DRMB200_EINVAL; }
    const int rd = check_implicit_damping(flags, dt);
    return rd != DRMB200_OK ? rd : check_implicit_gains(flags, dt, pd);
}

// 64 configurations per CTA when that still gives every SM a CTA and the per-link state leaves room for two CTAs per SM;
// 32 otherwise -- rollout batches are often below one wave of 64-thread CTAs, and a CTA stays resident for all steps.
// With Kern16 (the PD rollout's), a 32-row CTA that exceeds SMEM_CTA_MAX with the kernel's static shared memory falls
// back to 16 rows, refused only when that still does not fit: the PD layout's input streams and per-row gains push a
// 63-DoF chain past the limit at 32 rows.  The open-loop rollout's 32-row CTA fits every model the engine accepts.  A
// folded model only needs the 16-row rung with more than 50 reduced links, whose per-link state (14 x 16 floats each)
// still holds the fold's staging scratch (40 floats per original link, at most 64 links).
// floats_of(T) is the kernel's dynamic shared memory in floats.
template <auto Kern64, auto Kern32, auto Kern16 = nullptr, typename Args, typename F>
static int launch_rollout(const FoldChoice& fc, int64_t batch, F floats_of, const char* what, const Args& args,
                          cudaStream_t stream) {
    auto bytes_of = [&](int T) { return (size_t)floats_of(T) * sizeof(float); };
    TileChoice c = tile_64_or_32(bytes_of, 0, (batch + 63) / 64 >= device_sm_count());
    size_t static_bytes = 0;
    if constexpr (!std::is_same_v<decltype(Kern16), std::nullptr_t>) {
        const int rc = static_smem_bytes<Kern32>(&static_bytes);
        if (rc != DRMB200_OK) return rc;
        if (c.bytes + static_bytes > SMEM_CTA_MAX) c = {16, bytes_of(16)};
    }
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("model needs %zu B of shared memory per CTA (> 227 KB)", c.bytes + static_bytes);
        return DRMB200_ELIMIT;
    }
    const int64_t tiles = (batch + c.tile - 1) / c.tile;
    if constexpr (!std::is_same_v<decltype(Kern16), std::nullptr_t>) {
        if (c.tile == 16) return launch_kernel<Kern16>(tiles, 16, c.bytes, stream, false, what, *fc.prog, fc.fold, args);
    }
    return c.tile == 64 ? launch_kernel<Kern64>(tiles, 64, c.bytes, stream, false, what, *fc.prog, fc.fold, args)
                        : launch_kernel<Kern32>(tiles, 32, c.bytes, stream, false, what, *fc.prog, fc.fold, args);
}

int forward_dynamics_rollout_device(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                                    const float* f, int64_t batch, int32_t n_steps, float dt, uint32_t flags, float* q,
                                    float* qd, float* qdd, cudaStream_t stream) {
    FoldChoice fc;
    const int rc = rollout_program(topo, batch, n_steps, dt, flags, false, &fc);
    if (rc != DRMB200_OK) return rc;
    const TreeProgram& prog = *fc.prog;
    if (batch == 0 || n_steps == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q0 == nullptr || qd0 == nullptr || f == nullptr || q == nullptr || qd == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }

    RolloutArgs args;
    args.table = table; args.q0 = q0; args.qd0 = qd0; args.f = f; args.q = q; args.qd = qd; args.qdd = qdd;
    args.batch = batch; args.n_steps = n_steps; args.dt = dt; args.flags = flags;
    args.aligned = aligned16(q0, qd0, f, q, qd, qdd) && ((batch * prog.n_dofs) & 3) == 0;
    auto floats_of = [&](int T) { return RolloutSmem(T, prog.n_dofs, prog.n_links, prog.n_slots).total_floats; };
    if (flags & DRMB200_IMPLICIT_DAMPING)
        return launch_rollout<rollout_implicit_kernel<64>, rollout_implicit_kernel<32>>(fc, batch, floats_of, "rollout", args, stream);
    return launch_rollout<rollout_kernel<64>, rollout_kernel<32>>(fc, batch, floats_of, "rollout", args, stream);
}

int pd_rollout_device(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0, const float* q_ref,
                      const float* qd_ref, const float* f, const float* kp, const float* kd, int32_t gains_per_row,
                      const float* effort_limit, int64_t batch, int32_t n_steps, float dt, uint32_t flags, float* q, float* qd,
                      float* qdd, float* tau, cudaStream_t stream) {
    FoldChoice fc;
    const int rc = rollout_program(topo, batch, n_steps, dt, flags, true, &fc);
    if (rc != DRMB200_OK) return rc;
    const TreeProgram& prog = *fc.prog;
    if (gains_per_row != 0 && gains_per_row != 1) { set_error("gains_per_row=%d: must be 0 or 1", (int)gains_per_row); return DRMB200_EINVAL; }
    if (batch == 0 || n_steps == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q0 == nullptr || qd0 == nullptr || q_ref == nullptr || kp == nullptr || kd == nullptr ||
        q == nullptr || qd == nullptr || tau == nullptr) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }

    PDRolloutArgs args;
    args.table = table; args.q0 = q0; args.qd0 = qd0; args.q_ref = q_ref; args.qd_ref = qd_ref; args.f = f;
    args.kp = kp; args.kd = kd; args.lim = effort_limit; args.q = q; args.qd = qd; args.qdd = qdd; args.tau = tau;
    args.batch = batch; args.n_steps = n_steps; args.dt = dt; args.flags = flags; args.per_row = gains_per_row;
    args.aligned = aligned16(q0, qd0, q_ref, qd_ref, f, q, qd, qdd, tau) && (!gains_per_row || aligned16(kp, kd)) &&
                   ((batch * prog.n_dofs) & 3) == 0;
    const int n_in = 1 + (qd_ref != nullptr) + (f != nullptr);
    if (flags & DRMB200_IMPLICIT_GAINS) {
        auto gains_floats_of = [&](int T) {
            return PDRolloutSmem(T, prog.n_dofs, prog.n_links, prog.n_slots, n_in, gains_per_row != 0, true).total_floats;
        };
        if (flags & DRMB200_IMPLICIT_DAMPING)
            return launch_rollout<pd_rollout_implicit_gains_kernel<64, true>, pd_rollout_implicit_gains_kernel<32, true>,
                                  pd_rollout_implicit_gains_kernel<16, true>>(fc, batch, gains_floats_of, "pd rollout", args,
                                                                              stream);
        return launch_rollout<pd_rollout_implicit_gains_kernel<64, false>, pd_rollout_implicit_gains_kernel<32, false>,
                              pd_rollout_implicit_gains_kernel<16, false>>(fc, batch, gains_floats_of, "pd rollout", args,
                                                                           stream);
    }
    auto floats_of = [&](int T) {
        return PDRolloutSmem(T, prog.n_dofs, prog.n_links, prog.n_slots, n_in, gains_per_row != 0).total_floats;
    };
    if (flags & DRMB200_IMPLICIT_DAMPING)
        return launch_rollout<pd_rollout_implicit_kernel<64>, pd_rollout_implicit_kernel<32>, pd_rollout_implicit_kernel<16>>(
            fc, batch, floats_of, "pd rollout", args, stream);
    return launch_rollout<pd_rollout_kernel<64>, pd_rollout_kernel<32>, pd_rollout_kernel<16>>(fc, batch, floats_of,
                                                                                              "pd rollout", args, stream);
}

// The reverse-time adjoint of both rollouts.  Workspace: [ABA adjoint workspace | a_q | a_qd | g_qdd_t | gq | gqd (| gf
// with feedback | u_t | c_t | c-bar | qdd for the implicit gains)], each [B, n] fp32.  The feedback bound covers the
// implicit gains, with or without them.
int64_t rollout_adjoint_workspace_bytes(const drmb200_topology_t* topo, int64_t batch, bool feedback) {
    if (topo == nullptr || topo->n_links < 1 || topo->n_links > DRMB200_MAX_LINKS || batch < 0) return 0;
    return round256(forward_dynamics_backward_workspace_bytes(topo, batch)) +
           (feedback ? 10 : 5) * round256(batch * topo->n_dofs * (int64_t)sizeof(float));
}

// tau: the [T, B, n] torques the forward applied.  Open loop (fb == NULL): f_grad receives the ABA adjoint's f gradient.
// With feedback, fb holds the kernel's PD fields and [T, B, n] bases of its per-step inputs and gradients, which the loop
// offsets to each step; the ABA adjoint's f gradient goes to the gf slice.  want_final: q0_grad, qd0_grad or a feedback
// gradient is wanted, so the post-update of step 0 runs.
static int rollout_adjoint(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                           const float* tau, int64_t batch, int32_t n_steps, float dt, uint32_t flags, const float* q,
                           const float* qd, const float* g_q, const float* g_qd, const float* g_qdd, float* q0_grad,
                           float* qd0_grad, float* f_grad, float* table_grad, const AdjStepArgs* fb, bool want_final,
                           void* workspace, cudaStream_t stream) {
    const int64_t count = batch * topo->n_dofs;
    const int64_t slice = round256(count * (int64_t)sizeof(float));
    char* ws = static_cast<char*>(workspace);
    void* fd_ws = ws;
    ws += round256(forward_dynamics_backward_workspace_bytes(topo, batch));
    float* a_q = reinterpret_cast<float*>(ws);
    float* a_qd = reinterpret_cast<float*>(ws + slice);
    float* g_step = reinterpret_cast<float*>(ws + 2 * slice);
    float* gq = reinterpret_cast<float*>(ws + 3 * slice);
    float* gqd = reinterpret_cast<float*>(ws + 4 * slice);
    float* gf = fb ? reinterpret_cast<float*>(ws + 5 * slice) : nullptr;
    const bool gains = fb != nullptr && (flags & DRMB200_IMPLICIT_GAINS);
    float* u_step = gains ? reinterpret_cast<float*>(ws + 6 * slice) : nullptr;
    float* c_step = gains ? reinterpret_cast<float*>(ws + 7 * slice) : nullptr;
    float* c_bar = gains ? reinterpret_cast<float*>(ws + 8 * slice) : nullptr;
    float* qdd_s = gains ? reinterpret_cast<float*>(ws + 9 * slice) : nullptr;

    int64_t blocks = (count + 255) / 256;
    if (blocks > (int64_t)device_sm_count() * 8) blocks = (int64_t)device_sm_count() * 8;
    auto step_kernel = [&](const AdjStepArgs& a) {
        if (gains)
            return launch_kernel<pd_rollout_implicit_gains_adjoint_step_kernel>(blocks, 256, 0, stream, false,
                                                                                "pd rollout adjoint step", a);
        return fb ? launch_kernel<rollout_adjoint_step_kernel<true>>(blocks, 256, 0, stream, false, "pd rollout adjoint step", a)
                  : launch_kernel<rollout_adjoint_step_kernel<false>>(blocks, 256, 0, stream, false, "rollout adjoint step", a);
    };
    auto at = [&](auto* p, int s) { return p ? p + (int64_t)s * count : nullptr; };

    AdjStepArgs a = fb ? *fb : AdjStepArgs{};
    a.a_q = a_q; a.a_qd = a_qd; a.g_step = g_step; a.gq = gq; a.gqd = gqd; a.gf = gf;
    a.n = topo->n_dofs; a.count = count; a.dt = dt;
    a.c_bar = c_bar; a.qdd_s = qdd_s; a.u_step = u_step; a.c_step = c_step;
    // the feedback post-update of step s reads its state (q0 / qd0, then the forward's outputs) and inputs, writes its
    // gradients
    auto post = [&](int s) {
        if (fb == nullptr) return;
        a.qs = s == 0 ? q0 : q + (int64_t)(s - 1) * count;
        a.qds = s == 0 ? qd0 : qd + (int64_t)(s - 1) * count;
        a.q_ref = at(fb->q_ref, s); a.qd_ref = at(fb->qd_ref, s); a.f = at(fb->f, s); a.g_tau = at(fb->g_tau, s);
        a.f_grad = at(fb->f_grad, s); a.q_ref_grad = at(fb->q_ref_grad, s); a.qd_ref_grad = at(fb->qd_ref_grad, s);
        a.last_post = s == n_steps - 1;
    };
    for (int t = n_steps - 1; t >= 0; --t) {
        a.first = (t == n_steps - 1) ? 1 : 0;
        a.final = 0;
        if (!a.first) post(t + 1);
        a.g_q = at(g_q, t);
        a.g_qd = at(g_qd, t);
        a.g_qdd = at(g_qdd, t);
        const float* qt = t == 0 ? q0 : q + (int64_t)(t - 1) * count;     // step inputs: (q0, qd0), then the forward's outputs
        const float* qdt = t == 0 ? qd0 : qd + (int64_t)(t - 1) * count;
        if (gains) {
            a.qt = qt; a.qdt = qdt;
            a.q_ref_t = at(fb->q_ref, t); a.qd_ref_t = at(fb->qd_ref, t); a.f_t = at(fb->f, t); a.g_tau_t = at(fb->g_tau, t);
        }
        int rc = step_kernel(a);
        if (rc != DRMB200_OK) return rc;
        // the implicit gains' ABA ran on u_t with the pivot addends c_t (the pre-update just wrote both), not on tau_t
        rc = forward_dynamics_backward_device(topo, table, qt, qdt, gains ? u_step : tau + (int64_t)t * count, batch, flags,
                                              g_step, gq, gqd, fb ? gf : at(f_grad, t), table_grad, fd_ws, stream,
                                              /*accumulate_partials=*/t != n_steps - 1, /*reduce=*/t == 0, dt, c_step, c_bar,
                                              qdd_s);
        if (rc != DRMB200_OK) return rc;
    }
    if (!want_final) return DRMB200_OK;
    a.first = 0;
    a.final = 1;
    post(0);
    a.out_q = q0_grad;
    a.out_qd = qd0_grad;
    return step_kernel(a);
}

int64_t forward_dynamics_rollout_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    return rollout_adjoint_workspace_bytes(topo, batch, false);
}

int forward_dynamics_rollout_backward_device(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                                             const float* f, int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                                             const float* q, const float* qd, const float* g_q, const float* g_qd,
                                             const float* g_qdd, float* q0_grad, float* qd0_grad, float* f_grad,
                                             float* table_grad, void* workspace, cudaStream_t stream) {
    if (topo == nullptr) { set_error("null topology"); return DRMB200_EINVAL; }
    if (batch < 0 || n_steps < 0) { set_error("batch=%lld, n_steps=%d: must be >= 0", (long long)batch, (int)n_steps); return DRMB200_EINVAL; }
    if (check_implicit_damping(flags, dt) != DRMB200_OK) return DRMB200_EINVAL;
    if (check_implicit_gains(flags, dt, false) != DRMB200_OK) return DRMB200_EINVAL;
    if (batch == 0 || n_steps == 0 || topo->n_dofs == 0) return DRMB200_OK;
    if (q0_grad == nullptr && qd0_grad == nullptr && f_grad == nullptr && table_grad == nullptr) return DRMB200_OK;
    if (table == nullptr || q0 == nullptr || qd0 == nullptr || f == nullptr || (n_steps > 1 && (q == nullptr || qd == nullptr))) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    if (workspace == nullptr) { set_error("rollout backward needs its workspace (drmb200_forward_dynamics_rollout_backward_workspace_bytes)"); return DRMB200_EINVAL; }
    return rollout_adjoint(topo, table, q0, qd0, f, batch, n_steps, dt, flags, q, qd, g_q, g_qd, g_qdd, q0_grad, qd0_grad,
                           f_grad, table_grad, nullptr, q0_grad != nullptr || qd0_grad != nullptr, workspace, stream);
}

int64_t pd_rollout_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    return rollout_adjoint_workspace_bytes(topo, batch, true);
}

int pd_rollout_backward_device(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                               const float* q_ref, const float* qd_ref, const float* f, const float* kp, const float* kd,
                               int32_t gains_per_row, const float* effort_limit, int64_t batch, int32_t n_steps, float dt,
                               uint32_t flags, const float* q, const float* qd, const float* tau, const float* g_q,
                               const float* g_qd, const float* g_qdd, const float* g_tau, float* q0_grad, float* qd0_grad,
                               float* q_ref_grad, float* qd_ref_grad, float* f_grad, float* kp_grad, float* kd_grad,
                               float* table_grad, void* workspace, cudaStream_t stream) {
    if (topo == nullptr) { set_error("null topology"); return DRMB200_EINVAL; }
    if (batch < 0 || n_steps < 0) { set_error("batch=%lld, n_steps=%d: must be >= 0", (long long)batch, (int)n_steps); return DRMB200_EINVAL; }
    if (check_implicit_damping(flags, dt) != DRMB200_OK) return DRMB200_EINVAL;
    if (check_implicit_gains(flags, dt, true) != DRMB200_OK) return DRMB200_EINVAL;
    if (gains_per_row != 0 && gains_per_row != 1) { set_error("gains_per_row=%d: must be 0 or 1", (int)gains_per_row); return DRMB200_EINVAL; }
    if (batch == 0 || n_steps == 0 || topo->n_dofs == 0) return DRMB200_OK;
    const bool want_elementwise = q0_grad || qd0_grad || q_ref_grad || qd_ref_grad || f_grad || kp_grad || kd_grad;
    if (!want_elementwise && table_grad == nullptr) return DRMB200_OK;
    if (table == nullptr || q0 == nullptr || qd0 == nullptr || q_ref == nullptr || kp == nullptr || kd == nullptr ||
        tau == nullptr || (n_steps > 1 && (q == nullptr || qd == nullptr))) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    if (workspace == nullptr) { set_error("pd rollout backward needs its workspace (drmb200_pd_rollout_backward_workspace_bytes)"); return DRMB200_EINVAL; }

    AdjStepArgs fb = {};
    fb.q_ref = q_ref; fb.qd_ref = qd_ref; fb.f = f; fb.g_tau = g_tau;
    fb.f_grad = f_grad; fb.q_ref_grad = q_ref_grad; fb.qd_ref_grad = qd_ref_grad;
    fb.kp_grad = kp_grad; fb.kd_grad = kd_grad; fb.kp = kp; fb.kd = kd; fb.lim = effort_limit; fb.per_row = gains_per_row;
    return rollout_adjoint(topo, table, q0, qd0, tau, batch, n_steps, dt, flags, q, qd, g_q, g_qd, g_qdd, q0_grad, qd0_grad,
                           nullptr, table_grad, &fb, want_elementwise, workspace, stream);
}

}  // namespace drm
