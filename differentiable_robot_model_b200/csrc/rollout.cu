// rollout.cu -- batched forward-dynamics rollouts (sm_90a): T steps of semi-implicit Euler over the articulated-body
// algorithm in ONE launch, and the reverse-time adjoint of the same rollout.
//
// Step t, fp32, in exactly this order (qdd_t is what drmb200_forward_dynamics returns for (q_t, qd_t, f_t)):
//   qdd_t = FD(q_t, qd_t, f_t);   qd_{t+1} = qd_t + dt * qdd_t;   q_{t+1} = q_t + dt * qd_{t+1}
// each "+ dt *" one rounded multiply and one rounded add (__fmul_rn / __fadd_rn, never contracted to an FMA), so that the
// trajectory is bit-identical to a loop of forward-dynamics launches followed by `qd = qd + dt * qdd; q = q + dt * qd`.
//
// Forward mapping: the articulated-body kernel's (aba.cu) -- one thread per configuration, T per CTA, the same per-thread
// body (aba_body.cuh) -- with a time loop inside.  Once per CTA the table is staged (and folded, "rnea_fold") and the
// (q0, qd0) tile loaded; the state then lives in shared memory for all steps.  Per step the f_t tile arrives by TMA bulk
// copy into a double buffer (f_{t+1} is issued before step t computes; two mbarriers, phase parity t / 2), and the q / qd /
// qdd tiles of step t leave as bulk stores.  s_q / s_qd are both the live state and the store source, so thread 0 waits for
// the previous store's READS only right before the next integrate: the store drains while the next step's passes run.  qdd
// is double-buffered for the same reason.  Tiles whose size or base is not 16-byte aligned take cooperative copies.
//
// Algorithmic HBM bytes per configuration-step: f in 4n, q / qd / qdd out 12n = 16n (112 B at n = 7; 12n without qdd).
//
// Adjoint (drmb200_forward_dynamics_rollout_backward): a host loop t = T-1 ... 0 over the analytic ABA adjoint
// (backward_aba.cu), with running adjoints a_q, a_qd of the state (start at zero):
//   a_q += g_q[t];  a_qd += g_qd[t];  a_qd' = a_qd + dt a_q;  g_qdd_t = dt a_qd' + g_qdd[t]
//   (gq, gqd, gf) = ABA adjoint at (q_t, qd_t, f_t) with g_qdd_t;  f_grad[t] = gf;  a_q += gq;  a_qd = a_qd' + gqd
// and q0_grad = a_q, qd0_grad = a_qd at the end.  One element-wise launch per step fuses the post-update of step t+1 with
// the pre-update of step t; the table gradient of all steps is summed in the adjoint's per-CTA partial tables and reduced
// once, so a backward is 2T + 2 launches.
#include "aba_body.cuh"
#include "launch.cuh"

namespace drm {

int forward_dynamics_backward_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t,
                                     uint32_t, const float*, float*, float*, float*, float*, void*, cudaStream_t, bool, bool);
int64_t forward_dynamics_backward_workspace_bytes(const drmb200_topology_t*, int64_t);

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

template <int T>
__global__ void __launch_bounds__(T)
rollout_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const RolloutArgs args) {
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
            aba_body<T>(prog, s_tab, s_q + tid * n, s_qd + tid * n, s_ft + tid * n, s_qddt + tid * n, s_link + tid, s_slot + tid,
                        args.flags);

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

// ---------------------------------------------------------------------------------------------
// adjoint: the element-wise update between two ABA adjoint launches
// ---------------------------------------------------------------------------------------------
struct AdjStepArgs {
    float* a_q;                 // running adjoints of q_t / qd_t  [B, n]
    float* a_qd;
    float* g_step;              // g_qdd_t handed to the ABA adjoint
    const float* gq;            // ABA adjoint of step t + 1 (post-update; unused when first)
    const float* gqd;
    const float* g_q;           // upstream gradients of step t, NULL = zero
    const float* g_qd;
    const float* g_qdd;
    float* out_q;               // final: q0_grad / qd0_grad (NULL = not wanted)
    float* out_qd;
    int64_t count;
    float dt;
    int32_t first;              // t = T - 1: the running adjoints start at zero
    int32_t final;              // after step 0: post-update only, written to out_q / out_qd
};

__global__ void __launch_bounds__(256) rollout_adjoint_step_kernel(const AdjStepArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.count; i += (int64_t)gridDim.x * blockDim.x) {
        float aq = 0.f, aqd = 0.f;
        if (!a.first) {                                        // post-update of step t + 1
            aq = __fadd_rn(a.a_q[i], a.gq[i]);
            aqd = __fadd_rn(a.a_qd[i], a.gqd[i]);
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
        a.a_q[i] = aq;
        a.a_qd[i] = aqd;
        a.g_step[i] = g;
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
int forward_dynamics_rollout_device(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                                    const float* f, int64_t batch, int32_t n_steps, float dt, uint32_t flags, float* q,
                                    float* qd, float* qdd, cudaStream_t stream) {
    FoldChoice fc;
    const int rc = select_fold(topo, false, &fc);                   // "rnea_fold", as drmb200_forward_dynamics
    if (rc != DRMB200_OK) return rc;
    const TreeProgram& prog = *fc.prog;
    if (batch < 0 || n_steps < 0) { set_error("batch=%lld, n_steps=%d: must be >= 0", (long long)batch, (int)n_steps); return DRMB200_EINVAL; }
    if (batch == 0 || n_steps == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q0 == nullptr || qd0 == nullptr || f == nullptr || q == nullptr || qd == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }

    RolloutArgs args;
    args.table = table; args.q0 = q0; args.qd0 = qd0; args.f = f; args.q = q; args.qd = qd; args.qdd = qdd;
    args.batch = batch; args.n_steps = n_steps; args.dt = dt; args.flags = flags;
    args.aligned = aligned16(q0, qd0, f, q, qd, qdd) && ((batch * prog.n_dofs) & 3) == 0;

    // 64 configurations per CTA when that still gives every SM a CTA and the per-link state leaves room for two CTAs per
    // SM; 32 otherwise -- rollout batches are often below one wave of 64-thread CTAs, and a CTA stays resident for all steps
    const TileChoice c = tile_64_or_32([&](int T) {
        return (size_t)RolloutSmem(T, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float);
    }, 0, (batch + 63) / 64 >= device_sm_count());
    if (c.bytes > SMEM_CTA_MAX) { set_error("model needs %zu B of shared memory per CTA (> 227 KB)", c.bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (batch + c.tile - 1) / c.tile;
    return c.tile == 64 ? launch_kernel<rollout_kernel<64>>(tiles, 64, c.bytes, stream, false, "rollout", prog, fc.fold, args)
                        : launch_kernel<rollout_kernel<32>>(tiles, 32, c.bytes, stream, false, "rollout", prog, fc.fold, args);
}

static int64_t round256(int64_t bytes) { return (bytes + 255) & ~(int64_t)255; }

// [ABA adjoint workspace | a_q | a_qd | g_qdd_t | gq | gqd], each [B, n] fp32
int64_t forward_dynamics_rollout_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    if (topo == nullptr || topo->n_links < 1 || topo->n_links > DRMB200_MAX_LINKS || batch < 0) return 0;
    return round256(forward_dynamics_backward_workspace_bytes(topo, batch)) + 5 * round256(batch * topo->n_dofs * (int64_t)sizeof(float));
}

int forward_dynamics_rollout_backward_device(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                                             const float* f, int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                                             const float* q, const float* qd, const float* g_q, const float* g_qd,
                                             const float* g_qdd, float* q0_grad, float* qd0_grad, float* f_grad,
                                             float* table_grad, void* workspace, cudaStream_t stream) {
    if (topo == nullptr) { set_error("null topology"); return DRMB200_EINVAL; }
    if (batch < 0 || n_steps < 0) { set_error("batch=%lld, n_steps=%d: must be >= 0", (long long)batch, (int)n_steps); return DRMB200_EINVAL; }
    if (batch == 0 || n_steps == 0 || topo->n_dofs == 0) return DRMB200_OK;
    if (q0_grad == nullptr && qd0_grad == nullptr && f_grad == nullptr && table_grad == nullptr) return DRMB200_OK;
    if (table == nullptr || q0 == nullptr || qd0 == nullptr || f == nullptr || (n_steps > 1 && (q == nullptr || qd == nullptr))) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    if (workspace == nullptr) { set_error("rollout backward needs its workspace (drmb200_forward_dynamics_rollout_backward_workspace_bytes)"); return DRMB200_EINVAL; }

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

    int64_t blocks = (count + 255) / 256;
    if (blocks > (int64_t)device_sm_count() * 8) blocks = (int64_t)device_sm_count() * 8;
    auto step_kernel = [&](const AdjStepArgs& a) {
        return launch_kernel<rollout_adjoint_step_kernel>(blocks, 256, 0, stream, false, "rollout adjoint step", a);
    };

    AdjStepArgs a = {};
    a.a_q = a_q; a.a_qd = a_qd; a.g_step = g_step; a.gq = gq; a.gqd = gqd; a.count = count; a.dt = dt;
    for (int t = n_steps - 1; t >= 0; --t) {
        const int64_t off = (int64_t)t * count;
        a.first = (t == n_steps - 1) ? 1 : 0;
        a.final = 0;
        a.g_q = g_q ? g_q + off : nullptr;
        a.g_qd = g_qd ? g_qd + off : nullptr;
        a.g_qdd = g_qdd ? g_qdd + off : nullptr;
        int rc = step_kernel(a);
        if (rc != DRMB200_OK) return rc;
        const float* qt = t == 0 ? q0 : q + off - count;        // step inputs: (q0, qd0), then the forward's outputs
        const float* qdt = t == 0 ? qd0 : qd + off - count;
        rc = forward_dynamics_backward_device(topo, table, qt, qdt, f + off, batch, flags, g_step, gq, gqd,
                                              f_grad ? f_grad + off : nullptr, table_grad, fd_ws, stream,
                                              /*accumulate_partials=*/t != n_steps - 1, /*reduce=*/t == 0);
        if (rc != DRMB200_OK) return rc;
    }
    if (q0_grad == nullptr && qd0_grad == nullptr) return DRMB200_OK;
    a.first = 0;
    a.final = 1;
    a.out_q = q0_grad;
    a.out_qd = qd0_grad;
    return step_kernel(a);
}

}  // namespace drm
