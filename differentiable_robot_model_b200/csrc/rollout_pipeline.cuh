// rollout_pipeline.cuh -- the per-CTA time loop shared by the one-launch rollout kernels (rollout.cu, contact_rollout.cu):
// state staging, the double-buffered per-step input tiles, the integrate and the per-step stores.  A kernel builds one
// RolloutPipeline<T> at entry and calls its phases from its own step loop:
//
//   pipe.begin(q0, qd0);  <stage the rest>;  __syncthreads();
//   for (t) { in = pipe.fetch(t);  <step body: reads in, writes q̈ and the extra tiles>;  pipe.integrate_and_store(t, ...); }
//   pipe.finish();
//
// The CTA's state (s_q, s_qd: T rows of n) lives in shared memory for all steps.  Each step reads 1 to 3 [T_steps, B, n]
// input streams; the present ones are packed in order in each half of the input double buffer (n_in tiles of T * n).
// Tiles go by TMA bulk copy when every base is 16-byte aligned and the tile is a multiple of 16 bytes, cooperatively else.
//
// Step t, fp32: qd_{t+1} = qd_t + dt * qdd_t;  q_{t+1} = q_t + dt * qd_{t+1}, each "+ dt *" one rounded multiply and one
// rounded add (__fmul_rn / __fadd_rn, never contracted to an FMA), so that a rollout is bit-identical to the stepwise
// torch loop `qd = qd + dt * qdd; q = q + dt * qd` around the single-step kernel.
//
// Ordering (bulk path; two mbarriers, step t waits on mbar[t & 1] at phase parity (t >> 1) & 1):
//   - fetch(t) issues step t + 1's inputs into half (t + 1) & 1.  That half was last read by the step body of step t - 1,
//     which every thread finished, and fenced against the async proxy, before the barrier in step t - 1's store phase.
//   - s_q / s_qd are both the live state and the source of the q / qd stores, so thread 0 waits for the previous step's
//     store READS (bulk_wait_read<0>) right before the integrate, and a barrier follows: the stores drain while the next
//     step body runs.  The extra tiles (q̈, τ) are double-buffered by the caller; the tile of step t is rewritten at step
//     t + 2, after that same wait in step t + 1.
//   - The integrate's and the step body's generic writes reach the bulk stores through fence_proxy_async and a barrier.
// Cooperative path: the next step's reads and writes of s_q / s_qd come after the barrier that ends fetch(t + 1).
#pragma once
#include "drm_common.cuh"

namespace drm {

template <int T>
struct RolloutPipeline {
    uint64_t* mbar;             // two mbarriers in static shared memory
    float* s_q;                 // [T, n] live state
    float* s_qd;
    float* s_in;                // input double buffer: 2 halves of n_in tiles
    const float* in0;           // input streams: in0 always, in1 / in2 when not null
    const float* in1;
    const float* in2;
    int n_in;
    float* q;                   // [T_steps, B, n] state outputs
    float* qd;
    int n, n_steps, tid, valid, tile_floats;
    int64_t tile_off, step;     // step: floats between the [B, n] slices of consecutive steps
    bool vec_ok, bulk;
    uint32_t bytes;
    float dt;

    // in0 is always given; a null in1 / in2 is an absent stream.  aligned: every base 16-byte aligned and
    // batch * n % 4 == 0, so every step's tiles are too.
    __device__ __forceinline__ RolloutPipeline(uint64_t* mbar_, float* s_q_, float* s_qd_, float* s_in_, const float* in0_,
                                               const float* in1_, const float* in2_, float* q_, float* qd_, int n_,
                                               int64_t batch, int n_steps_, float dt_, bool aligned)
        : mbar(mbar_), s_q(s_q_), s_qd(s_qd_), s_in(s_in_), in0(in0_), in1(in1_), in2(in2_),
          n_in(1 + (in1_ != nullptr) + (in2_ != nullptr)), q(q_), qd(qd_), n(n_), n_steps(n_steps_), tid(threadIdx.x),
          dt(dt_) {
        tile_off = (int64_t)blockIdx.x * T * n;
        valid = (int)min((int64_t)T, batch - (int64_t)blockIdx.x * T);
        tile_floats = valid * n;
        step = batch * n;
        vec_ok = aligned;
        bulk = aligned && ((tile_floats & 3) == 0);
        bytes = (uint32_t)tile_floats * 4u;
    }

    __device__ __forceinline__ float* in_buf(int b) const { return s_in + b * n_in * T * n; }

    // thread 0: step t's input tiles into `dst` by TMA, completing on `bar`
    __device__ __forceinline__ void issue(int t, float* dst, uint64_t* bar) const {
        const int64_t off = (int64_t)t * step + tile_off;
        bulk_g2s(dst, in0 + off, bytes, bar);
        if (in1 != nullptr) bulk_g2s(dst + T * n, in1 + off, bytes, bar);
        if (in2 != nullptr) bulk_g2s(dst + (n_in - 1) * T * n, in2 + off, bytes, bar);
    }

    // the (q0, qd0) tile and step 0's inputs in one transaction; the caller stages the rest and ends with a barrier
    __device__ __forceinline__ void begin(const float* q0, const float* qd0) const {
        if (bulk) {
            if (tid == 0) {
                mbar_init(&mbar[0], 1);
                mbar_init(&mbar[1], 1);
                fence_mbar_init();
                mbar_arrive_expect_tx(&mbar[0], (uint32_t)(2 + n_in) * bytes);
                bulk_g2s(s_q, q0 + tile_off, bytes, &mbar[0]);
                bulk_g2s(s_qd, qd0 + tile_off, bytes, &mbar[0]);
                issue(0, s_in, &mbar[0]);
            }
        } else {
            coop_copy(s_q, q0 + tile_off, tile_floats, vec_ok);
            coop_copy(s_qd, qd0 + tile_off, tile_floats, vec_ok);
        }
    }

    // prefetch step t + 1's inputs, wait for step t's; returns step t's input buffer
    __device__ __forceinline__ float* fetch(int t) const {
        const int b = t & 1;
        float* buf = in_buf(b);
        if (bulk) {
            if (tid == 0 && t + 1 < n_steps) {
                mbar_arrive_expect_tx(&mbar[b ^ 1], (uint32_t)n_in * bytes);
                issue(t + 1, in_buf(b ^ 1), &mbar[b ^ 1]);
            }
            mbar_wait(&mbar[b], (uint32_t)(t >> 1) & 1u);
        } else {
            const int64_t off = (int64_t)t * step + tile_off;
            coop_copy(buf, in0 + off, tile_floats, vec_ok);
            if (in1 != nullptr) coop_copy(buf + T * n, in1 + off, tile_floats, vec_ok);
            if (in2 != nullptr) coop_copy(buf + (n_in - 1) * T * n, in2 + off, tile_floats, vec_ok);
            __syncthreads();
        }
        return buf;
    }

    // the integrate with this thread's q̈ row (element k at qdd[k * qdd_stride]), then the stores of step t: q, qd and the
    // extra tiles x0, x1 (to out0 / out1; a null out is not stored)
    __device__ __forceinline__ void integrate_and_store(int t, const float* qdd, int qdd_stride, float* out0, const float* x0,
                                                        float* out1 = nullptr, const float* x1 = nullptr) const {
        if (bulk) {
            if (tid == 0) bulk_wait_read<0>();           // the stores of step t - 1 have read s_q / s_qd and its extra tiles
            __syncthreads();
        }
        if (tid < valid) {
            float* qr = s_q + tid * n;
            float* qdr = s_qd + tid * n;
            for (int k = 0; k < n; ++k) {
                const float v = __fadd_rn(qdr[k], __fmul_rn(dt, qdd[k * qdd_stride]));
                qdr[k] = v;
                qr[k] = __fadd_rn(qr[k], __fmul_rn(dt, v));
            }
        }
        const int64_t off = (int64_t)t * step + tile_off;
        if (bulk) {
            fence_proxy_async();
            __syncthreads();
            if (tid == 0) {
                bulk_s2g(q + off, s_q, bytes);
                bulk_s2g(qd + off, s_qd, bytes);
                if (out0 != nullptr) bulk_s2g(out0 + off, x0, bytes);
                if (out1 != nullptr) bulk_s2g(out1 + off, x1, bytes);
                bulk_commit();
            }
        } else {
            __syncthreads();
            coop_copy(q + off, s_q, tile_floats, vec_ok);
            coop_copy(qd + off, s_qd, tile_floats, vec_ok);
            if (out0 != nullptr) coop_copy(out0 + off, x0, tile_floats, vec_ok);
            if (out1 != nullptr) coop_copy(out1 + off, x1, tile_floats, vec_ok);
        }
    }

    // the last stores have read shared memory before the CTA exits
    __device__ __forceinline__ void finish() const {
        if (bulk && tid == 0) bulk_wait_read<0>();
    }
};

}  // namespace drm
