// backward_common.cuh -- helpers shared by the reverse-mode kernels (backward.cu: FK / Jacobian, backward_rnea.cu: RNEA).
#pragma once
#include "launch.cuh"

namespace drm {

constexpr int BWD_MAX_GRID = 132 * 8;         // upper bound of persistent CTAs (workspace sizing; H100: 132 SMs)
constexpr size_t BWD_SMEM_BUDGET = 200 * 1024;
constexpr float GRAVITY_B = 9.81f;

// ---------------------------------------------------------------------------------------------
// block-level sum of NV per-thread values into the CTA accumulator row `acc_row` (entries map(j))
// ---------------------------------------------------------------------------------------------
// Transposed, two stages, fixed order (deterministic): every thread drops its NV <= 32 values into a padded scratch
// matrix; in each warp lane j adds up value j of the warp's 32 threads (32 independent conflict-free loads, four
// interleaved add chains -- no serial shuffle trees, whose latency these low-occupancy kernels cannot hide); warp 0
// then adds the per-warp partials.  Scratch: block_accumulate_floats(NV, T) floats, laid out [per-warp partials | values];
// the partials sit at a FIXED offset so that calls with different NV sharing one scratch cannot have a late reader of the
// partials overlap an early writer of the next call's values (racecheck-clean, scripts/gpu_sanitize.sh).
__host__ __device__ constexpr int block_accumulate_floats(int nv, int t) { return (t / 32) * 32 + nv * (t + 1); }

template <int NV, int T, typename Map>
__device__ __forceinline__ void block_accumulate(float* scratch, float* acc_row, const float (&vals)[NV], bool active,
                                                 Map map) {
    static_assert(NV <= 32 && T % 32 == 0, "one lane per value");
    constexpr int SCR_LD = T + 1;             // padded leading dimension of the reduction scratch
    constexpr int NW = T / 32;
    float* partial = scratch;                 // [NW][32]
    float* values = scratch + NW * 32;        // [NV][SCR_LD]
    const int tid = threadIdx.x;
#pragma unroll
    for (int j = 0; j < NV; ++j) values[j * SCR_LD + tid] = active ? vals[j] : 0.f;
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    if (lane < NV) {
        const float* row = values + lane * SCR_LD + warp * 32;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int c = 0; c < 32; c += 4) { s0 += row[c]; s1 += row[c + 1]; s2 += row[c + 2]; s3 += row[c + 3]; }
        const float s = (s0 + s1) + (s2 + s3);
        if (NW == 1) acc_row[map(lane)] += s;
        else partial[warp * 32 + lane] = s;
    }
    __syncthreads();
    if (NW > 1 && warp == 0 && lane < NV) {
        float s = partial[lane];
#pragma unroll
        for (int w = 1; w < NW; ++w) s += partial[w * 32 + lane];
        acc_row[map(lane)] += s;
    }
}

__device__ __forceinline__ void tile_load_or_zero(float* dst, const float* src, int nfloats, int total, bool vec_ok) {
    if (src != nullptr) {
        coop_copy(dst, src, nfloats, vec_ok);
    } else {
        for (int i = threadIdx.x; i < total; i += blockDim.x) dst[i] = 0.f;
    }
}

// dL/dR of the xyzw quaternion (branch structure of spatial_vector_algebra.py:116-135), exact derivative
// (the reference's autograd treats the 0.5/sqrt(t) factor as a constant -- SURVEY.md quirk 5).
__device__ __forceinline__ M3 quat_backward(const M3& R, float4 g) {
    M3 b = zero3();
    const float tr = (R.a00 + R.a11) + R.a22;
    const float t4 = tr + 1.0f;
    if (t4 > 1.0f) {
        const float y = 0.5f * rsqrt_nr(t4);
        const float u0 = R.a21 - R.a12, u1 = R.a02 - R.a20, u2 = R.a10 - R.a01;
        const float tb = g.w * y - (y / (2.f * t4)) * (g.x * u0 + g.y * u1 + g.z * u2 + g.w * t4);
        b.a00 = b.a11 = b.a22 = tb;
        b.a21 = g.x * y; b.a12 = -g.x * y; b.a02 = g.y * y; b.a20 = -g.y * y; b.a10 = g.z * y; b.a01 = -g.z * y;
    } else if (R.a22 > fmaxf(R.a00, R.a11)) {
        const float t = R.a22 - (R.a00 + R.a11) + 1.0f;
        const float y = 0.5f * rsqrt_nr(t);
        const float u0 = R.a20 + R.a02, u1 = R.a12 + R.a21, u3 = R.a10 - R.a01;
        const float tb = g.z * y - (y / (2.f * t)) * (g.x * u0 + g.y * u1 + g.z * t + g.w * u3);
        b.a22 = tb; b.a00 = -tb; b.a11 = -tb;
        b.a20 = b.a02 = g.x * y; b.a12 = b.a21 = g.y * y; b.a10 = g.w * y; b.a01 = -g.w * y;
    } else if (R.a11 > R.a00) {
        const float t = R.a11 - (R.a22 + R.a00) + 1.0f;
        const float y = 0.5f * rsqrt_nr(t);
        const float u0 = R.a01 + R.a10, u2 = R.a12 + R.a21, u3 = R.a02 - R.a20;
        const float tb = g.y * y - (y / (2.f * t)) * (g.x * u0 + g.y * t + g.z * u2 + g.w * u3);
        b.a11 = tb; b.a22 = -tb; b.a00 = -tb;
        b.a01 = b.a10 = g.x * y; b.a12 = b.a21 = g.z * y; b.a02 = g.w * y; b.a20 = -g.w * y;
    } else {
        const float t = R.a00 - (R.a11 + R.a22) + 1.0f;
        const float y = 0.5f * rsqrt_nr(t);
        const float u1 = R.a01 + R.a10, u2 = R.a20 + R.a02, u3 = R.a21 - R.a12;
        const float tb = g.x * y - (y / (2.f * t)) * (g.x * t + g.y * u1 + g.z * u2 + g.w * u3);
        b.a00 = tb; b.a11 = -tb; b.a22 = -tb;
        b.a01 = b.a10 = g.y * y; b.a20 = b.a02 = g.z * y; b.a21 = g.w * y; b.a12 = -g.w * y;
    }
    return b;
}


// A persistent kernel: as many CTAs as fit on the device at once (occupancy queried per call, after Kern's
// dynamic-shared-memory attribute has been raised), at most BWD_MAX_GRID and at most one per tile.  *grid_out: the CTA
// count, i.e. the number of partial tables the kernel writes.
template <auto Kern, typename... Args>
static int launch_persistent(int block, size_t smem_bytes, int64_t tiles, cudaStream_t stream, const char* what, int* grid_out,
                             const Args&... args) {
    const int rc = ensure_dynamic_smem<Kern>(smem_bytes);
    if (rc != DRMB200_OK) return rc;
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, Kern, block, smem_bytes);
    if (e != cudaSuccess || per_sm < 1) { set_error("%s: kernel does not fit on an SM (%zu B smem)", what, smem_bytes); return DRMB200_ECUDA; }
    int64_t grid = (int64_t)sms * per_sm;
    if (grid > BWD_MAX_GRID) grid = BWD_MAX_GRID;
    if (grid > tiles) grid = tiles;
    *grid_out = (int)grid;
    return launch_kernel<Kern>(grid, block, smem_bytes, stream, false, what, args...);
}


int64_t table_grad_workspace_bytes(const drmb200_topology_t* topo, int64_t batch);     // backward.cu

// sums the per-CTA partial tables in fixed order and adds them to table_grad (defined in backward.cu)
int launch_reduce(const float* partials, int grid, const drmb200_topology_t* topo, float* table_grad, cudaStream_t stream);

}  // namespace drm
