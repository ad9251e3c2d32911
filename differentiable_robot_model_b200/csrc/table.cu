// table.cu -- link-parameter rows -> link table, forward and analytic backward (sm_90a).
//
// The host gathers, per link, the raw parameters the reference keeps in per-link modules
//   raw[i] = [ rpy(3) | trans(3) | mass | com(3) | inertia_mat(9, at the COM) | damping ]     (20 floats)
// (rigid_body.py:47-49, spatial_vector_algebra.py:312-314) and this pair of tiny kernels turns them into the
// [n_links, 28] table of include/drm_b200.h and back:
//   F  = Rz(yaw) Ry(pitch) Rx(roll)                      rigid_body.py:138-143
//   Io = I_c + m (|c|^2 I - c c^T)   (= I_c + m S(c)S(c)^T), mc = m c    spatial_vector_algebra.py:323-327
// With learnable link parameters the table must be rebuilt -- differentiably -- on every call; done with
// torch ops that is ~60 tiny launches forward and ~100 autograd nodes backward per training step, several times
// the cost of the RNEA forward + backward kernels themselves.  One thread per link; n_links <= 64.
#include "drm_common.cuh"

namespace drm {

constexpr int RAW_STRIDE = 20;

__global__ void build_table_kernel(const float* __restrict__ raw, int n_links, float* __restrict__ table) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_links) return;
    const float* r = raw + i * RAW_STRIDE;
    float* t = table + i * DRMB200_TABLE_STRIDE;
    float sr, cr, sp, cp, sy, cy;
    sincosf(r[0], &sr, &cr);
    sincosf(r[1], &sp, &cp);
    sincosf(r[2], &sy, &cy);
    t[0] = cy * cp; t[1] = cy * sp * sr - sy * cr; t[2] = cy * sp * cr + sy * sr;
    t[3] = sy * cp; t[4] = sy * sp * sr + cy * cr; t[5] = sy * sp * cr - cy * sr;
    t[6] = -sp;     t[7] = cp * sr;                t[8] = cp * cr;
    t[9] = r[3]; t[10] = r[4]; t[11] = r[5];
    const float m = r[6], cx = r[7], cy_ = r[8], cz = r[9];
    const float* I = r + 10;
    t[12] = I[0] + m * (cy_ * cy_ + cz * cz); t[13] = I[1] - m * cx * cy_;            t[14] = I[2] - m * cx * cz;
    t[15] = I[3] - m * cx * cy_;            t[16] = I[4] + m * (cx * cx + cz * cz); t[17] = I[5] - m * cy_ * cz;
    t[18] = I[6] - m * cx * cz;             t[19] = I[7] - m * cy_ * cz;            t[20] = I[8] + m * (cx * cx + cy_ * cy_);
    t[21] = m * cx; t[22] = m * cy_; t[23] = m * cz;
    t[24] = m; t[25] = r[19]; t[26] = 0.f; t[27] = 0.f;
}

__global__ void build_table_backward_kernel(const float* __restrict__ raw, const float* __restrict__ g_table,
                                            int n_links, float* __restrict__ g_raw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_links) return;
    const float* r = raw + i * RAW_STRIDE;
    const float* g = g_table + i * DRMB200_TABLE_STRIDE;
    float* o = g_raw + i * RAW_STRIDE;
    float sr, cr, sp, cp, sy, cy;
    sincosf(r[0], &sr, &cr);
    sincosf(r[1], &sp, &cp);
    sincosf(r[2], &sy, &cy);
    // F and its partial derivatives, element by element (row-major)
    const float F[9] = {cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr,
                        sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr,
                        -sp, cp * sr, cp * cr};
    const float dR[9] = {0.f, cy * sp * cr + sy * sr, -cy * sp * sr + sy * cr,          // d/droll
                         0.f, sy * sp * cr - cy * sr, -sy * sp * sr - cy * cr,
                         0.f, cp * cr, -cp * sr};
    const float dP[9] = {-cy * sp, cy * cp * sr, cy * cp * cr,                          // d/dpitch
                         -sy * sp, sy * cp * sr, sy * cp * cr,
                         -cp, -sp * sr, -sp * cr};
    const float dY[9] = {-F[3], -F[4], -F[5], F[0], F[1], F[2], 0.f, 0.f, 0.f};         // d/dyaw = S(e_z) F
    float gr = 0.f, gp = 0.f, gy = 0.f;
#pragma unroll
    for (int e = 0; e < 9; ++e) { gr = fmaf(g[e], dR[e], gr); gp = fmaf(g[e], dP[e], gp); gy = fmaf(g[e], dY[e], gy); }
    o[0] = gr; o[1] = gp; o[2] = gy;
    o[3] = g[9]; o[4] = g[10]; o[5] = g[11];
    const float m = r[6], cx = r[7], cy_ = r[8], cz = r[9];
    const float* G = g + 12;                  // Io-bar
    const float c2 = cx * cx + cy_ * cy_ + cz * cz;
    const float trG = G[0] + G[4] + G[8];
    // <G, |c|^2 I - c c^T>
    const float cGc = cx * (G[0] * cx + G[1] * cy_ + G[2] * cz) + cy_ * (G[3] * cx + G[4] * cy_ + G[5] * cz) +
                      cz * (G[6] * cx + G[7] * cy_ + G[8] * cz);
    o[6] = g[24] + (g[21] * cx + g[22] * cy_ + g[23] * cz) + (c2 * trG - cGc);
    // d/dc of m <G, |c|^2 I - c c^T> = m (2 tr(G) c - (G + G^T) c)
    const float sx = (G[0] + G[0]) * cx + (G[1] + G[3]) * cy_ + (G[2] + G[6]) * cz;
    const float sy2 = (G[3] + G[1]) * cx + (G[4] + G[4]) * cy_ + (G[5] + G[7]) * cz;
    const float sz = (G[6] + G[2]) * cx + (G[7] + G[5]) * cy_ + (G[8] + G[8]) * cz;
    o[7] = m * (g[21] + 2.f * trG * cx - sx);
    o[8] = m * (g[22] + 2.f * trG * cy_ - sy2);
    o[9] = m * (g[23] + 2.f * trG * cz - sz);
#pragma unroll
    for (int e = 0; e < 9; ++e) o[10 + e] = G[e];
    o[19] = g[25];
}

// ---------------------------------------------------------------------------------------------
// Fused parametrisation: ONE flat parameter vector -> raw rows -> table, and back
// ---------------------------------------------------------------------------------------------
// When link parameters are being learned the reference evaluates one tiny nn.Module per (link, parameter) on every
// call (rigid_body_params.py:14-56; 21 of them in BASELINE config 5), and autograd leaves one AccumulateGrad node per
// module behind.  Here every learnable entry of the raw block is a function of ONE flat device vector:
//   raw[j] = const_raw[j]                              src[j] < 0   (URDF constant)
//          = flat[src[j]]                              kind[j] == 0 (UnconstrainedScalar / UnconstrainedTensor)
//          = flat[src[j]]^2 + off[j]                   kind[j] == 1 (PositiveScalar: l^2 + min_val)
// so the forward is this one kernel (raw rows are kept for the backward) and the backward writes the gradient of the
// flat vector directly -- one optimiser tensor, one fused Adam launch.
__global__ void build_table_fused_kernel(const float* __restrict__ const_raw, const float* __restrict__ flat,
                                         const int32_t* __restrict__ src, const int32_t* __restrict__ kind,
                                         const float* __restrict__ off, int n_links, float* __restrict__ raw_out,
                                         float* __restrict__ table) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_links) return;
    float* r = raw_out + i * RAW_STRIDE;
#pragma unroll 4
    for (int j = 0; j < RAW_STRIDE; ++j) {
        const int k = i * RAW_STRIDE + j;
        const int sidx = src[k];
        float v = const_raw[k];
        if (sidx >= 0) { const float p = flat[sidx]; v = kind[k] == 1 ? fmaf(p, p, off[k]) : p; }
        r[j] = v;
    }
    float* t = table + i * DRMB200_TABLE_STRIDE;
    float sr, cr, sp, cp, sy, cy;
    sincosf(r[0], &sr, &cr);
    sincosf(r[1], &sp, &cp);
    sincosf(r[2], &sy, &cy);
    t[0] = cy * cp; t[1] = cy * sp * sr - sy * cr; t[2] = cy * sp * cr + sy * sr;
    t[3] = sy * cp; t[4] = sy * sp * sr + cy * cr; t[5] = sy * sp * cr - cy * sr;
    t[6] = -sp;     t[7] = cp * sr;                t[8] = cp * cr;
    t[9] = r[3]; t[10] = r[4]; t[11] = r[5];
    const float m = r[6], cx = r[7], cy_ = r[8], cz = r[9];
    const float* I = r + 10;
    t[12] = I[0] + m * (cy_ * cy_ + cz * cz); t[13] = I[1] - m * cx * cy_;            t[14] = I[2] - m * cx * cz;
    t[15] = I[3] - m * cx * cy_;            t[16] = I[4] + m * (cx * cx + cz * cz); t[17] = I[5] - m * cy_ * cz;
    t[18] = I[6] - m * cx * cz;             t[19] = I[7] - m * cy_ * cz;            t[20] = I[8] + m * (cx * cx + cy_ * cy_);
    t[21] = m * cx; t[22] = m * cy_; t[23] = m * cz;
    t[24] = m; t[25] = r[19]; t[26] = 0.f; t[27] = 0.f;
}

// raw_grad (as build_table_backward_kernel) scattered into the gradient of the flat vector; entries of `flat` that feed
// nothing (modules on fixed-joint origins, which the reference freezes) get zero
__global__ void scatter_flat_grad_kernel(const float* __restrict__ g_raw, const float* __restrict__ flat,
                                         const int32_t* __restrict__ src, const int32_t* __restrict__ kind, int n_raw,
                                         int n_flat, float* __restrict__ g_flat) {
    for (int k = threadIdx.x; k < n_flat; k += blockDim.x) g_flat[k] = 0.f;
    __syncthreads();
    for (int k = threadIdx.x; k < n_raw; k += blockDim.x) {
        const int sidx = src[k];
        if (sidx >= 0) g_flat[sidx] = kind[k] == 1 ? 2.f * flat[sidx] * g_raw[k] : g_raw[k];
    }
}

// The link-table build is usually the library's first launch in a process whose CUDA context was created by another runtime
// instance (torch's).  When that first call is a plain <<<>>> launch, this library's (statically linked) runtime probes
// cuKernelGetFunction before it has loaded its module into the context; the probe returns CUDA_ERROR_INVALID_HANDLE
// internally, the runtime then loads the module and the launch succeeds -- harmless, but compute-sanitizer reports the
// internal return code as "1 error" (the r01 memcheck logs; reproduced and bisected with scripts/gpu_sanitize_r02.sh: the
// error appears iff this kernel is the first call and vanishes when an attribute query comes first).  So: query first.
static void warm_runtime_once() {
    static bool done_by_dev[64] = {false};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return; }
    if (done_by_dev[dev & 63]) return;
    cudaFuncAttributes attr;
    if (cudaFuncGetAttributes(&attr, build_table_kernel) != cudaSuccess) cudaGetLastError();
    done_by_dev[dev & 63] = true;
}

int build_table_fused_device(const float* const_raw, const float* flat, const int32_t* src, const int32_t* kind,
                             const float* off, int32_t n_links, float* raw_out, float* table, cudaStream_t stream) {
    if (n_links < 1 || n_links > DRMB200_MAX_LINKS) { set_error("n_links=%d outside [1, %d]", n_links, DRMB200_MAX_LINKS); return DRMB200_ELIMIT; }
    if (const_raw == nullptr || flat == nullptr || src == nullptr || kind == nullptr || off == nullptr || raw_out == nullptr || table == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    warm_runtime_once();
    build_table_fused_kernel<<<1, 64, 0, stream>>>(const_raw, flat, src, kind, off, n_links, raw_out, table);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("build_table_fused launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}

int build_table_fused_backward_device(const float* raw, const float* g_table, const float* flat, const int32_t* src,
                                      const int32_t* kind, int32_t n_links, int32_t n_flat, float* g_raw_scratch,
                                      float* g_flat, cudaStream_t stream) {
    if (n_links < 1 || n_links > DRMB200_MAX_LINKS) { set_error("n_links=%d outside [1, %d]", n_links, DRMB200_MAX_LINKS); return DRMB200_ELIMIT; }
    if (raw == nullptr || g_table == nullptr || flat == nullptr || src == nullptr || kind == nullptr || g_raw_scratch == nullptr || g_flat == nullptr || n_flat < 0) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    build_table_backward_kernel<<<1, 64, 0, stream>>>(raw, g_table, n_links, g_raw_scratch);
    scatter_flat_grad_kernel<<<1, 256, 0, stream>>>(g_raw_scratch, flat, src, kind, n_links * RAW_STRIDE, n_flat, g_flat);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("build_table_fused_backward launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch(2);
    return DRMB200_OK;
}

int build_table_device(const float* raw, int32_t n_links, float* table, cudaStream_t stream) {
    if (n_links < 1 || n_links > DRMB200_MAX_LINKS) { set_error("n_links=%d outside [1, %d]", n_links, DRMB200_MAX_LINKS); return DRMB200_ELIMIT; }
    if (raw == nullptr || table == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    warm_runtime_once();
    build_table_kernel<<<1, 64, 0, stream>>>(raw, n_links, table);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("build_table launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}

int build_table_backward_device(const float* raw, const float* g_table, int32_t n_links, float* g_raw,
                                cudaStream_t stream) {
    if (n_links < 1 || n_links > DRMB200_MAX_LINKS) { set_error("n_links=%d outside [1, %d]", n_links, DRMB200_MAX_LINKS); return DRMB200_ELIMIT; }
    if (raw == nullptr || g_table == nullptr || g_raw == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    build_table_backward_kernel<<<1, 64, 0, stream>>>(raw, g_table, n_links, g_raw);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("build_table_backward launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}

}  // namespace drm
