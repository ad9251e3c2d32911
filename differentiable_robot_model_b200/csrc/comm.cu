// comm.cu -- the one exchange step of the data path, fused with the optimiser: SUM all-reduce of the link-parameter gradient
// over NVLink peer memory + Adam update, in ONE kernel (sm_90a, one process per GPU).
//
// The batch of joint configurations shards across GPUs with no data-path collective (SURVEY.md section 8e); the single
// exception is parameter learning (BASELINE config 5): the gradient of the (fused, flat) link-parameter vector is a batch
// sum, so the shards' gradients must be added before the optimiser step.  The vector is tiny (91 floats for the 21
// inertial tensors of the Kuka), so the step is pure latency: an NCCL all-reduce launch + the optimiser launch are a
// large share of the step at 8 GPUs.  Here every rank
//   1. stores its gradient into a slot of EVERY peer's inbox with plain st.global over NVLink / NVSwitch peer mappings
//      (cudaIpc handles, exchanged once through torch.distributed), __threadfence_system(), then raises a per-source
//      sequence flag in each peer's inbox;
//   2. waits until all `world` flags of its own inbox carry this step's sequence number;
//   3. sums the `world` slots in rank order -- every rank adds the same numbers in the same order, so all ranks hold
//      bit-identical parameters without a broadcast -- and applies Adam (torch.optim.Adam's arithmetic) in place.
// Inbox slots are double-buffered by sequence parity (a rank can run at most one step ahead of a peer: it needs that peer's
// flag of step k+1, which the peer raises only after it has finished reading step k).  The kernel is an ordinary launch
// (no cooperative / cluster launch), so the whole training step, this kernel included, is captured in one CUDA graph.
#include <cstring>
#include "drm_common.cuh"

namespace drm {

constexpr int COMM_MAX_WORLD = 16;

struct CommDev {                       // by-value kernel parameter
    int32_t rank, world, max_floats;
    float* data[COMM_MAX_WORLD];       // data[r]: rank r's inbox, [2 parities][world][max_floats]
    uint32_t* flags[COMM_MAX_WORLD];   // flags[r]: rank r's flags, [world] monotonic sequence numbers (one per source)
    uint32_t* seq;                     // this rank's step counter (device memory; advanced by the kernel -> graph-replayable)
    uint32_t* error;                   // set to 1 if a peer did not show up in time
};

struct Comm {
    CommDev dev;
    void* local = nullptr;             // cudaMalloc'ed block: flags | seq | error | data
    void* peers[COMM_MAX_WORLD] = {};  // opened IPC mappings (null for self)
    int device = 0;
    bool connected = false;
};

constexpr size_t COMM_HEADER_BYTES = 256;          // flags [16] u32 | seq | error, padded

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ float ld_volatile_f32(const float* p) {
    float v;
    asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(256)
allreduce_adam_kernel(const CommDev c, float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ exp_avg,
                      float* __restrict__ exp_avg_sq, int n, float lr, float beta1, float beta2, float eps) {
    const int tid = threadIdx.x;
    const uint32_t seq = *c.seq + 1u;                  // every thread reads it before thread 0 advances it at the end
    const uint32_t par = seq & 1u;
    const int W = c.world;
    if (W > 1) {
        // 1. my gradient -> slot `rank` of every inbox (peer stores over NVLink; my own inbox too)
        for (int i = tid; i < n; i += blockDim.x) {
            const float g = grad[i];
            for (int r = 0; r < W; ++r) c.data[r][((size_t)par * W + c.rank) * c.max_floats + i] = g;
        }
        __threadfence_system();
        __syncthreads();
        if (tid < W) st_release_sys(c.flags[tid] + c.rank, seq);
        // 2. all sources of this step have arrived in my inbox
        if (tid < W) {
            const uint32_t* f = c.flags[c.rank] + tid;
            unsigned spins = 0;
            while ((int32_t)(ld_acquire_sys(f) - seq) < 0) {
                __nanosleep(64);
                if (++spins > (1u << 25)) { *c.error = 1u; break; }        // ~2 s: a peer is missing; do not hang the GPU
            }
        }
        __syncthreads();
    }
    // 3. rank-ordered sum + Adam (torch.optim.Adam: bias-corrected step size, eps added to sqrt(v_hat))
    const float t = (float)seq;
    const float bc1 = 1.f - powf(beta1, t), bc2 = 1.f - powf(beta2, t);
    const float step_size = lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
    const float* inbox = c.data[c.rank] + (size_t)par * W * c.max_floats;
    for (int i = tid; i < n; i += blockDim.x) {
        float g;
        if (W > 1) {
            g = 0.f;
            for (int s = 0; s < W; ++s) g += ld_volatile_f32(inbox + (size_t)s * c.max_floats + i);
        } else {
            g = grad[i];
        }
        const float m = fmaf(beta1, exp_avg[i], (1.f - beta1) * g);
        const float v = fmaf(beta2, exp_avg_sq[i], (1.f - beta2) * g * g);
        exp_avg[i] = m;
        exp_avg_sq[i] = v;
        param[i] -= step_size * (m / (sqrtf(v) * inv_sqrt_bc2 + eps));
    }
    __syncthreads();
    if (tid == 0) *c.seq = seq;
}

#define COMM_CK(call)                                                                         \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            set_error("%s: %s", #call, cudaGetErrorString(e__));                              \
            return DRMB200_ECUDA;                                                             \
        }                                                                                     \
    } while (0)

static size_t comm_bytes(int world, int max_floats) { return COMM_HEADER_BYTES + (size_t)2 * world * max_floats * sizeof(float); }

int comm_create(int32_t rank, int32_t world, int32_t max_floats, Comm** out, void* ipc_handle_out) {
    if (out == nullptr || ipc_handle_out == nullptr) { set_error("null argument"); return DRMB200_EINVAL; }
    if (world < 1 || world > COMM_MAX_WORLD || rank < 0 || rank >= world || max_floats < 1) { set_error("bad rank / world / size (%d, %d, %d)", rank, world, max_floats); return DRMB200_EINVAL; }
    Comm* c = new Comm();
    COMM_CK(cudaGetDevice(&c->device));
    COMM_CK(cudaMalloc(&c->local, comm_bytes(world, max_floats)));
    COMM_CK(cudaMemset(c->local, 0, comm_bytes(world, max_floats)));
    COMM_CK(cudaDeviceSynchronize());
    c->dev.rank = rank; c->dev.world = world; c->dev.max_floats = max_floats;
    char* base = static_cast<char*>(c->local);
    c->dev.flags[rank] = reinterpret_cast<uint32_t*>(base);
    c->dev.seq = reinterpret_cast<uint32_t*>(base + 64);
    c->dev.error = reinterpret_cast<uint32_t*>(base + 128);
    c->dev.data[rank] = reinterpret_cast<float*>(base + COMM_HEADER_BYTES);
    cudaIpcMemHandle_t h;
    memset(&h, 0, sizeof(h));
    if (world > 1) COMM_CK(cudaIpcGetMemHandle(&h, c->local));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(ipc_handle_out, &h, 64);
    c->connected = world == 1;
    *out = c;
    return DRMB200_OK;
}

int comm_connect(Comm* c, const void* all_handles) {
    if (c == nullptr || all_handles == nullptr) { set_error("null argument"); return DRMB200_EINVAL; }
    const char* hs = static_cast<const char*>(all_handles);
    for (int r = 0; r < c->dev.world; ++r) {
        if (r == c->dev.rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, hs + 64 * r, 64);
        void* p = nullptr;
        COMM_CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        c->peers[r] = p;
        c->dev.flags[r] = reinterpret_cast<uint32_t*>(p);
        c->dev.data[r] = reinterpret_cast<float*>(static_cast<char*>(p) + COMM_HEADER_BYTES);
    }
    c->connected = true;
    return DRMB200_OK;
}

int comm_destroy(Comm* c) {
    if (c == nullptr) return DRMB200_OK;
    for (int r = 0; r < COMM_MAX_WORLD; ++r) if (c->peers[r]) cudaIpcCloseMemHandle(c->peers[r]);
    if (c->local) cudaFree(c->local);
    delete c;
    return DRMB200_OK;
}

int comm_error(Comm* c) {
    if (c == nullptr) return 0;
    uint32_t e = 0;
    if (cudaMemcpy(&e, c->dev.error, sizeof(e), cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); return -1; }
    return (int)e;
}

int allreduce_adam(Comm* c, float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int32_t n, float lr,
                   float beta1, float beta2, float eps, cudaStream_t stream) {
    if (c == nullptr || param == nullptr || grad == nullptr || exp_avg == nullptr || exp_avg_sq == nullptr) { set_error("null argument"); return DRMB200_EINVAL; }
    if (!c->connected) { set_error("communicator not connected (drmb200_comm_connect)"); return DRMB200_EINVAL; }
    if (n < 0 || n > c->dev.max_floats) { set_error("n=%d outside [0, %d]", n, c->dev.max_floats); return DRMB200_EINVAL; }
    allreduce_adam_kernel<<<1, 256, 0, stream>>>(c->dev, param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("allreduce_adam launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}

}  // namespace drm

extern "C" {

typedef struct drmb200_comm drmb200_comm_t;

int drmb200_comm_create(int32_t rank, int32_t world, int32_t max_floats, drmb200_comm_t** comm, void* ipc_handle_out) {
    return drm::comm_create(rank, world, max_floats, reinterpret_cast<drm::Comm**>(comm), ipc_handle_out);
}
int drmb200_comm_connect(drmb200_comm_t* comm, const void* all_ipc_handles) {
    return drm::comm_connect(reinterpret_cast<drm::Comm*>(comm), all_ipc_handles);
}
int drmb200_comm_destroy(drmb200_comm_t* comm) { return drm::comm_destroy(reinterpret_cast<drm::Comm*>(comm)); }
int drmb200_comm_error(drmb200_comm_t* comm) { return drm::comm_error(reinterpret_cast<drm::Comm*>(comm)); }
int drmb200_allreduce_adam(drmb200_comm_t* comm, float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int32_t n,
                           float lr, float beta1, float beta2, float eps, void* cuda_stream) {
    return drm::allreduce_adam(reinterpret_cast<drm::Comm*>(comm), param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps,
                               static_cast<cudaStream_t>(cuda_stream));
}

}  // extern "C"
