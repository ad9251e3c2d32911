// c_api.cu -- extern "C" entry points declared in include/drm_b200.h.
//
// Plain pointers and sizes only; no torch types.  Every function validates its arguments before
// touching the device, never throws and never synchronises (the *_host variant excepted).
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <mutex>
#include <string>
#include "drm_common.cuh"

namespace drm {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};
// Tuning knobs for A/B measurements, overridable with the environment (DRMB200_<NAME IN CAPITALS>) or drmb200_set_option().
struct Option { const char* name; const char* env; int def; };
static const Option g_option_table[] = {
    {"fk_variant", "DRMB200_FK_VARIANT", 1},     // 0: staging: 1 = TMA bulk copies (default), 0 = cooperative float4 copies
    {"fk_tile", "DRMB200_FK_TILE", 0},           // 1: CTA-tile kernel: configurations per CTA, 64 / 128 / 256; 0 = by batch size
    {"fk_unroll", "DRMB200_FK_UNROLL", 2},       // 2: 0 rolled walk, 1 unrolled register-Jacobian kernel (paths <= 8 links),
                                                 //    2 = auto: unrolled only for even n_dofs
    {"fk_packed", "DRMB200_FK_PACKED", 1},       // 3: 1 f32x2 pair arithmetic (default), 0 scalar, 2 two configurations per thread
    {"rnea_packed", "DRMB200_RNEA_PACKED", 1},   // 4: f32x2 pair arithmetic in the RNEA kernel
    {"host_fused", "DRMB200_HOST_FUSED", 1},     // 5: drmb200_fk_jacobian_host on page-locked buffers: 1 = one launch whose TMA
                                                 //    copies cross PCIe themselves (default), 0 = staged H2D -> kernel -> D2H
    {"fk_reserved", "DRMB200_FK_RESERVED", 0},   // 6: unused (was the per-warp pipeline kernel A/B)
    {"fk_pdl", "DRMB200_FK_PDL", 0},             // 7: programmatic dependent launch of the FK kernels: 0 off (default);
                                                 //    2 = a launch may run ahead of the FK launches before it on the stream up
                                                 //    to its first global write (the library falls back to an ordinary launch when
                                                 //    an input overlaps an output of the launches still in flight, see
                                                 //    pdl_mode_for_launch in fk_jacobian.cu); 1 = wait before the first global
                                                 //    read (A/B only: slower than 0)
    {"tree_warps", "DRMB200_TREE_WARPS", 0},     // 8: multi-ee tree kernel: warps per CTA (1..4), 0 = auto
    {"tree_grid_cap", "DRMB200_TREE_GRID_CAP", 0},   // 9: multi-ee tree kernel: resident CTAs per SM, 0 = as many as fit
    {"tree_bufs", "DRMB200_TREE_BUFS", 1},       // 10: multi-ee tree kernel: output tiles per warp (1 or 2)
    {"rnea_fold", "DRMB200_RNEA_FOLD", 1},       // 11: inverse-dynamics kernel: fold fixed links into their movable ancestors (default)
    {"rnea_tile", "DRMB200_RNEA_TILE", 0},       // 12: inverse-dynamics kernel: configurations per CTA, 64 / 128, 0 = by batch size
    {"rnea_bwd_chain", "DRMB200_RNEA_BWD_CHAIN", 1},   // 13: inverse-dynamics adjoint of serial chains: 1 = two-sweep kernel (default), 0 = the general tree kernel
};
constexpr int N_OPTIONS = sizeof(g_option_table) / sizeof(g_option_table[0]);
static std::atomic<int> g_options[N_OPTIONS];
static std::atomic<int> g_options_set[N_OPTIONS];

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int get_option(int which) {
    if (!g_options_set[which].load(std::memory_order_acquire)) {
        const char* e = getenv(g_option_table[which].env);
        g_options[which].store(e ? atoi(e) : g_option_table[which].def, std::memory_order_relaxed);
        g_options_set[which].store(1, std::memory_order_release);
    }
    return g_options[which].load(std::memory_order_relaxed);
}
static int set_option_by_name(const char* name, int value) {
    if (name == nullptr) return DRMB200_EINVAL;
    for (int i = 0; i < N_OPTIONS; ++i)
        if (std::string(name) == g_option_table[i].name) {
            g_options[i].store(value, std::memory_order_relaxed);
            g_options_set[i].store(1, std::memory_order_release);
            return DRMB200_OK;
        }
    return DRMB200_EINVAL;
}

// implemented in the kernel translation units
int fk_jacobian_device(const drmb200_topology_t*, int32_t, const float*, const float*, int64_t, float*, float*,
                       float*, float*, cudaStream_t);
int fk_jacobian_multi_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, int64_t, float*,
                             float*, float*, float*, cudaStream_t);
int fk_jacobian_backward_device(const drmb200_topology_t*, int32_t, const float*, const float*, int64_t,
                                const float*, const float*, const float*, const float*, float*, float*, void*,
                                cudaStream_t);
int inverse_dynamics_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*,
                            int64_t, uint32_t, float*, cudaStream_t);
int dynamic_state_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t, uint32_t,
                         float*, float*, float*, float*, cudaStream_t);
int mass_matrix_prefolded_device(const drmb200_topology_t*, const float*, const float*, int64_t, float*, cudaStream_t);
int forward_dynamics_prefolded_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t,
                                      uint32_t, float*, cudaStream_t);
int64_t folded_table_rows(const drmb200_topology_t*);
int fold_table_device(const drmb200_topology_t*, const float*, float*, cudaStream_t);
int inverse_dynamics_prefolded_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t,
                                      uint32_t, float*, cudaStream_t);
int inverse_dynamics_backward_device(const drmb200_topology_t*, const float*, const float*, const float*,
                                     const float*, int64_t, uint32_t, const float*, float*, float*, float*,
                                     float*, void*, cudaStream_t);
int forward_dynamics_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*,
                            int64_t, uint32_t, float*, cudaStream_t);
int forward_dynamics_backward_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*,
                                     int64_t, uint32_t, const float*, float*, float*, float*, float*, void*, cudaStream_t);
int forward_dynamics_implicit_damping_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*,
                                             int64_t, uint32_t, float, float*, cudaStream_t);
int forward_dynamics_implicit_damping_backward_device(const drmb200_topology_t*, const float*, const float*, const float*,
                                                      const float*, int64_t, uint32_t, float, const float*, float*, float*,
                                                      float*, float*, void*, cudaStream_t);
int forward_dynamics_rollout_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t,
                                    int32_t, float, uint32_t, float*, float*, float*, cudaStream_t);
int64_t forward_dynamics_rollout_backward_workspace_bytes(const drmb200_topology_t*, int64_t);
int forward_dynamics_rollout_backward_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*,
                                             int64_t, int32_t, float, uint32_t, const float*, const float*, const float*,
                                             const float*, const float*, float*, float*, float*, float*, void*, cudaStream_t);
int pd_rollout_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, const float*, const float*,
                      const float*, const float*, int32_t, const float*, int64_t, int32_t, float, uint32_t, float*, float*, float*,
                      float*, cudaStream_t);
int64_t pd_rollout_backward_workspace_bytes(const drmb200_topology_t*, int64_t);
int pd_rollout_backward_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, const float*,
                               const float*, const float*, const float*, int32_t, const float*, int64_t, int32_t, float, uint32_t,
                               const float*, const float*, const float*, const float*, const float*, const float*, const float*,
                               float*, float*, float*, float*, float*, float*, float*, float*, void*, cudaStream_t);
int inverse_dynamics_derivatives_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t,
                                        uint32_t, float*, float*, cudaStream_t, bool);
int forward_dynamics_derivatives_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t,
                                        uint32_t, float*, float*, float*, cudaStream_t, bool);
int inverse_kinematics_device(const drmb200_topology_t*, int32_t, const float*, const float*, const float*, const float*,
                              const float*, const float*, const float*, int64_t, int32_t, float, float, float, float*, float*,
                              float*, uint8_t*, float*, cudaStream_t);
int inverse_kinematics_multi_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, const float*,
                                    const float*, const float*, const float*, const float*, int64_t, int32_t, float, float, float,
                                    float*, float*, float*, uint8_t*, float*, cudaStream_t);
int operational_space_dynamics_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, const float*,
                                      const float*, int64_t, uint32_t, int32_t, float*, float*, float*, float*, cudaStream_t);
int contact_dynamics_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, const float*,
                            const float*, const float*, int64_t, uint32_t, int32_t, float, float*, float*, uint8_t*, cudaStream_t);
int contact_impulse_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, const float*,
                           const float*, int64_t, int32_t, float, float*, float*, uint8_t*, cudaStream_t);
int64_t contact_backward_workspace_bytes(const drmb200_topology_t*, int32_t, const int32_t*, int32_t, int64_t);
int contact_dynamics_backward_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, const float*,
                                     const float*, const float*, const float*, const float*, const uint8_t*, int64_t, uint32_t,
                                     int32_t, float, const float*, const float*, float*, float*, float*, float*, float*, void*,
                                     cudaStream_t);
int contact_impulse_backward_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, const float*,
                                    const float*, const float*, const float*, const uint8_t*, int64_t, int32_t, float,
                                    const float*, const float*, float*, float*, float*, float*, void*, cudaStream_t);
int contact_rollout_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, const float*,
                           const float*, const float*, const float*, int64_t, int32_t, float, uint32_t, int32_t, float, float,
                           float*, float*, float*, float*, float*, uint8_t*, cudaStream_t);
int dynamics_regressor_device(const drmb200_topology_t*, const float*, const float*, const float*, const float*, int64_t, uint32_t,
                              float*, cudaStream_t);
int energy_momentum_device(const drmb200_topology_t*, const float*, const float*, const float*, int64_t, float*, float*, float*,
                           float*, float*, float*, cudaStream_t);
int64_t table_grad_workspace_bytes(const drmb200_topology_t*, int64_t);
int64_t forward_dynamics_backward_workspace_bytes(const drmb200_topology_t*, int64_t);
int mass_matrix_device(const drmb200_topology_t*, const float*, const float*, int64_t, float*, cudaStream_t);
int build_table_device(const float*, int32_t, float*, cudaStream_t);
int kinematic_state_device(const drmb200_topology_t*, const float*, const float*, const float*, int64_t, float*, float*,
                           float*, cudaStream_t);
int build_table_backward_device(const float*, const float*, int32_t, float*, cudaStream_t);
int build_table_fused_device(const float*, const float*, const int32_t*, const int32_t*, const float*, int32_t, float*, float*,
                             cudaStream_t);
int build_table_fused_backward_device(const float*, const float*, const float*, const int32_t*, const int32_t*, const int32_t*,
                                      int32_t, int32_t, float*, float*, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// host-buffer pipeline for FK + Jacobian
// ---------------------------------------------------------------------------------------------
struct HostPipe {
    int device = -1;
    static constexpr int NSTAGE = 3;
    int64_t chunk = 0;          // configurations per stage buffer
    int n_dofs = 0;
    cudaStream_t stream[NSTAGE] = {};
    float* d_q[NSTAGE] = {};
    float* d_pos[NSTAGE] = {};
    float* d_quat[NSTAGE] = {};
    float* d_jl[NSTAGE] = {};
    float* d_ja[NSTAGE] = {};
    void release() {
        for (int s = 0; s < NSTAGE; ++s) {
            if (d_q[s]) cudaFree(d_q[s]);
            if (d_pos[s]) cudaFree(d_pos[s]);
            if (d_quat[s]) cudaFree(d_quat[s]);
            if (d_jl[s]) cudaFree(d_jl[s]);
            if (d_ja[s]) cudaFree(d_ja[s]);
            if (stream[s]) cudaStreamDestroy(stream[s]);
            d_q[s] = d_pos[s] = d_quat[s] = d_jl[s] = d_ja[s] = nullptr;
            stream[s] = nullptr;
        }
        chunk = 0;
    }
};
static HostPipe g_pipe;
static std::mutex g_pipe_mu;

#define CK(call)                                                                              \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            set_error("%s: %s", #call, cudaGetErrorString(e__));                              \
            return DRMB200_ECUDA;                                                             \
        }                                                                                     \
    } while (0)

// device alias of a page-locked host pointer (null stays null); false for pageable memory
static bool pinned_alias(const void* host, const void** dev) {
    *dev = nullptr;
    if (host == nullptr) return true;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, host) != cudaSuccess) { cudaGetLastError(); return false; }
    if (a.type != cudaMemoryTypeHost || a.devicePointer == nullptr) return false;
    *dev = a.devicePointer;
    return true;
}

static int fk_jacobian_host_impl(const drmb200_topology_t* topo, int32_t ee_link, int32_t device,
                                 const float* table, const float* q_host, int64_t batch, float* pos_host,
                                 float* quat_host, float* jl_host, float* ja_host) {
    if (topo == nullptr || q_host == nullptr || table == nullptr) { set_error("null argument"); return DRMB200_EINVAL; }
    if (batch < 0) { set_error("batch < 0"); return DRMB200_EINVAL; }
    if ((jl_host == nullptr) != (ja_host == nullptr)) { set_error("jac_lin/jac_ang must both be given or both null"); return DRMB200_EINVAL; }
    if (batch == 0) return DRMB200_OK;
    const int n = topo->n_dofs;
    std::lock_guard<std::mutex> lock(g_pipe_mu);
    struct DeviceGuard {                  // the caller's current device is restored on every return path
        int prev = -1;
        DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; } }
        ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
    } guard;
    CK(cudaSetDevice(device));
    // Fused path: when every host buffer is page-locked (cudaHostAlloc / cudaHostRegister / torch pin_memory) it has a
    // device alias under unified addressing, and the kernel's own TMA bulk copies read the q tiles from and write the
    // output tiles to HOST memory directly over PCIe -- no staging buffers in HBM, no separate copy operations, the
    // transfer overlaps the arithmetic tile by tile inside ONE launch.  Pageable buffers take the staged pipeline below.
    if (get_option(5) != 0) {
        const void* dq = nullptr; const void* dpos = nullptr; const void* dquat = nullptr; const void* djl = nullptr; const void* dja = nullptr;
        if (pinned_alias(q_host, &dq) && pinned_alias(pos_host, &dpos) && pinned_alias(quat_host, &dquat) &&
            pinned_alias(jl_host, &djl) && pinned_alias(ja_host, &dja)) {
            static cudaStream_t zc_stream[64] = {};
            cudaStream_t& st = zc_stream[device & 63];
            if (st == nullptr) CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
            int rc = fk_jacobian_device(topo, ee_link, table, static_cast<const float*>(dq), batch,
                                        static_cast<float*>(const_cast<void*>(dpos)), static_cast<float*>(const_cast<void*>(dquat)),
                                        static_cast<float*>(const_cast<void*>(djl)), static_cast<float*>(const_cast<void*>(dja)), st);
            if (rc != DRMB200_OK) return rc;
            CK(cudaStreamSynchronize(st));
            return DRMB200_OK;
        }
    }
    // 64 Ki configurations per chunk (14.7 MB per stage for a 7-DoF arm): with 16 Ki chunks a 64 Ki call issues 24
    // async copies / launches and the host cost of each dominates.  Larger batches pipeline H2D / kernel / D2H of
    // successive chunks over the three stage streams.
    const int64_t want_chunk = 65536;
    if (g_pipe.device != device || g_pipe.n_dofs != n || g_pipe.chunk != want_chunk) {
        g_pipe.release();
        g_pipe.device = device;
        g_pipe.n_dofs = n;
        for (int s = 0; s < HostPipe::NSTAGE; ++s) {
            CK(cudaStreamCreateWithFlags(&g_pipe.stream[s], cudaStreamNonBlocking));
            CK(cudaMalloc(&g_pipe.d_q[s], want_chunk * n * sizeof(float)));
            CK(cudaMalloc(&g_pipe.d_pos[s], want_chunk * 3 * sizeof(float)));
            CK(cudaMalloc(&g_pipe.d_quat[s], want_chunk * 4 * sizeof(float)));
            CK(cudaMalloc(&g_pipe.d_jl[s], want_chunk * 3 * n * sizeof(float)));
            CK(cudaMalloc(&g_pipe.d_ja[s], want_chunk * 3 * n * sizeof(float)));
        }
        g_pipe.chunk = want_chunk;
    }
    int64_t done = 0;
    int s = 0;
    while (done < batch) {
        const int64_t b = (batch - done < g_pipe.chunk) ? (batch - done) : g_pipe.chunk;
        cudaStream_t st = g_pipe.stream[s];
        // stream order on `st` guarantees the previous D2H out of this stage's buffers has finished
        CK(cudaMemcpyAsync(g_pipe.d_q[s], q_host + done * n, b * n * sizeof(float), cudaMemcpyHostToDevice, st));
        int rc = fk_jacobian_device(topo, ee_link, table, g_pipe.d_q[s], b, pos_host ? g_pipe.d_pos[s] : nullptr,
                                    quat_host ? g_pipe.d_quat[s] : nullptr, jl_host ? g_pipe.d_jl[s] : nullptr,
                                    ja_host ? g_pipe.d_ja[s] : nullptr, st);
        if (rc != DRMB200_OK) return rc;
        if (pos_host) CK(cudaMemcpyAsync(pos_host + done * 3, g_pipe.d_pos[s], b * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (quat_host) CK(cudaMemcpyAsync(quat_host + done * 4, g_pipe.d_quat[s], b * 4 * sizeof(float), cudaMemcpyDeviceToHost, st));
        if (jl_host) {
            CK(cudaMemcpyAsync(jl_host + done * 3 * n, g_pipe.d_jl[s], b * 3 * n * sizeof(float), cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(ja_host + done * 3 * n, g_pipe.d_ja[s], b * 3 * n * sizeof(float), cudaMemcpyDeviceToHost, st));
        }
        done += b;
        s = (s + 1) % HostPipe::NSTAGE;
    }
    for (int i = 0; i < HostPipe::NSTAGE; ++i) CK(cudaStreamSynchronize(g_pipe.stream[i]));
    return DRMB200_OK;
}

}  // namespace drm

extern "C" {

int drmb200_version(void) { return 100; }   // 0.1.0
const char* drmb200_last_error(void) { return drm::g_err; }
int64_t drmb200_launch_count(void) { return drm::g_launches.load(); }

// not part of the reference-facing surface: A/B switch used by bench.py and the tests
int drmb200_set_option(const char* name, int value) {
    if (drm::set_option_by_name(name, value) == DRMB200_OK) return DRMB200_OK;
    drm::set_error("unknown option");
    return DRMB200_EINVAL;
}
int drmb200_get_option(const char* name, int* value) {
    if (name == nullptr || value == nullptr) { drm::set_error("null argument"); return DRMB200_EINVAL; }
    for (int k = 0; k < drm::N_OPTIONS; ++k)
        if (std::string(name) == drm::g_option_table[k].name) { *value = drm::get_option(k); return DRMB200_OK; }
    drm::set_error("unknown option '%s'", name);
    return DRMB200_EINVAL;
}

int drmb200_fk_jacobian(const drmb200_topology_t* topo, int32_t ee_link, const float* table, const float* q,
                        int64_t batch, float* pos, float* quat, float* jac_lin, float* jac_ang, void* cuda_stream) {
    return drm::fk_jacobian_device(topo, ee_link, table, q, batch, pos, quat, jac_lin, jac_ang,
                                   static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_fk_jacobian_multi(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                              const float* q, int64_t batch, float* pos, float* quat, float* jac_lin, float* jac_ang,
                              void* cuda_stream) {
    return drm::fk_jacobian_multi_device(topo, n_ee, ee_links, table, q, batch, pos, quat, jac_lin, jac_ang,
                                         static_cast<cudaStream_t>(cuda_stream));
}

int64_t drmb200_table_grad_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    return drm::table_grad_workspace_bytes(topo, batch);
}

int drmb200_fk_jacobian_backward(const drmb200_topology_t* topo, int32_t ee_link, const float* table, const float* q,
                                 int64_t batch, const float* g_pos, const float* g_quat, const float* g_jac_lin,
                                 const float* g_jac_ang, float* q_grad, float* table_grad, void* workspace,
                                 void* cuda_stream) {
    return drm::fk_jacobian_backward_device(topo, ee_link, table, q, batch, g_pos, g_quat, g_jac_lin, g_jac_ang,
                                            q_grad, table_grad, workspace, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_inverse_dynamics(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                             const float* qdd, int64_t batch, uint32_t flags, float* tau, void* cuda_stream) {
    return drm::inverse_dynamics_device(topo, table, q, qd, qdd, batch, flags, tau,
                                        static_cast<cudaStream_t>(cuda_stream));
}

int64_t drmb200_folded_table_rows(const drmb200_topology_t* topo) { return drm::folded_table_rows(topo); }

int drmb200_fold_link_table(const drmb200_topology_t* topo, const float* table, float* folded, void* cuda_stream) {
    return drm::fold_table_device(topo, table, folded, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_inverse_dynamics_prefolded(const drmb200_topology_t* topo, const float* folded, const float* q, const float* qd,
                                       const float* qdd, int64_t batch, uint32_t flags, float* tau, void* cuda_stream) {
    return drm::inverse_dynamics_prefolded_device(topo, folded, q, qd, qdd, batch, flags, tau,
                                                  static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_mass_matrix_prefolded(const drmb200_topology_t* topo, const float* folded, const float* q, int64_t batch, float* H,
                                  void* cuda_stream) {
    return drm::mass_matrix_prefolded_device(topo, folded, q, batch, H, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_forward_dynamics_prefolded(const drmb200_topology_t* topo, const float* folded, const float* q, const float* qd,
                                       const float* f, int64_t batch, uint32_t flags, float* qdd, void* cuda_stream) {
    return drm::forward_dynamics_prefolded_device(topo, folded, q, qd, f, batch, flags, qdd,
                                                  static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_dynamic_state(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                          const float* qdd, int64_t batch, uint32_t flags, float* tau, float* vels, float* accs,
                          float* forces, void* cuda_stream) {
    return drm::dynamic_state_device(topo, table, q, qd, qdd, batch, flags, tau, vels, accs, forces,
                                     static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_inverse_dynamics_backward(const drmb200_topology_t* topo, const float* table, const float* q,
                                      const float* qd, const float* qdd, int64_t batch, uint32_t flags,
                                      const float* g_tau, float* q_grad, float* qd_grad, float* qdd_grad,
                                      float* table_grad, void* workspace, void* cuda_stream) {
    return drm::inverse_dynamics_backward_device(topo, table, q, qd, qdd, batch, flags, g_tau, q_grad, qd_grad,
                                                 qdd_grad, table_grad, workspace,
                                                 static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_forward_dynamics(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                             const float* f, int64_t batch, uint32_t flags, float* qdd, void* cuda_stream) {
    return drm::forward_dynamics_device(topo, table, q, qd, f, batch, flags, qdd,
                                        static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_mass_matrix(const drmb200_topology_t* topo, const float* table, const float* q, int64_t batch, float* H,
                        void* cuda_stream) {
    return drm::mass_matrix_device(topo, table, q, batch, H, static_cast<cudaStream_t>(cuda_stream));
}

int64_t drmb200_forward_dynamics_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    return drm::forward_dynamics_backward_workspace_bytes(topo, batch);
}

int drmb200_forward_dynamics_backward(const drmb200_topology_t* topo, const float* table, const float* q,
                                      const float* qd, const float* f, int64_t batch, uint32_t flags,
                                      const float* g_qdd, float* q_grad, float* qd_grad, float* f_grad,
                                      float* table_grad, void* workspace, void* cuda_stream) {
    return drm::forward_dynamics_backward_device(topo, table, q, qd, f, batch, flags, g_qdd, q_grad, qd_grad, f_grad,
                                                 table_grad, workspace, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_forward_dynamics_implicit_damping(const drmb200_topology_t* topo, const float* table, const float* q,
                                              const float* qd, const float* f, int64_t batch, uint32_t flags, float dt,
                                              float* qdd, void* cuda_stream) {
    return drm::forward_dynamics_implicit_damping_device(topo, table, q, qd, f, batch, flags, dt, qdd,
                                                         static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_forward_dynamics_implicit_damping_backward(const drmb200_topology_t* topo, const float* table, const float* q,
                                                       const float* qd, const float* f, int64_t batch, uint32_t flags,
                                                       float dt, const float* g_qdd, float* q_grad, float* qd_grad,
                                                       float* f_grad, float* table_grad, void* workspace, void* cuda_stream) {
    return drm::forward_dynamics_implicit_damping_backward_device(topo, table, q, qd, f, batch, flags, dt, g_qdd, q_grad,
                                                                  qd_grad, f_grad, table_grad, workspace,
                                                                  static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_forward_dynamics_rollout(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                                     const float* f, int64_t batch, int32_t n_steps, float dt, uint32_t flags, float* q,
                                     float* qd, float* qdd, void* cuda_stream) {
    return drm::forward_dynamics_rollout_device(topo, table, q0, qd0, f, batch, n_steps, dt, flags, q, qd, qdd,
                                                static_cast<cudaStream_t>(cuda_stream));
}

int64_t drmb200_forward_dynamics_rollout_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    return drm::forward_dynamics_rollout_backward_workspace_bytes(topo, batch);
}

int drmb200_forward_dynamics_rollout_backward(const drmb200_topology_t* topo, const float* table, const float* q0,
                                              const float* qd0, const float* f, int64_t batch, int32_t n_steps, float dt,
                                              uint32_t flags, const float* q, const float* qd, const float* g_q,
                                              const float* g_qd, const float* g_qdd, float* q0_grad, float* qd0_grad,
                                              float* f_grad, float* table_grad, void* workspace, void* cuda_stream) {
    return drm::forward_dynamics_rollout_backward_device(topo, table, q0, qd0, f, batch, n_steps, dt, flags, q, qd, g_q, g_qd,
                                                         g_qdd, q0_grad, qd0_grad, f_grad, table_grad, workspace,
                                                         static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_pd_rollout(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                       const float* q_ref, const float* qd_ref, const float* f, const float* kp, const float* kd,
                       int32_t gains_per_row, const float* effort_limit, int64_t batch, int32_t n_steps, float dt,
                       uint32_t flags, float* q, float* qd, float* qdd, float* tau, void* cuda_stream) {
    return drm::pd_rollout_device(topo, table, q0, qd0, q_ref, qd_ref, f, kp, kd, gains_per_row, effort_limit, batch, n_steps,
                                  dt, flags, q, qd, qdd, tau, static_cast<cudaStream_t>(cuda_stream));
}

int64_t drmb200_pd_rollout_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch) {
    return drm::pd_rollout_backward_workspace_bytes(topo, batch);
}

int drmb200_pd_rollout_backward(const drmb200_topology_t* topo, const float* table, const float* q0, const float* qd0,
                                const float* q_ref, const float* qd_ref, const float* f, const float* kp, const float* kd,
                                int32_t gains_per_row, const float* effort_limit, int64_t batch, int32_t n_steps, float dt,
                                uint32_t flags, const float* q, const float* qd, const float* tau, const float* g_q,
                                const float* g_qd, const float* g_qdd, const float* g_tau, float* q0_grad, float* qd0_grad,
                                float* q_ref_grad, float* qd_ref_grad, float* f_grad, float* kp_grad, float* kd_grad,
                                float* table_grad, void* workspace, void* cuda_stream) {
    return drm::pd_rollout_backward_device(topo, table, q0, qd0, q_ref, qd_ref, f, kp, kd, gains_per_row, effort_limit, batch,
                                           n_steps, dt, flags, q, qd, tau, g_q, g_qd, g_qdd, g_tau, q0_grad, qd0_grad,
                                           q_ref_grad, qd_ref_grad, f_grad, kp_grad, kd_grad, table_grad, workspace,
                                           static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_inverse_dynamics_derivatives(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                         const float* qdd, int64_t batch, uint32_t flags, float* dtau_dq, float* dtau_dqd,
                                         void* cuda_stream) {
    return drm::inverse_dynamics_derivatives_device(topo, table, q, qd, qdd, batch, flags, dtau_dq, dtau_dqd,
                                                    static_cast<cudaStream_t>(cuda_stream), false);
}

int drmb200_inverse_dynamics_derivatives_prefolded(const drmb200_topology_t* topo, const float* folded, const float* q,
                                                   const float* qd, const float* qdd, int64_t batch, uint32_t flags,
                                                   float* dtau_dq, float* dtau_dqd, void* cuda_stream) {
    return drm::inverse_dynamics_derivatives_device(topo, folded, q, qd, qdd, batch, flags, dtau_dq, dtau_dqd,
                                                    static_cast<cudaStream_t>(cuda_stream), true);
}

int drmb200_forward_dynamics_derivatives(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                         const float* f, int64_t batch, uint32_t flags, float* dqdd_dq, float* dqdd_dqd,
                                         float* dqdd_df, void* cuda_stream) {
    return drm::forward_dynamics_derivatives_device(topo, table, q, qd, f, batch, flags, dqdd_dq, dqdd_dqd, dqdd_df,
                                                    static_cast<cudaStream_t>(cuda_stream), false);
}

int drmb200_forward_dynamics_derivatives_prefolded(const drmb200_topology_t* topo, const float* folded, const float* q,
                                                   const float* qd, const float* f, int64_t batch, uint32_t flags,
                                                   float* dqdd_dq, float* dqdd_dqd, float* dqdd_df, void* cuda_stream) {
    return drm::forward_dynamics_derivatives_device(topo, folded, q, qd, f, batch, flags, dqdd_dq, dqdd_dqd, dqdd_df,
                                                    static_cast<cudaStream_t>(cuda_stream), true);
}

int drmb200_inverse_kinematics(const drmb200_topology_t* topo, int32_t ee_link, const float* table, const float* q0,
                               const float* target_pos, const float* target_quat, const float* lower, const float* upper,
                               const float* damping_in, int64_t batch, int32_t max_iters, float damping_init, float pos_tol,
                               float rot_tol, float* q, float* pos_err, float* rot_err, uint8_t* converged, float* damping_out,
                               void* cuda_stream) {
    return drm::inverse_kinematics_device(topo, ee_link, table, q0, target_pos, target_quat, lower, upper, damping_in, batch,
                                          max_iters, damping_init, pos_tol, rot_tol, q, pos_err, rot_err, converged, damping_out,
                                          static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_inverse_kinematics_multi(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                     const float* q0, const float* target_pos, const float* target_quat, const float* lower,
                                     const float* upper, const float* damping_in, int64_t batch, int32_t max_iters,
                                     float damping_init, float pos_tol, float rot_tol, float* q, float* pos_err, float* rot_err,
                                     uint8_t* converged, float* damping_out, void* cuda_stream) {
    return drm::inverse_kinematics_multi_device(topo, n_ee, ee_links, table, q0, target_pos, target_quat, lower, upper, damping_in,
                                                batch, max_iters, damping_init, pos_tol, rot_tol, q, pos_err, rot_err, converged,
                                                damping_out, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_operational_space_dynamics(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                       const float* q, const float* qd, const float* f, int64_t batch, uint32_t flags,
                                       int32_t position_only, float* inv_inertia, float* acceleration, float* velocity,
                                       float* bias_acceleration, void* cuda_stream) {
    return drm::operational_space_dynamics_device(topo, n_ee, ee_links, table, q, qd, f, batch, flags, position_only, inv_inertia,
                                                  acceleration, velocity, bias_acceleration,
                                                  static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_contact_dynamics(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                             const float* q, const float* qd, const float* f, const float* accel_ref, int64_t batch,
                             uint32_t flags, int32_t position_only, float regularization, float* qdd, float* force,
                             uint8_t* solved, void* cuda_stream) {
    return drm::contact_dynamics_device(topo, n_ee, ee_links, table, q, qd, f, accel_ref, batch, flags, position_only,
                                        regularization, qdd, force, solved, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_contact_impulse(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                            const float* q, const float* qd, const float* velocity_ref, int64_t batch, int32_t position_only,
                            float regularization, float* qd_plus, float* impulse, uint8_t* solved, void* cuda_stream) {
    return drm::contact_impulse_device(topo, n_ee, ee_links, table, q, qd, velocity_ref, batch, position_only, regularization,
                                       qd_plus, impulse, solved, static_cast<cudaStream_t>(cuda_stream));
}

int64_t drmb200_contact_backward_workspace_bytes(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links,
                                                 int32_t position_only, int64_t batch) {
    return drm::contact_backward_workspace_bytes(topo, n_ee, ee_links, position_only, batch);
}

int drmb200_contact_dynamics_backward(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                      const float* q, const float* qd, const float* f, const float* accel_ref, const float* qdd,
                                      const float* force, const uint8_t* solved, int64_t batch, uint32_t flags,
                                      int32_t position_only, float regularization, const float* g_qdd, const float* g_force,
                                      float* q_grad, float* qd_grad, float* f_grad, float* accel_ref_grad, float* table_grad,
                                      void* workspace, void* cuda_stream) {
    return drm::contact_dynamics_backward_device(topo, n_ee, ee_links, table, q, qd, f, accel_ref, qdd, force, solved, batch,
                                                 flags, position_only, regularization, g_qdd, g_force, q_grad, qd_grad, f_grad,
                                                 accel_ref_grad, table_grad, workspace, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_contact_impulse_backward(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                     const float* q, const float* qd, const float* velocity_ref, const float* qd_plus,
                                     const float* impulse, const uint8_t* solved, int64_t batch, int32_t position_only,
                                     float regularization, const float* g_qd_plus, const float* g_impulse, float* q_grad,
                                     float* qd_grad, float* velocity_ref_grad, float* table_grad, void* workspace,
                                     void* cuda_stream) {
    return drm::contact_impulse_backward_device(topo, n_ee, ee_links, table, q, qd, velocity_ref, qd_plus, impulse, solved,
                                                batch, position_only, regularization, g_qd_plus, g_impulse, q_grad, qd_grad,
                                                velocity_ref_grad, table_grad, workspace, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_contact_rollout(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                            const float* q0, const float* qd0, const float* f, const float* target_pos,
                            const float* target_quat, int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                            int32_t position_only, float regularization, float stabilization, float* q, float* qd, float* qdd,
                            float* force, float* accel_ref, uint8_t* solved, void* cuda_stream) {
    return drm::contact_rollout_device(topo, n_ee, ee_links, table, q0, qd0, f, target_pos, target_quat, batch, n_steps, dt,
                                       flags, position_only, regularization, stabilization, q, qd, qdd, force, accel_ref,
                                       solved, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_dynamics_regressor(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                               const float* qdd, int64_t batch, uint32_t flags, float* Y, void* cuda_stream) {
    return drm::dynamics_regressor_device(topo, table, q, qd, qdd, batch, flags, Y, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_energy_momentum(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd, int64_t batch,
                            float* kinetic, float* potential, float* momentum, float* com, float* com_velocity,
                            float* com_jacobian, void* cuda_stream) {
    return drm::energy_momentum_device(topo, table, q, qd, batch, kinetic, potential, momentum, com, com_velocity, com_jacobian,
                                       static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_kinematic_state(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                            int64_t batch, float* poses, float* quats, float* vels, void* cuda_stream) {
    return drm::kinematic_state_device(topo, table, q, qd, batch, poses, quats, vels, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_build_link_table(const float* raw, int32_t n_links, float* table, void* cuda_stream) {
    return drm::build_table_device(raw, n_links, table, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_build_link_table_backward(const float* raw, const float* table_grad, int32_t n_links, float* raw_grad,
                                      void* cuda_stream) {
    return drm::build_table_backward_device(raw, table_grad, n_links, raw_grad, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_build_link_table_fused(const float* const_raw, const float* flat, const int32_t* src, const int32_t* kind,
                                   const float* off, int32_t n_links, float* raw_out, float* table, void* cuda_stream) {
    return drm::build_table_fused_device(const_raw, flat, src, kind, off, n_links, raw_out, table,
                                         static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_build_link_table_fused_backward(const float* raw, const float* table_grad, const float* flat,
                                            const int32_t* first_reader, const int32_t* next_reader, const int32_t* kind,
                                            int32_t n_links, int32_t n_flat, float* raw_grad_scratch, float* flat_grad,
                                            void* cuda_stream) {
    return drm::build_table_fused_backward_device(raw, table_grad, flat, first_reader, next_reader, kind, n_links, n_flat,
                                                  raw_grad_scratch, flat_grad, static_cast<cudaStream_t>(cuda_stream));
}

int drmb200_fk_jacobian_host(const drmb200_topology_t* topo, int32_t ee_link, int32_t device, const float* table,
                             const float* q_host, int64_t batch, float* pos_host, float* quat_host,
                             float* jac_lin_host, float* jac_ang_host) {
    return drm::fk_jacobian_host_impl(topo, ee_link, device, table, q_host, batch, pos_host, quat_host, jac_lin_host,
                                      jac_ang_host);
}

}  // extern "C"
