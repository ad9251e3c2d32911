// launch.cuh -- the host side of a kernel launch, shared by every kernel wrapper: the shared-memory limits and tile rules
// the wrappers size their CTAs by, the per-(kernel, device) function attributes and the launch with its checks.
//
// The wrappers may be called from several host threads at once.  The attribute caches are therefore atomics, one per
// (kernel instantiation, device): the template parameter Kern is the kernel, the device index (& 63) picks the slot.
#pragma once
#include <atomic>
#include <mutex>
#include "drm_common.cuh"

namespace drm {

constexpr size_t SMEM_TWO_CTAS = 113 * 1024;    // a CTA at most this large leaves room for a second one on the SM
constexpr size_t SMEM_CTA_MAX = 227 * 1024;     // the most shared memory one CTA may have

// bytes rounded up to a multiple of 256: the alignment of every slice a wrapper carves out of a caller's workspace
inline int64_t round256(int64_t bytes) { return (bytes + 255) & ~(int64_t)255; }

// every pointer 16-byte aligned (float4 and TMA bulk copies); a null pointer counts as aligned
template <typename... P>
inline bool aligned16(const P*... p) { return (((reinterpret_cast<uintptr_t>(p) & 15u) == 0) && ...); }

// DRMB200_IMPLICIT_DAMPING (include/drm_b200.h) needs DRMB200_DAMPING and a finite step dt > 0; without the flag, OK
inline int check_implicit_damping(uint32_t flags, float dt) {
    if (!(flags & DRMB200_IMPLICIT_DAMPING)) return DRMB200_OK;
    if (!(flags & DRMB200_DAMPING)) { set_error("DRMB200_IMPLICIT_DAMPING needs DRMB200_DAMPING"); return DRMB200_EINVAL; }
    if (!(dt > 0.f && dt <= 3.40282347e38f)) {                  // NaN and inf fail too
        set_error("dt=%g: implicit damping needs a finite step > 0", (double)dt);
        return DRMB200_EINVAL;
    }
    return DRMB200_OK;
}

// DRMB200_IMPLICIT_GAINS (include/drm_b200.h): the PD rollouts only (pd_rollout: whether the caller is one) and a finite
// step dt > 0; without the flag, OK
inline int check_implicit_gains(uint32_t flags, float dt, bool pd_rollout) {
    if (!(flags & DRMB200_IMPLICIT_GAINS)) return DRMB200_OK;
    if (!pd_rollout) { set_error("DRMB200_IMPLICIT_GAINS is for drmb200_pd_rollout(_backward) only"); return DRMB200_EINVAL; }
    if (!(dt > 0.f && dt <= 3.40282347e38f)) {                  // NaN and inf fail too
        set_error("dt=%g: implicit gains need a finite step > 0", (double)dt);
        return DRMB200_EINVAL;
    }
    return DRMB200_OK;
}

// ---------------------------------------------------------------------------------------------
// tile rules: bytes_of(t) is the dynamic shared memory of a CTA of tile t, static_bytes the kernel's static shared memory.
// A rule returns the tile and its dynamic bytes; the caller refuses the choice (ELIMIT) when bytes + static_bytes exceeds
// SMEM_CTA_MAX.
// ---------------------------------------------------------------------------------------------
struct TileChoice { int tile; size_t bytes; };

// 64 while two CTAs still fit an SM (and the caller wants 64), else 32
template <typename F>
inline TileChoice tile_64_or_32(F bytes_of, size_t static_bytes = 0, bool want_64 = true) {
    const int t = want_64 && bytes_of(64) + static_bytes <= SMEM_TWO_CTAS ? 64 : 32;
    return {t, bytes_of(t)};
}

// the largest of 64, 32, ..., 1 with which two CTAs still fit an SM, else 1
template <typename F>
inline TileChoice tile_ladder(F bytes_of, size_t static_bytes) {
    int t = 64;
    while (t > 1 && bytes_of(t) + static_bytes > SMEM_TWO_CTAS) t >>= 1;
    return {t, bytes_of(t)};
}

// the largest of start, start - 1, ..., 1 with which two CTAs still fit an SM, else 1
template <typename F>
inline TileChoice tile_count_down(int start, F bytes_of, size_t static_bytes) {
    int t = start;
    while (t > 1 && bytes_of(t) + static_bytes > SMEM_TWO_CTAS) --t;
    return {t, bytes_of(t)};
}

// ---------------------------------------------------------------------------------------------
// per-(kernel, device) function attributes
// ---------------------------------------------------------------------------------------------
template <auto Kern>
struct KernelAttrs {
    static inline std::atomic<size_t> dynamic_smem[64];     // what cudaFuncAttributeMaxDynamicSharedMemorySize allows
    static inline std::atomic<size_t> static_smem[64];      // sharedSizeBytes + 1; 0: not queried yet
    static inline std::mutex grow;                          // held while dynamic_smem grows
};

inline int device_slot() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev & 63;
}

// static shared memory of Kern (cudaFuncGetAttributes, once per device)
template <auto Kern>
int static_smem_bytes(size_t* bytes) {
    std::atomic<size_t>& slot = KernelAttrs<Kern>::static_smem[device_slot()];
    size_t v = slot.load();
    if (v == 0) {
        cudaFuncAttributes fa;
        const cudaError_t e = cudaFuncGetAttributes(&fa, Kern);
        if (e != cudaSuccess) { set_error("cudaFuncGetAttributes: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
        v = fa.sharedSizeBytes + 1;
        slot.store(v);
    }
    *bytes = v - 1;
    return DRMB200_OK;
}

// Kern's dynamic-shared-memory attribute on the current device, raised to at least `bytes`.  The recorded size is written
// under the lock and only after cudaFuncSetAttribute succeeded, so a thread that finds `bytes` recorded may launch with it.
template <auto Kern>
int ensure_dynamic_smem(size_t bytes) {
    std::atomic<size_t>& allowed = KernelAttrs<Kern>::dynamic_smem[device_slot()];
    if (bytes <= allowed.load()) return DRMB200_OK;
    std::lock_guard<std::mutex> lock(KernelAttrs<Kern>::grow);
    if (bytes <= allowed.load()) return DRMB200_OK;
    const cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%zu B smem): %s", bytes, cudaGetErrorString(e)); return DRMB200_ECUDA; }
    allowed.store(bytes);
    return DRMB200_OK;
}

// ---------------------------------------------------------------------------------------------
// the launch: grid check, shared-memory attribute, <<<>>> (or cudaLaunchKernelEx with programmatic stream serialisation
// when pdl is set), launch error -> DRMB200_ECUDA "<what> launch: ...", launch count
// ---------------------------------------------------------------------------------------------
template <auto Kern, typename... Args>
int launch_kernel(int64_t grid, int block, size_t smem_bytes, cudaStream_t stream, bool pdl, const char* what,
                  const Args&... args) {
    if (grid > 0x7fffffffLL) { set_error("batch too large for one launch"); return DRMB200_EINVAL; }
    const int rc = ensure_dynamic_smem<Kern>(smem_bytes);
    if (rc != DRMB200_OK) return rc;
    cudaError_t e;
    if (pdl) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)grid);
        cfg.blockDim = dim3(block);
        cfg.dynamicSmemBytes = smem_bytes;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        e = cudaLaunchKernelEx(&cfg, Kern, args...);
        if (e == cudaSuccess) e = cudaGetLastError();
    } else {
        Kern<<<(unsigned)grid, block, smem_bytes, stream>>>(args...);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s launch: %s", what, cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}

}  // namespace drm
