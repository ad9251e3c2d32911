// ik_common.cuh -- what the single-link (inverse_kinematics.cu) and multi-link (inverse_kinematics_multi.cu)
// Levenberg-Marquardt kernels share: the damping bounds, the joint clamp, the signed gather of the walked table rows, the
// target normalisation, the rotation-vector pose error and the host-side argument checks.  With one link and M <= n_u the
// multi-link kernel is bit-identical to the single-link one; sharing these keeps it so.
#pragma once
#include "drm_common.cuh"

namespace drm {

// compiled-in constants (include/drm_b200.h documents them; DESIGN.md §3 records the evidence behind them)
constexpr float IK_LAMBDA_MIN = 1e-5f;
constexpr float IK_LAMBDA_MAX = 1e5f;

__device__ __forceinline__ float clamp_joint(float x, const float* s_lim, int n, int c, bool limits) {
    return limits ? fminf(fmaxf(x, s_lim[c]), s_lim[n + c]) : x;
}

// the canonical rows of the walked links, `count` floats, from the program's signed gather map (bit 15: negate)
__device__ __forceinline__ void stage_walked_rows(float* s_tab, const float* __restrict__ table, const uint16_t* tab_map, int count,
                                                  int T) {
    for (int i = threadIdx.x; i < count; i += T) {
        const uint32_t mp = tab_map[i];
        const float v = __ldg(table + (mp & 0x7fffu));
        s_tab[i] = (mp & 0x8000u) ? -v : v;
    }
}

// a target quaternion in slots tq[0], tq[T], tq[2T], tq[3T], normalised in place
__device__ __forceinline__ void normalize_target_quat(float* tq, int T) {
    const float inv = 1.f / sqrtf(fmaf(tq[0], tq[0], fmaf(tq[T], tq[T], fmaf(tq[2 * T], tq[2 * T], tq[3 * T] * tq[3 * T]))));
    tq[0] *= inv; tq[T] *= inv; tq[2 * T] *= inv; tq[3 * T] *= inv;
}

// Rotation error r = rotvec(quat* (x) conj(quat(R))) of the canonical-frame rotation R of a link with axis code `axis`
// against its normalised target quaternion quat* (xyzw in slots tq[0], tq[T], tq[2T], tq[3T]), the shorter way round.
// Returns |r|^2.
__device__ __forceinline__ float rotvec_error(M3 R, int axis, const float* tq, int T, float& rx, float& ry, float& rz) {
    if (axis != 0) R = unpermute_cols(R, axis);
    const float4 c = quat_xyzw(R);
    const float ax = tq[0], ay = tq[T], az = tq[2 * T], aw = tq[3 * T];
    // q_err = quat* (x) conj(quat(R)), Hamilton product, xyzw
    float w = fmaf(aw, c.w, fmaf(ax, c.x, fmaf(ay, c.y, az * c.z)));
    float x = fmaf(-aw, c.x, fmaf(ax, c.w, fmaf(-ay, c.z, az * c.y)));
    float y = fmaf(-aw, c.y, fmaf(ax, c.z, fmaf(ay, c.w, -az * c.x)));
    float zz = fmaf(-aw, c.z, fmaf(-ax, c.y, fmaf(ay, c.x, az * c.w)));
    if (w < 0.f) { w = -w; x = -x; y = -y; zz = -zz; }
    const float s = sqrtf(fmaf(x, x, fmaf(y, y, zz * zz)));
    const float g = s > 0.f ? 2.f * atan2f(s, w) / s : 0.f;
    rx = g * x; ry = g * y; rz = g * zz;
    return fmaf(rx, rx, fmaf(ry, ry, rz * rz));
}

// the argument checks both entry points make after their program is built: DRMB200_EINVAL with a message, else OK
inline int check_ik_arguments(const float* table, const float* q0, const float* target_pos, const float* lower, const float* upper,
                              int64_t batch, int32_t max_iters, float damping_init, float pos_tol, float rot_tol, const float* q,
                              const float* pos_err, const float* rot_err, const uint8_t* converged, const float* damping_out) {
    if (max_iters < 0) { set_error("max_iters=%d < 0", max_iters); return DRMB200_EINVAL; }
    if (!(pos_tol >= 0.f) || !(rot_tol >= 0.f)) { set_error("tolerances must be >= 0 (pos_tol=%g, rot_tol=%g)", pos_tol, rot_tol); return DRMB200_EINVAL; }
    if ((lower == nullptr) != (upper == nullptr)) { set_error("lower and upper must both be given or both be null"); return DRMB200_EINVAL; }
    if (!(damping_init > 0.f)) { set_error("damping_init=%g must be > 0", damping_init); return DRMB200_EINVAL; }
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch > 0 && (table == nullptr || q0 == nullptr || target_pos == nullptr || q == nullptr || pos_err == nullptr ||
                      rot_err == nullptr || converged == nullptr || damping_out == nullptr)) {
        set_error("null pointer argument");
        return DRMB200_EINVAL;
    }
    return DRMB200_OK;
}

}  // namespace drm
