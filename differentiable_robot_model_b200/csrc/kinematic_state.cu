// kinematic_state.cu -- world pose and body-frame spatial velocity of EVERY link in one launch (sm_90a).
//
// Replaces DifferentiableRobotModel.update_kinematic_state (robot_model.py:140-195) -- the pass that leaves
// `_bodies[i].pose` / `_bodies[i].vel` behind in the reference -- and, with the quaternion output enabled,
// compute_forward_kinematics_all_links (robot_model.py:198-221; there: a depth-first recursion over Python objects
// plus one Python quaternion loop per link).
//
// One thread per configuration walks the whole tree in document order in canonical joint frames; the state of the
// previous link (R~ 9, p 3, w~ 3, v~ 3) stays in registers, branch points spill it to shared-memory slots (the same
// host-computed tree program as RNEA).  Outputs are written un-permuted (natural link frames) in a link-major,
// component-major layout
//     poses [n_links, 12, B]  (rows 0..8 = R row-major, 9..11 = p)
//     quats [n_links,  4, B]  xyzw                vels [n_links, 6, B]  (ang 3, lin 3)
// so that every store of a warp is one contiguous 128-byte line (threads = consecutive configurations): no staging
// needed for the outputs.  q / qd tiles are staged through shared memory like everywhere else.
// Algorithmic bytes per configuration: 4n (+4n) in, n_links * (48 [+16] [+24]) out.
#include "launch.cuh"

namespace drm {

constexpr int KS_TILE = 128;

struct KsArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;       // null: velocities are zero / not requested
    float* __restrict__ poses;          // null to skip
    float* __restrict__ quats;          // null to skip
    float* __restrict__ vels;           // null to skip
    int64_t batch;
    int32_t aligned;
};

struct KsSmem {
    int q, qd, table, slots, total_floats;
    __host__ __device__ KsSmem(int n, int n_links, int n_slots, bool with_vel) {
        int o = 0;
        q = o; o += KS_TILE * n;
        qd = o; o += with_vel ? KS_TILE * n : 0;
        table = o; o += n_links * 12;
        slots = o; o += n_slots * 18 * KS_TILE;
        total_floats = o;
    }
};

// natural vector from a canonical one:  x[idx(c)] = sgn(c) x~[c]
__device__ __forceinline__ V3 unpermute_vec(V3 xt, int code) {
    const int a = code < 0 ? -code : code;
    const float s = code < 0 ? -1.f : 1.f;
    const float c0 = xt.x, c1 = s * xt.y, c2 = s * xt.z;
    if (a == 1) return v3(c2, c0, c1);       // idx = (1,2,0): x[1] = c0, x[2] = c1, x[0] = c2
    if (a == 2) return v3(c1, c2, c0);       // idx = (2,0,1): x[2] = c0, x[0] = c1, x[1] = c2
    return v3(c0, c1, c2);
}

template <bool WITH_VEL>
__global__ void __launch_bounds__(KS_TILE)
kinematic_state_kernel(const __grid_constant__ TreeProgram prog, const KsArgs args) {
    extern __shared__ __align__(128) float smem[];
    const int n = prog.n_dofs, N = prog.n_links;
    const KsSmem L(n, N, prog.n_slots, WITH_VEL);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_tab = smem + L.table;
    float* s_slot = smem + L.slots;
    constexpr int T = KS_TILE;
    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, args.batch - tile_start);
    const bool vec_ok = args.aligned;

    coop_copy(s_q, args.q + tile_start * n, valid * n, vec_ok);
    if (WITH_VEL) coop_copy(s_qd, args.qd + tile_start * n, valid * n, vec_ok);
    for (int i = tid; i < N * 12; i += T) {           // canonical (F~, r~) of every link
        const int l = i / 12, e = i - l * 12;
        const int p = prog.parent[l];
        int src;
        const float sg = canon_map(e, p >= 0 ? (int)prog.axis[p] : 0, prog.axis[l], src);
        s_tab[i] = sg * __ldg(args.table + l * DRMB200_TABLE_STRIDE + src);
    }
    __syncthreads();
    if (tid >= valid) return;

    const int64_t B = args.batch;
    const int64_t b = tile_start + tid;
    const float* qrow = s_q + tid * n;
    const float* qdrow = s_qd + tid * n;

    auto emit = [&](int i, const M3& Rt, V3 p, V3 wt, V3 vt) {
        const int code = prog.axis[i];
        const M3 R = (code != 0) ? unpermute_cols(Rt, code) : Rt;
        if (args.poses != nullptr) {
            float* o = args.poses + ((int64_t)i * 12) * B + b;
            o[0] = R.a00; o[B] = R.a01; o[2 * B] = R.a02; o[3 * B] = R.a10; o[4 * B] = R.a11; o[5 * B] = R.a12;
            o[6 * B] = R.a20; o[7 * B] = R.a21; o[8 * B] = R.a22; o[9 * B] = p.x; o[10 * B] = p.y; o[11 * B] = p.z;
        }
        if (args.quats != nullptr) {
            const float4 qu = quat_xyzw(R);
            float* o = args.quats + ((int64_t)i * 4) * B + b;
            o[0] = qu.x; o[B] = qu.y; o[2 * B] = qu.z; o[3 * B] = qu.w;
        }
        if (WITH_VEL && args.vels != nullptr) {
            const V3 w = unpermute_vec(wt, code), v = unpermute_vec(vt, code);
            float* o = args.vels + ((int64_t)i * 6) * B + b;
            o[0] = w.x; o[B] = w.y; o[2 * B] = w.z; o[3 * B] = v.x; o[4 * B] = v.y; o[5 * B] = v.z;
        }
    };

    const V3 zero = v3(0.f, 0.f, 0.f);
    M3 R = identity3();
    V3 p = zero, w = zero, v = zero;
    emit(0, R, p, w, v);                               // the root: identity pose, zero velocity
    for (int i = 1; i < N; ++i) {
        M3 F; V3 r;
        load_Fr(s_tab + i * 12, F, r);
        const int src = prog.psrc[i];
        M3 Rp; V3 pp, wp, vp;
        if (src == 0) { Rp = R; pp = p; wp = w; vp = v; }
        else if (src < 0) { Rp = identity3(); pp = wp = vp = zero; }
        else {
            const float* sl = s_slot + (src - 1) * 18 * T + tid;
            Rp = ldm(sl, T); pp = ldv(sl + 9 * T, T); wp = ldv(sl + 12 * T, T); vp = ldv(sl + 15 * T, T);
        }
        p = mul_add(Rp, r, pp);
        M3 M = F;
        const int c = prog.dof[i];
        float qd_k = 0.f;
        if (c >= 0) {
            float sn, cs;
            sincos_pi2(qrow[c], sn, cs);
            rotate_z(M, cs, sn);
            if (WITH_VEL) qd_k = qdrow[c];
        }
        R = mul(Rp, M);
        if (WITH_VEL) {
            v = mulT(M, cross_add(wp, r, vp));         // v_i = E (v_p + w_p x r)
            w = mulT(M, wp); w.z += qd_k;              // w_i = E w_p + (0,0,qd)
        }
        emit(i, R, p, w, v);
        const int sv = prog.save[i];
        if (sv >= 0) {
            float* sl = s_slot + sv * 18 * T + tid;
            stm(sl, T, R); stv(sl + 9 * T, T, p); stv(sl + 12 * T, T, w); stv(sl + 15 * T, T, v);
        }
    }
}

int kinematic_state_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                           int64_t batch, float* poses, float* quats, float* vels, cudaStream_t stream) {
    TreeProgram prog;
    int rc = build_tree_program(topo, &prog);
    if (rc != DRMB200_OK) return rc;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || (poses == nullptr && quats == nullptr && vels == nullptr)) return DRMB200_OK;
    if (table == nullptr || q == nullptr) { set_error("table / q is null"); return DRMB200_EINVAL; }
    if (vels != nullptr && qd == nullptr) { set_error("velocities requested without qd"); return DRMB200_EINVAL; }
    const bool with_vel = vels != nullptr;
    KsArgs args;
    args.table = table; args.q = q; args.qd = qd; args.poses = poses; args.quats = quats; args.vels = vels; args.batch = batch;
    args.aligned = aligned16(q, qd);
    const KsSmem L(prog.n_dofs, prog.n_links, prog.n_slots, with_vel);
    const size_t smem_bytes = (size_t)L.total_floats * sizeof(float);
    if (smem_bytes > SMEM_CTA_MAX) { set_error("kinematic state kernel needs %zu B of shared memory (> 227 KB)", smem_bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (batch + KS_TILE - 1) / KS_TILE;
    return with_vel ? launch_kernel<kinematic_state_kernel<true>>(tiles, KS_TILE, smem_bytes, stream, false, "kinematic_state", prog, args)
                    : launch_kernel<kinematic_state_kernel<false>>(tiles, KS_TILE, smem_bytes, stream, false, "kinematic_state", prog, args);
}

}  // namespace drm
