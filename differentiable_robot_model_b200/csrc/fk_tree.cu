// fk_tree.cu -- FK + geometric Jacobians of SEVERAL end-effector links in ONE walk of the kinematic tree (sm_90a).
//
// The reference computes one end effector per call: compute_endeffector_jacobian (robot_model.py:627-667) runs the whole
// update_kinematic_state pass (robot_model.py:140-195) and then walks ee -> root.  A hand (Allegro: four fingertips off
// one palm, BASELINE config 4) or any multi-limb robot therefore re-walks the shared part of the tree once per fingertip.
// Here the host compiles the UNION of the root -> ee paths into a depth-first "multi program" and the kernel walks it once
// per configuration, emitting (pos, quat, J_lin, J_ang) of every requested link as it passes it:
//
//   * one WARP = one pipeline over tiles of 32 configurations (one configuration per lane, no CTA-wide barrier after the
//     table has been staged); persistent grid, the q tile of the next tile is in flight (TMA bulk load, own mbarrier)
//     while the current one is walked;
//   * the state (R, p) of the previous link stays in registers (f32x2 pair arithmetic as in fk_jacobian.cu), branch
//     points spill it to slot-major shared memory; every movable link parks its joint axis z_i and z_i x p_i in a
//     slot-major scratch indexed by its DEPTH among the movable links of the path (siblings reuse the slots);
//   * at an end effector the Jacobian columns of its path are assembled from the scratch (J_lin = z_i x p_ee - z_i x p_i,
//     robot_model.py:661) into one of TWO output tiles and handed to the TMA unit (1-D bulk stores) while the walk goes
//     on with the next finger into the other tile.  Columns off the path stay zero: the tiles are zeroed once per warp
//     and only the chunks that were written for another end effector are cleared again.
//   * n_dofs % 4 == 0 (Allegro, n = 16): per-lane rows of the natural [32][3][n] tile have a stride of 48 floats, so
//     scalar accesses are 16-way bank conflicts (the reason the CTA-tile kernel needed its 80-register unrolled variant
//     there).  The path columns are therefore assembled FOUR AT A TIME in registers and written as 16-byte chunks
//     (STS.128: 4 wavefronts per quarter-warp instead of 16 per scalar), and q is read as 16-byte chunks too.
//
// Outputs are [n_ee, B, ...] blocks.  Algorithmic HBM bytes per configuration: 4n + n_ee (28 + 24n)  (Allegro, 4 tips:
// 64 + 4 * 412 = 1712 B, SURVEY.md section 8d).
#include <cstring>
#include "drm_common.cuh"

namespace drm {

constexpr int MT_MAX_EE = 8;
constexpr int MT_WARPS_MAX = 4;

struct MultiProgram {
    int32_t n_steps;                       // links walked: union of the root -> ee paths, depth first, root excluded
    int32_t n_dofs;
    int32_t n_ee;
    int32_t n_state_slots;                 // branch points whose (R, p) is spilled
    int32_t n_jslots;                      // max number of movable links on any root -> ee path
    int32_t n_root_ee;                     // requested links that ARE the root (identity pose, zero Jacobian)
    int8_t link[DRMB200_MAX_LINKS];        // table row of step k
    int8_t psrc[DRMB200_MAX_LINKS];        // parent state: -1 root (identity), 0 registers (previous step), 1 + s slot s
    int8_t save[DRMB200_MAX_LINKS];        // -1, or the slot the state after this step is saved to
    int8_t dof[DRMB200_MAX_LINKS];         // q / Jacobian column, -1 for fixed joints
    int8_t jslot[DRMB200_MAX_LINKS];       // joint scratch slot (depth among the movable links of the path), or -1
    int8_t ee[DRMB200_MAX_LINKS];          // -1, or the index (0 .. n_ee) of the end effector emitted after this step
    int8_t axis[DRMB200_MAX_LINKS];        // axis code of the link of step k (un-permutation before the quaternion)
    int8_t root_ee[MT_MAX_EE];
    int8_t cslot[MT_MAX_EE][DRMB200_MAX_LINKS];   // per end effector and Jacobian column: joint scratch slot, or -1 (off the path)
    uint16_t tab_map[DRMB200_MAX_LINKS * 12];     // canonical (F~, r~) entry i of step k = i / 12 (see PathProgram)
};

struct MtArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;          // [B, n]
    float* __restrict__ pos;              // [n_ee, B, 3] or null
    float* __restrict__ quat;             // [n_ee, B, 4] or null
    float* __restrict__ jlin;             // [n_ee, B, 3, n] or null
    float* __restrict__ jang;             // [n_ee, B, 3, n] or null
    int64_t batch;
    int32_t aligned;
    int32_t use_bulk;
    int32_t pdl;                          // programmatic dependent launch: 0 off, 2 wait for the predecessor before the first global write
    int32_t nbuf;                         // output tiles per warp: 2 = the next end effector fills one tile while the TMA unit
                                          // drains the other, 1 = half the shared memory, the warp waits for the drain
};

struct MtWarpLayout {          // per-warp carve-up (floats); every region is a multiple of 32 floats = 128 bytes
    int quat, q, pos, jlin, jang, jscr, state, warp_floats;
    __host__ __device__ MtWarpLayout(int n, int n_jslots, int n_state_slots, bool with_jac, int nbuf) {
        int o = 0;
        quat = o;  o += nbuf * 32 * 4;
        q = o;     o += 2 * 32 * n;
        pos = o;   o += nbuf * 32 * 3;
        jlin = o;  o += with_jac ? nbuf * 32 * 3 * n : 0;
        jang = o;  o += with_jac ? nbuf * 32 * 3 * n : 0;
        jscr = o;  o += with_jac ? n_jslots * 6 * 32 : 0;
        state = o; o += n_state_slots * 12 * 32;
        warp_floats = o;
    }
};
__host__ __device__ __forceinline__ int mt_table_floats(int n_steps) { return (n_steps * 12 + 31) & ~31; }

__device__ __forceinline__ void mt_warp_copy(float* dst, const float* src, int nfloats, bool vec_ok, int lane) {
    if (vec_ok && (nfloats & 3) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = lane; i < (nfloats >> 2); i += 32) d4[i] = s4[i];
    } else {
        for (int i = lane; i < nfloats; i += 32) dst[i] = src[i];
    }
}

template <int NDOF, bool CHUNK, bool WITH_JAC>
__global__ void __launch_bounds__(32 * MT_WARPS_MAX)
fk_tree_kernel(const __grid_constant__ MultiProgram prog, const MtArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar[2 * MT_WARPS_MAX];

    const int n = NDOF > 0 ? NDOF : prog.n_dofs;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int nbuf = args.nbuf;
    const MtWarpLayout L(n, prog.n_jslots, prog.n_state_slots, WITH_JAC, nbuf);
    float* s_tab = smem;
    float* wbase = smem + mt_table_floats(prog.n_steps) + warp * L.warp_floats;
    const int64_t B = args.batch;

    // ---- prologue ------------------------------------------------------------------------------
    if (args.pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");     // see "fk_pdl" (drm_b200.h)
    bool waited = args.pdl != 2;                         // pdl 2: wait for the predecessor grid before the first global write
    if (lane == 0) {
        mbar_init(&mbar[2 * warp], 1);
        mbar_init(&mbar[2 * warp + 1], 1);
        fence_mbar_init();
    }
    if (WITH_JAC) {                                      // both output tiles start as zeros (columns off a path stay zero)
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float4* j4 = reinterpret_cast<float4*>(wbase + L.jlin);          // jlin[nbuf] and jang[nbuf] are adjacent
        for (int i = lane; i < (2 * nbuf * 32 * 3 * n) / 4; i += 32) j4[i] = z4;
    }
    __syncwarp();

    const int64_t n_tiles = (B + 31) >> 5;
    const int64_t tstride = (int64_t)gridDim.x * nwarps;
    int64_t t = (int64_t)blockIdx.x * nwarps + warp;
    const bool bulk_ok = args.use_bulk && args.aligned;
    const bool vec_ok = args.aligned;
    auto tile_valid = [&](int64_t tile) { return (int)min((int64_t)32, B - (tile << 5)); };
    auto issue_q = [&](int64_t tile, int buf) {          // lane 0 only
        const uint32_t bytes = (uint32_t)tile_valid(tile) * n * 4u;
        mbar_arrive_expect_tx(&mbar[2 * warp + buf], bytes);
        bulk_g2s(wbase + L.q + buf * 32 * n, args.q + (tile << 5) * n, bytes, &mbar[2 * warp + buf]);
    };
    if (t < n_tiles && lane == 0 && bulk_ok && (tile_valid(t) & 3) == 0) issue_q(t, 0);

    // canonical (F~, r~) rows of the walked links -> smem (signed gather, map precomputed on the host), once per CTA
    for (int i = threadIdx.x; i < prog.n_steps * 12; i += blockDim.x) {
        const uint32_t mp = prog.tab_map[i];
        const float v = __ldg(args.table + (mp & 0x7fffu));
        s_tab[i] = (mp & 0x8000u) ? -v : v;
    }
    __syncthreads();

    const uint32_t a_tab0 = smem_addr_opaque(s_tab);
    const uint32_t a_jscr = smem_addr_opaque(wbase + L.jscr + lane);
    const uint32_t a_state = smem_addr_opaque(wbase + L.state + lane);
    constexpr uint32_t E = 4u * 32u;                     // byte stride between the elements of a slot-major vector
    unsigned long long dirty[2] = {0ull, 0ull};          // per output tile: chunks / columns that hold non-zeros
    uint32_t emits = 0;                                  // uniform: number of end effectors emitted so far (tile = emits & 1)

    for (int it = 0; t < n_tiles; t += tstride, ++it) {
        const int buf = it & 1;
        const int valid = tile_valid(t);
        const bool bulk = bulk_ok && (valid & 3) == 0;
        const int64_t tn = t + tstride;
        if (tn < n_tiles && lane == 0 && bulk_ok && (tile_valid(tn) & 3) == 0) issue_q(tn, buf ^ 1);
        float* s_q = wbase + L.q + buf * 32 * n;
        if (bulk) {
            while (!mbar_try_wait(&mbar[2 * warp + buf], (uint32_t)(it >> 1) & 1u)) {}
        } else {
            mt_warp_copy(s_q, args.q + (t << 5) * n, valid * n, vec_ok, lane);
            __syncwarp();
        }
        const int64_t row0 = t << 5;
        const uint32_t a_q = smem_addr_opaque(s_q + lane * n);

        M3P Rp = identity3p();
        f32x2 pp = pk2(0.f, 0.f);
        float p2 = 0.f;
        float4 qc = make_float4(0.f, 0.f, 0.f, 0.f);     // CHUNK: the 16-byte chunk of this lane's q row last read
        int qc_idx = -1;

        // ---- emit one end effector: pose + Jacobian columns of its path -> output tile -> TMA -----------------------
        auto emit = [&](int e, int axis_code) {
            const int ob = nbuf == 2 ? (int)(emits & 1) : 0;
            ++emits;
            if (lane == 0) {                             // the stores issued from this tile (two emits / one emit ago) have read it
                if (nbuf == 2) bulk_wait_read<1>(); else bulk_wait_read<0>();
            }
            __syncwarp();
            float* o_pos = wbase + L.pos + ob * 32 * 3;
            float* o_quat = wbase + L.quat + ob * 32 * 4;
            float* o_jl = wbase + L.jlin + ob * 32 * 3 * n;
            float* o_ja = wbase + L.jang + ob * 32 * 3 * n;
            M3 R = unpack3(Rp);
            float px, py;
            upk2(pp, px, py);
            const V3 p = v3(px, py, p2);
            if (args.pos != nullptr) { o_pos[lane * 3 + 0] = p.x; o_pos[lane * 3 + 1] = p.y; o_pos[lane * 3 + 2] = p.z; }
            if (args.quat != nullptr) {
                if (axis_code != 0) R = unpermute_cols(R, axis_code);
                reinterpret_cast<float4*>(o_quat)[lane] = quat_xyzw(R);
            }
            if (WITH_JAC) {
                unsigned long long now = 0ull;
                const uint32_t a_jl = smem_addr_opaque(o_jl + lane * 3 * n), a_ja = smem_addr_opaque(o_ja + lane * 3 * n);
                const uint32_t n4 = 4u * n;
                if (CHUNK) {
                    for (int j = 0; j < (n >> 2); ++j) {
                        const int s0 = prog.cslot[e][4 * j], s1 = prog.cslot[e][4 * j + 1], s2 = prog.cslot[e][4 * j + 2],
                                  s3 = prog.cslot[e][4 * j + 3];
                        const uint32_t o = 16u * j;
                        if (s0 < 0 && s1 < 0 && s2 < 0 && s3 < 0) {                        // chunk off the path
                            if ((dirty[ob] >> j) & 1ull) {
                                const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
                                sts_f32x4(a_jl + o, z4); sts_f32x4(a_jl + o + n4, z4); sts_f32x4(a_jl + o + 2 * n4, z4);
                                sts_f32x4(a_ja + o, z4); sts_f32x4(a_ja + o + n4, z4); sts_f32x4(a_ja + o + 2 * n4, z4);
                            }
                            continue;
                        }
                        now |= 1ull << j;
                        float zx[4], zy[4], zz[4], lx[4], ly[4], lz[4];
                        const int ss[4] = {s0, s1, s2, s3};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            zx[i] = zy[i] = zz[i] = lx[i] = ly[i] = lz[i] = 0.f;
                            if (ss[i] >= 0) {
                                const uint32_t a = a_jscr + (uint32_t)ss[i] * 6u * E;
                                const V3 z = v3(lds_f32(a), lds_f32(a + E), lds_f32(a + 2 * E));
                                const V3 m = v3(lds_f32(a + 3 * E), lds_f32(a + 4 * E), lds_f32(a + 5 * E));
                                const V3 jl = cross_add(z, p, v3(-m.x, -m.y, -m.z));     // z x p_ee - z x p_i
                                zx[i] = z.x; zy[i] = z.y; zz[i] = z.z; lx[i] = jl.x; ly[i] = jl.y; lz[i] = jl.z;
                            }
                        }
                        sts_f32x4(a_jl + o, make_float4(lx[0], lx[1], lx[2], lx[3]));
                        sts_f32x4(a_jl + o + n4, make_float4(ly[0], ly[1], ly[2], ly[3]));
                        sts_f32x4(a_jl + o + 2 * n4, make_float4(lz[0], lz[1], lz[2], lz[3]));
                        sts_f32x4(a_ja + o, make_float4(zx[0], zx[1], zx[2], zx[3]));
                        sts_f32x4(a_ja + o + n4, make_float4(zy[0], zy[1], zy[2], zy[3]));
                        sts_f32x4(a_ja + o + 2 * n4, make_float4(zz[0], zz[1], zz[2], zz[3]));
                    }
                } else {
                    for (int c = 0; c < n; ++c) {
                        const int s = prog.cslot[e][c];
                        const uint32_t o = 4u * c;
                        if (s < 0) {
                            if ((dirty[ob] >> c) & 1ull) {
                                sts_f32(a_jl + o, 0.f); sts_f32(a_jl + o + n4, 0.f); sts_f32(a_jl + o + 2 * n4, 0.f);
                                sts_f32(a_ja + o, 0.f); sts_f32(a_ja + o + n4, 0.f); sts_f32(a_ja + o + 2 * n4, 0.f);
                            }
                            continue;
                        }
                        now |= 1ull << c;
                        const uint32_t a = a_jscr + (uint32_t)s * 6u * E;
                        const V3 z = v3(lds_f32(a), lds_f32(a + E), lds_f32(a + 2 * E));
                        const V3 m = v3(lds_f32(a + 3 * E), lds_f32(a + 4 * E), lds_f32(a + 5 * E));
                        const V3 jl = cross_add(z, p, v3(-m.x, -m.y, -m.z));
                        sts_f32(a_jl + o, jl.x); sts_f32(a_jl + o + n4, jl.y); sts_f32(a_jl + o + 2 * n4, jl.z);
                        sts_f32(a_ja + o, z.x); sts_f32(a_ja + o + n4, z.y); sts_f32(a_ja + o + 2 * n4, z.z);
                    }
                }
                dirty[ob] = now;
            }
            const int64_t r = (int64_t)e * B + row0;
            if (bulk) {
                fence_proxy_async();                     // generic-proxy smem writes -> visible to the async proxy
                __syncwarp();
                if (lane == 0) {
                    if (!waited) asm volatile("griddepcontrol.wait;" ::: "memory");
                    if (args.pos != nullptr) bulk_s2g(args.pos + r * 3, o_pos, (uint32_t)valid * 12u);
                    if (args.quat != nullptr) bulk_s2g(args.quat + r * 4, o_quat, (uint32_t)valid * 16u);
                    if (WITH_JAC) {
                        bulk_s2g(args.jlin + r * 3 * n, o_jl, (uint32_t)valid * 12u * n);
                        bulk_s2g(args.jang + r * 3 * n, o_ja, (uint32_t)valid * 12u * n);
                    }
                    bulk_commit();
                }
            } else {
                __syncwarp();
                if (!waited) asm volatile("griddepcontrol.wait;" ::: "memory");
                if (args.pos != nullptr) mt_warp_copy(args.pos + r * 3, o_pos, valid * 3, vec_ok, lane);
                if (args.quat != nullptr) mt_warp_copy(args.quat + r * 4, o_quat, valid * 4, vec_ok, lane);
                if (WITH_JAC) {
                    mt_warp_copy(args.jlin + r * 3 * n, o_jl, valid * 3 * n, vec_ok, lane);
                    mt_warp_copy(args.jang + r * 3 * n, o_ja, valid * 3 * n, vec_ok, lane);
                }
                __syncwarp();
            }
            waited = true;
        };

        for (int i = 0; i < prog.n_root_ee; ++i) emit(prog.root_ee[i], 0);      // the root itself: identity, zero columns

        // ---- depth-first walk of the union of the root -> ee paths --------------------------------------------------
        uint32_t a_tab = a_tab0;
        for (int k = 0; k < prog.n_steps; ++k, a_tab += 48) {
            M3 F; V3 r;
            load_Fr_s(a_tab, F, r);
            const int src = prog.psrc[k];
            if (src < 0) {
                Rp = identity3p(); pp = pk2(0.f, 0.f); p2 = 0.f;
            } else if (src > 0) {
                const uint32_t a = a_state + (uint32_t)(src - 1) * 12u * E;
                Rp.c0 = pk2(lds_f32(a), lds_f32(a + E)); Rp.c1 = pk2(lds_f32(a + 2 * E), lds_f32(a + 3 * E));
                Rp.c2 = pk2(lds_f32(a + 4 * E), lds_f32(a + 5 * E));
                Rp.a20 = lds_f32(a + 6 * E); Rp.a21 = lds_f32(a + 7 * E); Rp.a22 = lds_f32(a + 8 * E);
                pp = pk2(lds_f32(a + 9 * E), lds_f32(a + 10 * E)); p2 = lds_f32(a + 11 * E);
            }
            mul_add_p(Rp, r, pp, p2);                    // p_i = R_parent r_i + p_parent
            Rp = mul_p(Rp, F);                           // R_parent F~_i
            const int c = prog.dof[k];
            if (c >= 0) {
                float qv;
                if (CHUNK) {
                    if ((c >> 2) != qc_idx) { qc_idx = c >> 2; qc = lds_f32x4(a_q + 16u * qc_idx); }
                    const int w = c & 3;
                    qv = w == 0 ? qc.x : (w == 1 ? qc.y : (w == 2 ? qc.z : qc.w));
                } else {
                    qv = lds_f32(a_q + 4u * c);
                }
                float sn, cs;
                sincos_pi2(qv, sn, cs);
                if (WITH_JAC) {
                    float zx, zy, px, py;
                    upk2(Rp.c2, zx, zy);
                    upk2(pp, px, py);
                    const V3 z = v3(zx, zy, Rp.a22);     // joint axis in the world frame (unchanged by Rz)
                    const V3 m = cross(z, v3(px, py, p2));
                    const uint32_t a = a_jscr + (uint32_t)prog.jslot[k] * 6u * E;
                    sts_f32(a, z.x); sts_f32(a + E, z.y); sts_f32(a + 2 * E, z.z);
                    sts_f32(a + 3 * E, m.x); sts_f32(a + 4 * E, m.y); sts_f32(a + 5 * E, m.z);
                }
                rotate_z_p(Rp, cs, sn);
            }
            const int sv = prog.save[k];
            if (sv >= 0) {
                const uint32_t a = a_state + (uint32_t)sv * 12u * E;
                float lo, hi;
                upk2(Rp.c0, lo, hi); sts_f32(a, lo); sts_f32(a + E, hi);
                upk2(Rp.c1, lo, hi); sts_f32(a + 2 * E, lo); sts_f32(a + 3 * E, hi);
                upk2(Rp.c2, lo, hi); sts_f32(a + 4 * E, lo); sts_f32(a + 5 * E, hi);
                sts_f32(a + 6 * E, Rp.a20); sts_f32(a + 7 * E, Rp.a21); sts_f32(a + 8 * E, Rp.a22);
                upk2(pp, lo, hi); sts_f32(a + 9 * E, lo); sts_f32(a + 10 * E, hi); sts_f32(a + 11 * E, p2);
            }
            const int e = prog.ee[k];
            if (e >= 0) emit(e, prog.axis[k]);
        }
        __syncwarp();                                    // every lane is done with this tile's q buffer
    }
    if (lane == 0) bulk_wait_read<0>();                  // smem must stay intact until the copy engine has read it
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int build_multi_program(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, MultiProgram* prog) {
    if (topo == nullptr || ee_links == nullptr) { set_error("topology / ee_links is null"); return DRMB200_EINVAL; }
    const int N = topo->n_links;
    if (N < 1 || N > DRMB200_MAX_LINKS) { set_error("n_links=%d outside [1, %d]", N, DRMB200_MAX_LINKS); return DRMB200_ELIMIT; }
    if (topo->n_dofs < 0 || topo->n_dofs > N) { set_error("n_dofs=%d inconsistent", topo->n_dofs); return DRMB200_EINVAL; }
    if (n_ee < 1 || n_ee > MT_MAX_EE) { set_error("n_ee=%d outside [1, %d]", n_ee, MT_MAX_EE); return DRMB200_ELIMIT; }
    memset(prog, 0, sizeof(*prog));
    prog->n_dofs = topo->n_dofs;
    prog->n_ee = n_ee;
    int ee_of[DRMB200_MAX_LINKS];
    bool marked[DRMB200_MAX_LINKS];
    for (int i = 0; i < N; ++i) { ee_of[i] = -1; marked[i] = false; }
    for (int i = 1; i < N; ++i) {
        const int p = topo->parent[i], ax = topo->axis[i];
        if (p < 0 || p >= i) { set_error("link %d: parent %d violates topological order", i, p); return DRMB200_EINVAL; }
        if (ax < -3 || ax > 3) { set_error("link %d: bad axis code %d", i, ax); return DRMB200_EINVAL; }
        if (ax != 0 && (topo->dof[i] < 0 || topo->dof[i] >= topo->n_dofs)) { set_error("link %d: bad dof %d", i, (int)topo->dof[i]); return DRMB200_EINVAL; }
    }
    for (int e = 0; e < n_ee; ++e) {
        const int l = ee_links[e];
        if (l < 0 || l >= N) { set_error("ee_links[%d]=%d outside [0, %d)", e, l, N); return DRMB200_EINVAL; }
        if (ee_of[l] >= 0) { set_error("link %d requested twice", l); return DRMB200_EINVAL; }
        ee_of[l] = e;
        memset(prog->cslot[e], 0xff, sizeof(prog->cslot[e]));
        for (int a = l; a > 0; a = topo->parent[a]) marked[a] = true;
        if (l == 0) prog->root_ee[prog->n_root_ee++] = (int8_t)e;
    }
    // depth-first order over the marked sub-tree (children in index order), explicit stack
    int n_children[DRMB200_MAX_LINKS] = {0};
    for (int i = 1; i < N; ++i) if (marked[i]) ++n_children[topo->parent[i]];
    int depth[DRMB200_MAX_LINKS] = {0};           // movable links on the path root -> i, i included
    int step_of[DRMB200_MAX_LINKS];
    int slot_of[DRMB200_MAX_LINKS];
    int remaining[DRMB200_MAX_LINKS];             // children not yet walked (to free state slots)
    bool slot_busy[DRM_MAX_SLOTS] = {false};
    int stack[DRMB200_MAX_LINKS], sp = 0;
    for (int i = N - 1; i >= 1; --i) if (marked[i] && topo->parent[i] == 0) stack[sp++] = i;
    int k = 0, max_depth = 0, n_slots = 0, prev_link = -1;
    while (sp > 0) {
        const int l = stack[--sp];
        const int p = topo->parent[l], ax = topo->axis[l];
        step_of[l] = k;
        prog->link[k] = (int8_t)l;
        prog->axis[k] = (int8_t)ax;
        prog->dof[k] = ax != 0 ? topo->dof[l] : (int8_t)-1;
        depth[l] = depth[p] + (ax != 0 ? 1 : 0);
        prog->jslot[k] = ax != 0 ? (int8_t)(depth[l] - 1) : (int8_t)-1;
        if (depth[l] > max_depth) max_depth = depth[l];
        prog->psrc[k] = (p == 0) ? (int8_t)-1 : (p == prev_link ? (int8_t)0 : (int8_t)(1 + slot_of[p]));
        if (p != 0 && n_children[p] > 1 && --remaining[p] == 0) slot_busy[slot_of[p]] = false;
        prog->save[k] = -1;
        if (n_children[l] > 1) {
            int s = 0;
            while (s < DRM_MAX_SLOTS && slot_busy[s]) ++s;
            if (s == DRM_MAX_SLOTS) { set_error("tree needs more than %d live branch points", DRM_MAX_SLOTS); return DRMB200_ELIMIT; }
            slot_busy[s] = true; slot_of[l] = s; remaining[l] = n_children[l];
            prog->save[k] = (int8_t)s;
            if (s + 1 > n_slots) n_slots = s + 1;
        }
        prog->ee[k] = (int8_t)ee_of[l];
        const int pax = (p == 0) ? 0 : topo->axis[p];
        for (int e = 0; e < 12; ++e) {              // signed gather map of the canonical (F~, r~) row
            int src;
            const float sg = canon_map(e, pax, ax, src);
            prog->tab_map[k * 12 + e] = (uint16_t)((l * DRMB200_TABLE_STRIDE + src) | (sg < 0.f ? 0x8000 : 0));
        }
        for (int c = N - 1; c > l; --c) if (marked[c] && topo->parent[c] == l) stack[sp++] = c;
        prev_link = l;
        ++k;
    }
    prog->n_steps = k;
    prog->n_state_slots = n_slots;
    prog->n_jslots = max_depth;
    for (int e = 0; e < n_ee; ++e)
        for (int a = ee_links[e]; a > 0; a = topo->parent[a])
            if (topo->axis[a] != 0) prog->cslot[e][topo->dof[a]] = (int8_t)(depth[a] - 1);
    return DRMB200_OK;
}

template <int NDOF, bool CHUNK, bool WITH_JAC>
static int launch_fk_tree(const MultiProgram& prog, const MtArgs& args, cudaStream_t stream) {
    const MtWarpLayout L(prog.n_dofs, prog.n_jslots, prog.n_state_slots, WITH_JAC, args.nbuf);
    const size_t warp_bytes = (size_t)L.warp_floats * sizeof(float);
    const size_t tab_bytes = (size_t)mt_table_floats(prog.n_steps) * sizeof(float);
    const size_t cap = 227 * 1024 - 256;
    if (tab_bytes + warp_bytes > cap) { set_error("multi-ee FK needs %zu B of shared memory per warp (> 227 KB)", tab_bytes + warp_bytes); return DRMB200_ELIMIT; }
    const int64_t tiles = (args.batch + 31) >> 5;
    const int sms = device_sm_count();
    // warps per CTA: 2 keeps the CTA small enough that several fit per SM and the tiles of a small batch spread evenly
    int warps = get_option(8);
    if (warps < 1 || warps > MT_WARPS_MAX) warps = 2;
    while (warps > 1 && tab_bytes + warps * warp_bytes > cap) --warps;
    const size_t smem_bytes = tab_bytes + warps * warp_bytes;
    int per_sm = (int)(cap / (smem_bytes + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 16) per_sm = 16;
    const int grid_cap = get_option(9);
    if (grid_cap > 0 && grid_cap < per_sm) per_sm = grid_cap;
    int64_t ctas = (tiles + warps - 1) / warps;
    if (ctas > (int64_t)sms * per_sm) ctas = (int64_t)sms * per_sm;
    auto kern = fk_tree_kernel<NDOF, CHUNK, WITH_JAC>;
    static size_t configured_by_dev[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    size_t& configured = configured_by_dev[dev & 63];
    if (smem_bytes > configured) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%zu B smem): %s", smem_bytes, cudaGetErrorString(e)); return DRMB200_ECUDA; }
        configured = smem_bytes;
    }
    MtArgs largs = args;
    if (args.pdl < 0) {                                   // decide: hazards against the FK launches in flight, residency share
        const uintptr_t Bn = (uintptr_t)args.batch * (uintptr_t)prog.n_ee, n = (uintptr_t)prog.n_dofs;
        const PdlRange outs[4] = {pdl_range(args.pos, Bn * 12), pdl_range(args.quat, Bn * 16), pdl_range(args.jlin, Bn * 12 * n),
                                  pdl_range(args.jang, Bn * 12 * n)};
        const PdlRange ins[2] = {pdl_range(args.q, (uintptr_t)args.batch * 4 * n),
                                 pdl_range(args.table, (uintptr_t)DRMB200_MAX_LINKS * DRMB200_TABLE_STRIDE * 4)};
        const int mode = pdl_decide(stream, ins, 2, outs, (double)ctas * (double)smem_bytes);
        largs.pdl = mode == 2 ? 2 : 0;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)ctas);
    cfg.blockDim = dim3(32u * warps);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = largs.pdl ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, prog, largs);
    if (e != cudaSuccess) { set_error("fk_tree launch: %s", cudaGetErrorString(e)); return DRMB200_ECUDA; }
    count_launch();
    return DRMB200_OK;
}
template <int NDOF, bool CHUNK>
static int launch_fk_tree_j(bool with_jac, const MultiProgram& prog, const MtArgs& args, cudaStream_t stream) {
    return with_jac ? launch_fk_tree<NDOF, CHUNK, true>(prog, args, stream) : launch_fk_tree<NDOF, CHUNK, false>(prog, args, stream);
}

int fk_jacobian_multi_device(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                             const float* q, int64_t batch, float* pos, float* quat, float* jlin, float* jang,
                             cudaStream_t stream) {
    struct Cached { bool valid; int32_t n_ee; int32_t ee[MT_MAX_EE]; drmb200_topology_t topo; MultiProgram prog; };
    static thread_local Cached cache[2] = {};
    static thread_local int cache_next = 0;
    if (topo == nullptr || ee_links == nullptr) { set_error("topology / ee_links is null"); return DRMB200_EINVAL; }
    if (n_ee < 1 || n_ee > MT_MAX_EE) { set_error("n_ee=%d outside [1, %d]", n_ee, MT_MAX_EE); return DRMB200_ELIMIT; }
    const MultiProgram* cached = nullptr;
    for (auto& c : cache)
        if (c.valid && c.n_ee == n_ee && memcmp(c.ee, ee_links, n_ee * sizeof(int32_t)) == 0 && memcmp(&c.topo, topo, sizeof(*topo)) == 0) { cached = &c.prog; break; }
    if (cached == nullptr) {
        Cached& c = cache[cache_next];
        c.valid = false;
        int rc = build_multi_program(topo, n_ee, ee_links, &c.prog);
        if (rc != DRMB200_OK) return rc;
        c.topo = *topo; c.n_ee = n_ee; memcpy(c.ee, ee_links, n_ee * sizeof(int32_t)); c.valid = true;
        cache_next ^= 1;
        cached = &c.prog;
    }
    const MultiProgram& prog = *cached;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if ((jlin == nullptr) != (jang == nullptr)) { set_error("jac_lin and jac_ang must both be given or both be null"); return DRMB200_EINVAL; }
    if (batch == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr) { set_error("table / q is null"); return DRMB200_EINVAL; }
    if (pos == nullptr && quat == nullptr && jlin == nullptr) return DRMB200_OK;
    MtArgs args;
    args.table = table; args.q = q; args.pos = pos; args.quat = quat; args.jlin = jlin; args.jang = jang; args.batch = batch;
    auto al16 = [](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    // every [e] block must start 16-byte aligned too: B * 12 bytes (pos) is a multiple of 16 only when B % 4 == 0
    args.aligned = (al16(q) && al16(pos) && al16(quat) && al16(jlin) && al16(jang) && (n_ee == 1 || (batch & 3) == 0)) ? 1 : 0;
    args.use_bulk = get_option(0) != 0;
    args.nbuf = get_option(10) == 2 ? 2 : 1;
    args.pdl = -1;                                        // decided at launch (pdl_decide)
    const bool with_jac = jlin != nullptr;
    const int n = prog.n_dofs;
    if (n > 64) { set_error("n_dofs=%d > 64", n); return DRMB200_ELIMIT; }
    switch (n) {
        case 16: return launch_fk_tree_j<16, true>(with_jac, prog, args, stream);
        case 12: return launch_fk_tree_j<12, true>(with_jac, prog, args, stream);
        case 7: return launch_fk_tree_j<7, false>(with_jac, prog, args, stream);
        case 9: return launch_fk_tree_j<9, false>(with_jac, prog, args, stream);
        case 23: return launch_fk_tree_j<23, false>(with_jac, prog, args, stream);
        default: return (n % 4 == 0 && n > 0) ? launch_fk_tree_j<0, true>(with_jac, prog, args, stream)
                                              : launch_fk_tree_j<0, false>(with_jac, prog, args, stream);
    }
}

}  // namespace drm
