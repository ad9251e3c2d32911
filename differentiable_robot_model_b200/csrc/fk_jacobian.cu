// fk_jacobian.cu -- batched forward kinematics + geometric end-effector Jacobian (sm_90a).
//
// Replaces, in ONE launch, the reference's per-link PyTorch graph for
//   DifferentiableRobotModel.compute_forward_kinematics   (robot_model.py:224-248)
//   DifferentiableRobotModel.compute_endeffector_jacobian (robot_model.py:627-667)
// i.e. update_joint_state (rigid_body.py:130-157), the chain walk of update_kinematic_state
// (robot_model.py:173-193), CoordinateTransform.get_quaternion (spatial_vector_algebra.py:108-136)
// and the ee->root Jacobian walk (robot_model.py:652-665).
//
// Mapping: one thread per joint configuration, TILE configurations per CTA.
//   * The outputs of a link depend only on its ancestors, so the kernel walks just the root->ee
//     chain (the "path program", a by-value kernel parameter living in the constant bank).
//   * Canonical joint frames (drm_common.cuh): the link-table rows are staged into shared memory
//     through a signed permutation so that every movable joint is a +z rotation.  The inner loop
//     has no axis dispatch: R <- (R F~) Rz(q), joint axis z_i = third column, 39 FMA + sincos.
//   * q tile in / (pos, quat, J_lin, J_ang) tiles out are staged through shared memory in the
//     SAME row-major layout as global memory, so each tile moves as one contiguous block with
//     TMA 1-D bulk copies (cp.async.bulk + mbarrier; SASS UBLKCP) issued by one thread.  Ragged
//     tails / unaligned bases fall back to cooperative float4 copies.  n_dofs is a template
//     parameter for the common sizes so every smem access is base + immediate; per-thread rows have
//     odd strides for odd n_dofs (7 -> 7, 21 floats), hence no bank conflicts.
//   * The world rotation R (9) and position p (3) stay in registers along the chain.  Jacobian
//     columns need p_ee, known only at the end of the walk, so during the walk each path joint
//     stores z_i (= its J_ang column, final) and z_i x p_i in the J_lin slot of the smem tile; a
//     short second pass rewrites J_lin = z_i x p_ee - z_i x p_i.
//
// Algorithmic HBM bytes per configuration: 4n (q) + 12 (pos) + 16 (quat) + 24n (J) = 28n + 28
// (224 B for the 7-DoF Kuka iiwa) -- SURVEY.md section 8(d).
#include <cstring>
#include <mutex>
#include "launch.cuh"

namespace drm {

struct FkArgs {
    const float* __restrict__ table;     // [n_links, 28]
    const float* __restrict__ q;         // [B, n]
    float* __restrict__ pos;             // [B, 3] or null
    float* __restrict__ quat;            // [B, 4] or null
    float* __restrict__ jlin;            // [B, 3, n] or null
    float* __restrict__ jang;            // [B, 3, n] or null
    int64_t batch;
    int32_t aligned;                     // all base pointers 16-byte aligned
    int32_t use_bulk;                    // staging variant: 1 TMA bulk copies, 0 cooperative copies
    int32_t pdl;                         // programmatic dependent launch (per-warp kernel): 0 off, 1 wait before the first
                                         // global read, 2 wait before the first global write (caller-asserted independence)
};

// Programmatic dependent launch (PTX griddepcontrol): release the next launch on the stream / wait for the previous grid
__device__ __forceinline__ void grid_dep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// shared-memory carve-up (floats), natural global layout per region
struct FkSmemLayout {
    int q, pos, quat, jlin, jang, table, total_floats;
    __host__ __device__ FkSmemLayout(int tile, int n, int path_len, bool with_jac) {
        int o = 0;
        quat = o; o += tile * 4;               // 16-byte aligned rows first
        q = o;    o += tile * n;
        pos = o;  o += tile * 3;
        jlin = o; o += with_jac ? tile * 3 * n : 0;
        jang = o; o += with_jac ? tile * 3 * n : 0;
        table = o; o += path_len * 12;
        total_floats = o;
    }
};

// One link of the chain walk: p <- R r + p ; R <- R F~ ; for movable joints record the joint axis
// z (third column, unchanged by the z rotation) and m = z x p_i, then R <- R Rz(q).
template <bool FIRST, bool WITH_JAC>
__device__ __forceinline__ void walk_link(const float* row, const float* qrow, int c, M3P& R, f32x2& pp, float& p2,
                                          V3& z, V3& m) {
    M3 F; V3 r;
    load_Fr(row, F, r);
    if (FIRST) {                             // parent is the root: R = I, p = 0
        pp = pk2(r.x, r.y); p2 = r.z;
        R.c0 = pk2(F.a00, F.a10); R.c1 = pk2(F.a01, F.a11); R.c2 = pk2(F.a02, F.a12);
        R.a20 = F.a20; R.a21 = F.a21; R.a22 = F.a22;
    } else {
        mul_add_p(R, r, pp, p2);
        R = mul_p(R, F);
    }
    if (c >= 0) {
        float sn, cs;
        sincos_pi2(qrow[c], sn, cs);
        if (WITH_JAC) {
            float zx, zy, px, py;
            upk2(R.c2, zx, zy);
            upk2(pp, px, py);
            z = v3(zx, zy, R.a22);
            m = cross(z, v3(px, py, p2));
        }
        rotate_z_p(R, cs, sn);
    }
}

// Rolled chain walk on f32x2 pairs: rows 0,1 of R and (p.x, p.y) travel as lane pairs; same operations in the same order
// as the scalar walk.
// Explicit shared-window addresses (see smem_addr_opaque): table cursor a_tab, this thread's q row a_q and J rows a_jl / a_ja
// (n4 = 4 n_dofs bytes).  Each path joint parks z_i (its final J_ang column) and z_i x p_i in the thread's rows of the J tile.
template <bool WITH_JAC>
__device__ __forceinline__ void walk_rolled_packed(const PathProgram& prog, int len, uint32_t a_tab, uint32_t a_q,
                                                   uint32_t a_jl, uint32_t a_ja, uint32_t n4, M3& R, V3& p) {
    M3P Rp = identity3p();
    f32x2 pp = pk2(0.f, 0.f);
    float p2 = 0.f;
    for (int k = 0; k < len; ++k, a_tab += 48) {
        M3 F; V3 r;
        load_Fr_s(a_tab, F, r);
        mul_add_p(Rp, r, pp, p2);
        Rp = mul_p(Rp, F);
        const int c = prog.dof[k];
        if (c >= 0) {
            float sn, cs;
            sincos_pi2(lds_f32(a_q + 4u * c), sn, cs);
            if (WITH_JAC) {
                float zx, zy, px, py;
                upk2(Rp.c2, zx, zy);
                upk2(pp, px, py);
                const V3 z = v3(zx, zy, Rp.a22);
                const V3 m = cross(z, v3(px, py, p2));
                const uint32_t o = 4u * c;
                sts_f32(a_ja + o, z.x); sts_f32(a_ja + o + n4, z.y); sts_f32(a_ja + o + 2 * n4, z.z);
                sts_f32(a_jl + o, m.x); sts_f32(a_jl + o + n4, m.y); sts_f32(a_jl + o + 2 * n4, m.z);
            }
            rotate_z_p(Rp, cs, sn);
        }
    }
    R = unpack3(Rp);
    upk2(pp, p.x, p.y);
    p.z = p2;
}
// Second pass: J_lin[:,c] = z x (p_ee - p_i) = z x p_ee - z x p_i      (robot_model.py:661)
__device__ __forceinline__ void jlin_fixup(const PathProgram& prog, int len, uint32_t a_jl, uint32_t a_ja, uint32_t n4, V3 p) {
    for (int k = 0; k < len; ++k) {
        const int c = prog.dof[k];
        if (c < 0) continue;
        const uint32_t o = 4u * c;
        const V3 z = v3(lds_f32(a_ja + o), lds_f32(a_ja + o + n4), lds_f32(a_ja + o + 2 * n4));
        const V3 m = v3(lds_f32(a_jl + o), lds_f32(a_jl + o + n4), lds_f32(a_jl + o + 2 * n4));
        const V3 j = cross_add(z, p, v3(-m.x, -m.y, -m.z));
        sts_f32(a_jl + o, j.x); sts_f32(a_jl + o + n4, j.y); sts_f32(a_jl + o + 2 * n4, j.z);
    }
}

// Two configurations per thread: rows `a` and `b` of the tile ride in the two lanes of f32x2 pairs, so every arithmetic
// operation of the chain walk (R r~, R F~, the axis cross products, Rz) is issued for both configurations back to back,
// and table loads, loop control and addressing are shared.  Link-table operands are scalar broadcasts.
// sincos and the quaternion (per-lane branches, integer quadrant logic) run per lane.
__device__ __forceinline__ f32x2 neg2(f32x2 x) { return mul2(x, bc2(-1.f)); }

template <bool WITH_JAC>
__device__ __forceinline__ void pair_walk(const PathProgram& prog, const FkArgs& args, int n, int len, int a, int b,
                                          const float* s_q, float* s_pos, float* s_quat, float* s_jlin, float* s_jang,
                                          const float* s_tab) {
    f32x2 R00 = pk2(1.f, 1.f), R01 = pk2(0.f, 0.f), R02 = R01, R10 = R01, R11 = R00, R12 = R01, R20 = R01, R21 = R01, R22 = R00;
    f32x2 px = R01, py = R01, pz = R01;
    const float* qa = s_q + a * n;
    const float* qb = s_q + b * n;
    float* jla = s_jlin + a * 3 * n; float* jlb = s_jlin + b * 3 * n;
    float* jaa = s_jang + a * 3 * n; float* jab = s_jang + b * 3 * n;
    for (int k = 0; k < len; ++k) {
        M3 F; V3 r;
        load_Fr(s_tab + k * 12, F, r);
        // p_i = R_parent r_i + p_parent
        px = fma2(R00, bc2(r.x), fma2(R01, bc2(r.y), fma2(R02, bc2(r.z), px)));
        py = fma2(R10, bc2(r.x), fma2(R11, bc2(r.y), fma2(R12, bc2(r.z), py)));
        pz = fma2(R20, bc2(r.x), fma2(R21, bc2(r.y), fma2(R22, bc2(r.z), pz)));
        // R_parent F~_i  (same association order as mul(M3, M3))
        const f32x2 G00 = fma2(R00, bc2(F.a00), fma2(R01, bc2(F.a10), mul2(R02, bc2(F.a20))));
        const f32x2 G01 = fma2(R00, bc2(F.a01), fma2(R01, bc2(F.a11), mul2(R02, bc2(F.a21))));
        const f32x2 G02 = fma2(R00, bc2(F.a02), fma2(R01, bc2(F.a12), mul2(R02, bc2(F.a22))));
        const f32x2 G10 = fma2(R10, bc2(F.a00), fma2(R11, bc2(F.a10), mul2(R12, bc2(F.a20))));
        const f32x2 G11 = fma2(R10, bc2(F.a01), fma2(R11, bc2(F.a11), mul2(R12, bc2(F.a21))));
        const f32x2 G12 = fma2(R10, bc2(F.a02), fma2(R11, bc2(F.a12), mul2(R12, bc2(F.a22))));
        const f32x2 G20 = fma2(R20, bc2(F.a00), fma2(R21, bc2(F.a10), mul2(R22, bc2(F.a20))));
        const f32x2 G21 = fma2(R20, bc2(F.a01), fma2(R21, bc2(F.a11), mul2(R22, bc2(F.a21))));
        const f32x2 G22 = fma2(R20, bc2(F.a02), fma2(R21, bc2(F.a12), mul2(R22, bc2(F.a22))));
        R00 = G00; R01 = G01; R02 = G02; R10 = G10; R11 = G11; R12 = G12; R20 = G20; R21 = G21; R22 = G22;
        const int c = prog.dof[k];
        if (c >= 0) {
            float sa, ca, sb, cb;
            sincos_pi2(qa[c], sa, ca);
            sincos_pi2(qb[c], sb, cb);
            const f32x2 cs = pk2(ca, cb), sn = pk2(sa, sb), nsn = pk2(-sa, -sb);
            if (WITH_JAC) {
                // z = third column (unchanged by Rz); park z in J_ang (final) and p_i x z = -(z x p_i) in J_lin
                const f32x2 mx = fma2(py, R22, neg2(mul2(pz, R12)));
                const f32x2 my = fma2(pz, R02, neg2(mul2(px, R22)));
                const f32x2 mz = fma2(px, R12, neg2(mul2(py, R02)));
                float lo, hi;
                upk2(R02, lo, hi); jaa[c] = lo; jab[c] = hi;
                upk2(R12, lo, hi); jaa[n + c] = lo; jab[n + c] = hi;
                upk2(R22, lo, hi); jaa[2 * n + c] = lo; jab[2 * n + c] = hi;
                upk2(mx, lo, hi); jla[c] = lo; jlb[c] = hi;
                upk2(my, lo, hi); jla[n + c] = lo; jlb[n + c] = hi;
                upk2(mz, lo, hi); jla[2 * n + c] = lo; jlb[2 * n + c] = hi;
            }
            // R <- R Rz(q): col0' = c col0 + s col1, col1' = -s col0 + c col1
            const f32x2 t0 = fma2(cs, R00, mul2(sn, R01)), t1 = fma2(cs, R10, mul2(sn, R11)), t2 = fma2(cs, R20, mul2(sn, R21));
            R01 = fma2(cs, R01, mul2(nsn, R00)); R11 = fma2(cs, R11, mul2(nsn, R10)); R21 = fma2(cs, R21, mul2(nsn, R20));
            R00 = t0; R10 = t1; R20 = t2;
        }
    }
    if (WITH_JAC) {
        // J_lin[:,c] = z x (p_ee - p_i) = z x p_ee + (p_i x z)      (robot_model.py:661)
        const f32x2 npx = neg2(px), npy = neg2(py), npz = neg2(pz);
        for (int k = 0; k < len; ++k) {
            const int c = prog.dof[k];
            if (c < 0) continue;
            const f32x2 zx = pk2(jaa[c], jab[c]), zy = pk2(jaa[n + c], jab[n + c]), zz = pk2(jaa[2 * n + c], jab[2 * n + c]);
            const f32x2 mx = pk2(jla[c], jlb[c]), my = pk2(jla[n + c], jlb[n + c]), mz = pk2(jla[2 * n + c], jlb[2 * n + c]);
            const f32x2 jx = fma2(zy, pz, fma2(zz, npy, mx));
            const f32x2 jy = fma2(zz, px, fma2(zx, npz, my));
            const f32x2 jz = fma2(zx, py, fma2(zy, npx, mz));
            float lo, hi;
            upk2(jx, lo, hi); jla[c] = lo; jlb[c] = hi;
            upk2(jy, lo, hi); jla[n + c] = lo; jlb[n + c] = hi;
            upk2(jz, lo, hi); jla[2 * n + c] = lo; jlb[2 * n + c] = hi;
        }
    }
    M3 Ra, Rb;
    upk2(R00, Ra.a00, Rb.a00); upk2(R01, Ra.a01, Rb.a01); upk2(R02, Ra.a02, Rb.a02);
    upk2(R10, Ra.a10, Rb.a10); upk2(R11, Ra.a11, Rb.a11); upk2(R12, Ra.a12, Rb.a12);
    upk2(R20, Ra.a20, Rb.a20); upk2(R21, Ra.a21, Rb.a21); upk2(R22, Ra.a22, Rb.a22);
    if (args.pos != nullptr) {
        float lo, hi;
        upk2(px, lo, hi); s_pos[a * 3] = lo; s_pos[b * 3] = hi;
        upk2(py, lo, hi); s_pos[a * 3 + 1] = lo; s_pos[b * 3 + 1] = hi;
        upk2(pz, lo, hi); s_pos[a * 3 + 2] = lo; s_pos[b * 3 + 2] = hi;
    }
    if (args.quat != nullptr) {
        if (prog.ee_axis != 0) { Ra = unpermute_cols(Ra, prog.ee_axis); Rb = unpermute_cols(Rb, prog.ee_axis); }
        reinterpret_cast<float4*>(s_quat)[a] = quat_xyzw(Ra);
        reinterpret_cast<float4*>(s_quat)[b] = quat_xyzw(Rb);
    }
}

// MAXLEN > 0: paths of at most MAXLEN links, loops fully unrolled, the Jacobian columns (z_i, z_i x p_i)
//             wait in REGISTERS for p_ee and are written to the smem tile exactly once;
// MAXLEN = 0: any path length, rolled loop, columns parked in the smem tile and fixed up in a second pass.
template <int NDOF, int TILE, bool WITH_JAC, int MAXLEN>
__global__ void __launch_bounds__(TILE)
fk_jacobian_kernel(const __grid_constant__ PathProgram prog, const FkArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = NDOF > 0 ? NDOF : prog.n_dofs;
    const int len = prog.len;
    const FkSmemLayout L(TILE, n, len, WITH_JAC);
    float* s_q = smem + L.q;
    float* s_pos = smem + L.pos;
    float* s_quat = smem + L.quat;
    float* s_jlin = smem + L.jlin;
    float* s_jang = smem + L.jang;
    float* s_tab = smem + L.table;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * TILE;
    const int valid = (int)min((int64_t)TILE, args.batch - tile_start);
    // bulk copies need 16-byte multiples: rows are 4n / 12 / 16 / 12n bytes -> valid % 4 == 0
    const bool bulk = args.use_bulk && args.aligned && ((valid & 3) == 0);
    const bool vec_ok = args.aligned;   // base pointers 16-byte aligned; tile offsets always are

    // Programmatic dependent launch (see "fk_pdl" in drm_b200.h): the next launch on the stream may start now; this grid
    // waits for its predecessor before its first global read (pdl 1) or only before its first global write (pdl 2)
    if (args.pdl) grid_dep_launch_dependents();
    if (args.pdl == 1) grid_dep_wait();

    // ---- stage inputs --------------------------------------------------------------------------
    if (bulk) {
        if (tid == 0) {
            mbar_init(&mbar, 1);
            fence_mbar_init();
            const uint32_t bytes = (uint32_t)valid * n * 4u;
            mbar_arrive_expect_tx(&mbar, bytes);
            bulk_g2s(s_q, args.q + tile_start * n, bytes, &mbar);
        }
    } else {
        coop_copy(s_q, args.q + tile_start * n, valid * n, vec_ok);
    }
    // canonical (F~, r~) rows of the path links -> smem (signed gather, map precomputed on the host)
    for (int i = tid; i < len * 12; i += TILE) {
        const uint32_t mp = prog.tab_map[i];
        const float v = __ldg(args.table + (mp & 0x7fffu));
        s_tab[i] = (mp & 0x8000u) ? -v : v;
    }
    if (WITH_JAC && !prog.full_cover) {      // columns of joints off the path stay zero
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float4* j4 = reinterpret_cast<float4*>(s_jlin);      // jlin and jang are adjacent
        for (int i = tid; i < (TILE * 6 * n) / 4; i += TILE) j4[i] = z4;
    }
    __syncthreads();
    if (bulk) mbar_wait(&mbar, 0);

    // ---- chain walk ----------------------------------------------------------------------------
    if (MAXLEN == -2) {
        // two configurations per thread: rows tid and tid + TILE/2 (row strides stay odd -> conflict-free); the upper
        // half of the CTA only helps with staging.  A ragged tail may leave lane b on an unused row: computed, never copied.
        if (tid < TILE / 2 && tid < valid)
            pair_walk<WITH_JAC>(prog, args, n, len, tid, tid + TILE / 2, s_q, s_pos, s_quat, s_jlin, s_jang, s_tab);
    } else if (tid < valid) {
        M3 R = identity3();
        V3 p = v3(0.f, 0.f, 0.f);
        const float* qrow = s_q + tid * n;
        float* jl = s_jlin + tid * 3 * n;
        float* ja = s_jang + tid * 3 * n;

        if (MAXLEN > 0) {
            V3 zs[MAXLEN > 0 ? MAXLEN : 1], ms[MAXLEN > 0 ? MAXLEN : 1];
            M3P Rp = identity3p();           // f32x2 pair state, see drm_common.cuh
            f32x2 pp = pk2(0.f, 0.f);
            float p2 = 0.f;
#pragma unroll
            for (int k = 0; k < MAXLEN; ++k) {
                zs[k] = ms[k] = v3(0.f, 0.f, 0.f);
                if (k < len) {
                    if (k == 0) walk_link<true, WITH_JAC>(s_tab, qrow, prog.dof[0], Rp, pp, p2, zs[0], ms[0]);
                    else walk_link<false, WITH_JAC>(s_tab + k * 12, qrow, prog.dof[k], Rp, pp, p2, zs[k], ms[k]);
                }
            }
            R = unpack3(Rp);
            upk2(pp, p.x, p.y);
            p.z = p2;
            if (WITH_JAC) {
                // J_lin[:,c] = z x (p_ee - p_i) = z x p_ee - z x p_i      (robot_model.py:661)
#pragma unroll
                for (int k = 0; k < MAXLEN; ++k) {
                    if (k < len) {
                        const int c = prog.dof[k];
                        if (c >= 0) {
                            const V3 z = zs[k];
                            const V3 j = cross_add(z, p, v3(-ms[k].x, -ms[k].y, -ms[k].z));
                            ja[c] = z.x; ja[n + c] = z.y; ja[2 * n + c] = z.z;
                            jl[c] = j.x; jl[n + c] = j.y; jl[2 * n + c] = j.z;
                        }
                    }
                }
            }
        } else {
            // explicit shared-window addresses (see smem_addr_opaque): table cursor, this thread's q / J rows
            uint32_t a_tab = smem_addr_opaque(s_tab);
            const uint32_t a_q = smem_addr_opaque(qrow);
            const uint32_t a_jl = smem_addr_opaque(jl), a_ja = smem_addr_opaque(ja);
            const uint32_t n4 = 4u * n;
            if (MAXLEN < 0) {
                walk_rolled_packed<WITH_JAC>(prog, len, a_tab, a_q, a_jl, a_ja, n4, R, p);
            } else {
            for (int k = 0; k < len; ++k, a_tab += 48) {
                M3 F; V3 r;
                load_Fr_s(a_tab, F, r);
                p = mul_add(R, r, p);            // p_i = R_parent r_i + p_parent
                R = mul(R, F);                   // R_parent F~_i
                const int c = prog.dof[k];
                if (c >= 0) {
                    float sn, cs;
                    sincos_pi2(lds_f32(a_q + 4u * c), sn, cs);
                    if (WITH_JAC) {
                        const V3 z = col2(R);    // joint axis in the world frame (unchanged by Rz)
                        const V3 m = cross(z, p);
                        const uint32_t o = 4u * c;
                        sts_f32(a_ja + o, z.x); sts_f32(a_ja + o + n4, z.y); sts_f32(a_ja + o + 2 * n4, z.z);
                        sts_f32(a_jl + o, m.x); sts_f32(a_jl + o + n4, m.y); sts_f32(a_jl + o + 2 * n4, m.z);
                    }
                    rotate_z(R, cs, sn);
                }
            }
            }
            if (WITH_JAC) jlin_fixup(prog, len, a_jl, a_ja, n4, p);
        }

        if (args.pos != nullptr) { s_pos[tid * 3 + 0] = p.x; s_pos[tid * 3 + 1] = p.y; s_pos[tid * 3 + 2] = p.z; }
        if (args.quat != nullptr) {
            if (prog.ee_axis != 0) R = unpermute_cols(R, prog.ee_axis);     // uniform; fixed ee links skip it
            reinterpret_cast<float4*>(s_quat)[tid] = quat_xyzw(R);
        }
    }

    // ---- stream the output tiles back ----------------------------------------------------------
    if (bulk) {
        fence_proxy_async();                 // generic-proxy smem writes -> visible to the async proxy
        __syncthreads();
        if (tid == 0) {
            if (args.pdl == 2) grid_dep_wait();
            if (args.pos != nullptr) bulk_s2g(args.pos + tile_start * 3, s_pos, (uint32_t)valid * 12u);
            if (args.quat != nullptr) bulk_s2g(args.quat + tile_start * 4, s_quat, (uint32_t)valid * 16u);
            if (WITH_JAC) {
                bulk_s2g(args.jlin + tile_start * 3 * n, s_jlin, (uint32_t)valid * 12u * n);
                bulk_s2g(args.jang + tile_start * 3 * n, s_jang, (uint32_t)valid * 12u * n);
            }
            bulk_commit();
            bulk_wait_read<0>();             // smem must stay intact until the copy engine has read it
        }
    } else {
        __syncthreads();
        if (args.pdl == 2) grid_dep_wait();
        if (args.pos != nullptr) coop_copy(args.pos + tile_start * 3, s_pos, valid * 3, vec_ok);
        if (args.quat != nullptr) coop_copy(args.quat + tile_start * 4, s_quat, valid * 4, vec_ok);
        if (WITH_JAC) {
            coop_copy(args.jlin + tile_start * 3 * n, s_jlin, valid * 3 * n, vec_ok);
            coop_copy(args.jang + tile_start * 3 * n, s_jang, valid * 3 * n, vec_ok);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
int fk_jacobian_multi_device(const drmb200_topology_t*, int32_t, const int32_t*, const float*, const float*, int64_t, float*,
                             float*, float*, float*, cudaStream_t);      // fk_tree.cu

int build_path_program(const drmb200_topology_t* topo, int32_t ee_link, PathProgram* prog) {
    if (topo == nullptr) { set_error("topology is null"); return DRMB200_EINVAL; }
    if (topo->n_links < 1 || topo->n_links > DRMB200_MAX_LINKS) {
        set_error("n_links=%d outside [1, %d]", topo->n_links, DRMB200_MAX_LINKS);
        return DRMB200_ELIMIT;
    }
    if (topo->n_dofs < 0 || topo->n_dofs > topo->n_links) { set_error("n_dofs=%d inconsistent", topo->n_dofs); return DRMB200_EINVAL; }
    if (ee_link < 0 || ee_link >= topo->n_links) {
        set_error("ee_link=%d outside [0, %d)", ee_link, topo->n_links);
        return DRMB200_EINVAL;
    }
    int chain[DRMB200_MAX_LINKS];
    int len = 0;
    for (int l = ee_link; l > 0; l = topo->parent[l]) {
        if (topo->parent[l] < 0 || topo->parent[l] >= l) {
            set_error("link %d: parent %d violates topological order", l, (int)topo->parent[l]);
            return DRMB200_EINVAL;
        }
        chain[len++] = l;
    }
    prog->len = len;
    prog->n_dofs = topo->n_dofs;
    prog->ee_axis = 0;
    int covered = 0;
    for (int k = 0; k < len; ++k) {
        const int l = chain[len - 1 - k];
        const int ax = topo->axis[l];
        prog->link[k] = (int8_t)l;
        prog->axis[k] = (int8_t)ax;
        prog->paxis[k] = (k == 0) ? 0 : prog->axis[k - 1];
        prog->dof[k] = (ax != 0) ? topo->dof[l] : (int8_t)-1;
        if (ax != 0) {
            if (topo->dof[l] < 0 || topo->dof[l] >= topo->n_dofs || ax > 3 || ax < -3) {
                set_error("link %d: bad dof/axis (%d, %d)", l, (int)topo->dof[l], ax);
                return DRMB200_EINVAL;
            }
            ++covered;
        }
        if (k == len - 1) prog->ee_axis = ax;
        for (int e = 0; e < 12; ++e) {          // signed gather map of the canonical (F~, r~) row
            int src;
            const float sg = canon_map(e, prog->paxis[k], ax, src);
            prog->tab_map[k * 12 + e] = (uint16_t)((l * DRMB200_TABLE_STRIDE + src) | (sg < 0.f ? 0x8000 : 0));
        }
    }
    prog->full_cover = (covered == topo->n_dofs) ? 1 : 0;
    return DRMB200_OK;
}

template <int NDOF, int TILE, bool WITH_JAC, int MAXLEN>
static int launch_fk(const PathProgram& prog, const FkArgs& args, cudaStream_t stream) {
    constexpr auto kern = fk_jacobian_kernel<NDOF, TILE, WITH_JAC, MAXLEN>;
    const size_t smem_bytes = (size_t)FkSmemLayout(TILE, prog.n_dofs, prog.len, WITH_JAC).total_floats * sizeof(float);
    size_t static_bytes;
    const int rc = static_smem_bytes<kern>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    if (smem_bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("fk kernel needs %zu B of shared memory per CTA (> 227 KB)", smem_bytes + static_bytes);
        return DRMB200_ELIMIT;
    }
    return launch_kernel<kern>((args.batch + TILE - 1) / TILE, TILE, smem_bytes, stream, args.pdl != 0, "fk_jacobian", prog, args);
}

template <int NDOF, int TILE, bool WITH_JAC>
static int launch_fk_l(const PathProgram& prog, const FkArgs& args, cudaStream_t stream) {
    // Rolled vs unrolled: for odd n (Kuka, 7) the rolled kernel wins.  For even n the per-thread J rows have even
    // strides -> 16-way bank conflicts on every J access; the unrolled kernel touches the J tile once per column instead
    // of three times and wins (Allegro, n = 16).  Chosen by sweeps before the H100 port; not re-measured on the H100.
    const int opt = get_option(2);                     // 0 rolled, 1 unrolled, 2 auto
    const bool unrolled = prog.len <= 8 && (opt == 1 || (opt != 0 && (prog.n_dofs % 2) == 0));
    if (unrolled) return launch_fk<NDOF, TILE, WITH_JAC, 8>(prog, args, stream);
    // rolled walk: f32x2 pair arithmetic unless switched off for A/B measurements
    // fk_packed = 2: two configurations per thread in the two f32x2 lanes (A/B candidate, see pair_walk)
    const int packed = get_option(3);
    if (packed == 2) return launch_fk<NDOF, TILE, WITH_JAC, -2>(prog, args, stream);
    return packed != 0 ? launch_fk<NDOF, TILE, WITH_JAC, -1>(prog, args, stream)
                       : launch_fk<NDOF, TILE, WITH_JAC, 0>(prog, args, stream);
}
template <int NDOF, int TILE>
static int launch_fk_j(bool with_jac, const PathProgram& prog, const FkArgs& args, cudaStream_t stream) {
    return with_jac ? launch_fk_l<NDOF, TILE, true>(prog, args, stream) : launch_fk_l<NDOF, TILE, false>(prog, args, stream);
}
template <int NDOF>
static int launch_fk_t(int tile, bool with_jac, const PathProgram& prog, const FkArgs& args, cudaStream_t stream) {
    if (tile == 64) return launch_fk_j<NDOF, 64>(with_jac, prog, args, stream);
    if (tile == 256) return launch_fk_j<NDOF, 256>(with_jac, prog, args, stream);
    return launch_fk_j<NDOF, 128>(with_jac, prog, args, stream);
}

// ---- programmatic dependent launch: which mode is safe for THIS launch -------------------------------------------
// "fk_pdl" 2 lets a launch run ahead of its predecessors on the stream up to its first global WRITE.  Only FK launches
// release their dependents early, so the only stream-order hazard is a launch READING (q, table) what one of the FK
// launches still in flight ahead of it writes.  How many can be in flight: a launch starts only when every CTA of its
// predecessor has started, and a started CTA keeps its shared memory until its own predecessor grid has completed, so the
// grids ahead of a launch that are not yet complete are all fully resident -- at most 1 / f of them, f = the share of the
// GPU's shared memory one grid takes.  The library therefore (a) uses mode 2 only for launches with f >= 1/4 and (b) keeps
// the output ranges of the last 8 FK / multi-link FK launches per (device, stream) and falls back to an ordinary launch whenever an input
// of the new launch overlaps one of them.  Writes need no check: every launch waits for its predecessor before writing.
struct StreamLog { int dev; cudaStream_t stream; bool used; int head; PdlRange out[8][4]; };
static StreamLog g_logs[16];
static std::mutex g_log_mu;
static int g_log_clock = 0;

static bool overlaps(const PdlRange& a, const PdlRange& b) { return a.lo < b.hi && b.lo < a.hi; }

int device_sm_count() {
    static int sms_by_dev[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    int& sms = sms_by_dev[dev & 63];
    if (sms == 0 && (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)) { cudaGetLastError(); sms = 132; }
    return sms;
}

// mode the launch may use (0 or the requested one) + log its output ranges; f above = grid_smem_bytes over the
// device's shared memory (227 KB per SM)
int pdl_decide(cudaStream_t stream, const PdlRange* ins, int n_ins, const PdlRange outs[4], double grid_smem_bytes) {
    int mode = get_option(7);
    if (mode < 0 || mode > 2) mode = 0;
    const double smem_share = grid_smem_bytes / ((double)device_sm_count() * 227.0 * 1024.0);
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(g_log_mu);
    StreamLog* log = nullptr;
    for (auto& l : g_logs) if (l.used && l.dev == dev && l.stream == stream) { log = &l; break; }
    if (log == nullptr) {                                   // claim a slot (round robin; a recycled slot starts empty)
        log = &g_logs[g_log_clock++ & 15];
        *log = StreamLog();
        log->used = true; log->dev = dev; log->stream = stream;
        // nothing is known about the FK launches that may still be in flight on this stream (first use, or its history
        // was evicted by 16 other streams): this launch is an ordinary one -- it starts after everything before it on the
        // stream has completed, so whatever was forgotten cannot matter to the launches that follow it
        mode = 0;
    }
    if (mode == 2) {
        if (smem_share < 0.25) mode = 0;
        for (int k = 0; k < 8 && mode == 2; ++k)
            for (int o = 0; o < 4 && mode == 2; ++o)
                for (int i = 0; i < n_ins && mode == 2; ++i)
                    if (overlaps(log->out[k][o], ins[i])) mode = 0;
    }
    for (int o = 0; o < 4; ++o) log->out[log->head][o] = outs[o];
    log->head = (log->head + 1) & 7;
    return mode;
}

static int pdl_mode_for_launch(const PathProgram& prog, const FkArgs& args, int n_links, cudaStream_t stream) {
    const int n = prog.n_dofs;
    const uintptr_t B = (uintptr_t)args.batch;
    const PdlRange outs[4] = {pdl_range(args.pos, B * 12), pdl_range(args.quat, B * 16), pdl_range(args.jlin, B * 12 * n),
                              pdl_range(args.jang, B * 12 * n)};
    const PdlRange ins[2] = {pdl_range(args.q, B * 4 * n), pdl_range(args.table, (uintptr_t)n_links * DRMB200_TABLE_STRIDE * 4)};
    // share of the GPU's shared memory this grid takes (the residency bound above)
    const double smem_per_config = 4.0 * (n + 7 + (args.jlin ? 6 * n : 0));
    return pdl_decide(stream, ins, 2, outs, smem_per_config * (double)args.batch);
}

int fk_jacobian_device(const drmb200_topology_t* topo, int32_t ee_link, const float* table, const float* q,
                       int64_t batch, float* pos, float* quat, float* jlin, float* jang, cudaStream_t stream) {
    // the path program depends only on (topology, ee_link): keep the last few per thread instead of rebuilding the
    // 1.8 KB structure (and its signed gather map) on every call -- first-order for batch-1 calls
    struct CachedProgram { bool valid; int32_t ee; drmb200_topology_t topo; PathProgram prog; };
    static thread_local CachedProgram cache[4] = {};
    static thread_local int cache_next = 0;
    if (topo == nullptr) { set_error("topology is null"); return DRMB200_EINVAL; }
    const PathProgram* cached = nullptr;
    for (auto& c : cache)
        if (c.valid && c.ee == ee_link && memcmp(&c.topo, topo, sizeof(*topo)) == 0) { cached = &c.prog; break; }
    if (cached == nullptr) {
        CachedProgram& c = cache[cache_next];
        c.valid = false;
        int rc = build_path_program(topo, ee_link, &c.prog);
        if (rc != DRMB200_OK) return rc;
        c.topo = *topo; c.ee = ee_link; c.valid = true;
        cache_next = (cache_next + 1) & 3;
        cached = &c.prog;
    }
    const PathProgram& prog = *cached;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if ((jlin == nullptr) != (jang == nullptr)) { set_error("jac_lin and jac_ang must both be given or both be null"); return DRMB200_EINVAL; }
    if (batch == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr) { set_error("table / q is null"); return DRMB200_EINVAL; }
    if (pos == nullptr && quat == nullptr && jlin == nullptr) return DRMB200_OK;

    FkArgs args;
    args.table = table; args.q = q; args.pos = pos; args.quat = quat; args.jlin = jlin; args.jang = jang;
    args.batch = batch;
    args.aligned = aligned16(q, pos, quat, jlin, jang);
    args.use_bulk = get_option(0) != 0;
    const bool with_jac = jlin != nullptr;
    // n_dofs % 4 == 0 (Allegro, n = 16): the per-lane rows of this kernel's natural-layout tiles are 16-way bank
    // conflicts; the tree-walk kernel (fk_tree.cu) assembles 16-byte column chunks instead.  For one Allegro fingertip the
    // tree kernel was the faster of the two at 2^21 per launch and the slower at 32 768 -- so large batches are routed to
    // the tree kernel, small ones stay (chosen before the H100 port; not re-measured on the H100).
    if ((prog.n_dofs & 3) == 0 && prog.n_dofs > 0 && batch >= 262144 && get_option(2) == 2)
        return fk_jacobian_multi_device(topo, 1, &ee_link, table, q, batch, pos, quat, jlin, jang, stream);
    args.pdl = pdl_mode_for_launch(prog, args, topo->n_links, stream);


    // Tile size (Kuka, rolled kernel; chosen by sweeps before the H100 port, not re-measured on the H100):
    //   large batches: tile 64 (shared memory, 32 n + 28 bytes per configuration, is the occupancy limiter: smaller
    //                  tiles pack SMs tighter); 256 is slowest
    //   batches up to 1 Ki per SM without programmatic dependent launch: tile 128 (fewer CTAs, shorter sub-wave ramp)
    //   wide rows (n > 8, e.g. the 16-DoF Allegro hand): 128 (even row strides: bank conflicts hurt the narrower tile more)
    //   with programmatic dependent launch (fk_pdl 2) consecutive launches overlap and the sub-wave ramp no longer
    //   matters: tile 64
    int tile = get_option(1);
    if (tile != 64 && tile != 128 && tile != 256)
        tile = (prog.n_dofs > 8 || (batch <= (int64_t)device_sm_count() * 1024 && args.pdl != 2)) ? 128 : 64;
    // a long path with many Jacobian columns (e.g. a 63-DoF chain) does not fit 128 rows: take 64 (the kernel's static
    // shared memory counts against the same 227 KB, hence the margin)
    if (tile == 128 && (size_t)FkSmemLayout(128, prog.n_dofs, prog.len, with_jac).total_floats * sizeof(float) + 1024 > SMEM_CTA_MAX)
        tile = 64;
    switch (prog.n_dofs) {
        case 2: return launch_fk_t<2>(tile, with_jac, prog, args, stream);
        case 7: return launch_fk_t<7>(tile, with_jac, prog, args, stream);
        case 9: return launch_fk_t<9>(tile, with_jac, prog, args, stream);
        case 12: return launch_fk_t<12>(tile, with_jac, prog, args, stream);
        case 16: return launch_fk_t<16>(tile, with_jac, prog, args, stream);
        case 23: return launch_fk_t<23>(tile, with_jac, prog, args, stream);
        default: return launch_fk_t<0>(tile, with_jac, prog, args, stream);
    }
}

}  // namespace drm
