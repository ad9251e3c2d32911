// rnea.cu -- batched recursive Newton-Euler inverse dynamics (sm_90a).
//
// Replaces, in ONE launch, DifferentiableRobotModel.compute_inverse_dynamics (robot_model.py:306-375):
// update_kinematic_state (robot_model.py:140-195, velocities), update_joint_acc (rigid_body.py:159-165),
// iterative_newton_euler (robot_model.py:251-303: acceleration pass root->leaves, force pass
// leaves->root, spatial_vector_algebra.py:204-236, 281-291, 321-338), the axis projection
// (robot_model.py:353-365) and the damping term (robot_model.py:368-373).
//
// Closed form (SURVEY.md section 8a, verified against the reference), link i, parent p, in the canonical
// joint frames of drm_common.cuh (every joint axis is e_z, joint rate (0,0,qd)):
//   M = F~ Rz(q),  E = M^T,  r = r~
//   w_i  = E w_p + (0,0,qd)                 v_i = E (v_p + w_p x r)
//   al_i = E al_p + (0,0,qdd) + w_i x (0,0,qd)
//   a_i  = E (a_p + al_p x r) + v_i x (0,0,qd)                        (a_0 = (0,0,9.81))
//   h(W,V) = ( m V - mc x W ,  I_o W + mc x V )
//   f_i  = h_lin(al,a) + w x h_lin(w,v)
//   n_i  = h_ang(al,a) + w x h_ang(w,v) + v x h_lin(w,v)
//   f_p += M f_i ;  n_p += r x (M f_i) + M n_i ;  tau_k = n_i.z + d_i qd_k
//
// Mapping: one thread per configuration (RNEA_TILE per CTA).  The motion state (w, v, al, a) of the
// current link lives in registers; only branch points of the tree spill it to shared-memory slots
// (host-computed "tree program", by-value kernel parameter).  Per-link body wrenches (f, n) and the
// joint (cos, sin) are kept in shared memory, slot-major ([slot][thread] -> conflict-free), for the
// leaves->root pass, where children accumulate into their parent's slot.
// q / qd / qdd tiles in and the tau tile out are staged in the global row-major layout and moved
// with TMA 1-D bulk copies (cooperative float4 copies for ragged tails / unaligned bases).
//
// Algorithmic HBM bytes per configuration: 12n in + 4n out = 16n (112 B at n = 7).  At roughly
// 2 kflop per 7-DoF configuration the kernel is FP32-issue-bound, not HBM-bound (SURVEY.md 8d).
#include <cstdlib>
#include <cstring>
#include "launch.cuh"

namespace drm {

// configurations per CTA: template parameter T of the kernel, 64 or 128 (see rnea_tile)
constexpr float GRAVITY = 9.81f;     // robot_model.py:347

struct RneaArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ qdd;
    float* __restrict__ tau;             // [B, n] or null (DUMP launches may skip it)
    float* __restrict__ vels;            // DUMP: [n_links, 6, B] body-frame spatial velocity  (ang 3, lin 3), or null
    float* __restrict__ accs;            // DUMP: [n_links, 6, B] body-frame spatial acceleration (ang 3, lin 3), or null
    float* __restrict__ forces;          // DUMP: [n_links, 6, B] accumulated body wrench (ang = torque 3, lin = force 3), or null
    int64_t batch;
    uint32_t flags;
    int32_t aligned;
};

// natural vector from a canonical one:  x[idx(c)] = sgn(c) x~[c]
__device__ __forceinline__ V3 rnea_unpermute(V3 xt, int code) {
    const int a = code < 0 ? -code : code;
    const float s = code < 0 ? -1.f : 1.f;
    const float c0 = xt.x, c1 = s * xt.y, c2 = s * xt.z;
    if (a == 1) return v3(c2, c0, c1);
    if (a == 2) return v3(c1, c2, c0);
    return v3(c0, c1, c2);
}

struct RneaSmemLayout {
    int q, qd, qdd, tau, table, link, slots, total_floats;
    __host__ __device__ RneaSmemLayout(int RNEA_TILE, int n, int n_links, int n_slots) {
        int o = 0;
        q = o;   o += RNEA_TILE * n;
        qd = o;  o += RNEA_TILE * n;
        qdd = o; o += RNEA_TILE * n;
        tau = qdd;                                        // qdd is dead after pass 1: tau is written over it
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o;  o += n_links * 8 * RNEA_TILE;          // per link: f(3) n(3) cos sin, slot-major
        slots = o; o += n_slots * 12 * RNEA_TILE;         // branch-point motion states
        total_floats = o;
    }
};

// DUMP additionally writes the per-link state the reference leaves in `_bodies[i].vel / .acc / .force`
// (robot_model.py:183-193, 262-301), un-permuted to the natural link frames, link-major / component-major (coalesced).
// (A per-warp pipeline version of this kernel -- persistent grid, no CTA barrier, like fk_tree.cu -- was slower than this
// CTA-tile form on the Panda: the kernel is issue-bound and the extra loop / addressing instructions cost more than the
// barrier stalls they remove.)
template <int T, bool PACKED, bool DUMP, bool FOLD>
__global__ void __launch_bounds__(T)
rnea_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold, const RneaArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = prog.n_dofs;
    const int N = prog.n_links;
    const RneaSmemLayout L(T, n, N, prog.n_slots);
    float* s_q = smem + L.q;
    float* s_qd = smem + L.qd;
    float* s_qdd = smem + L.qdd;
    float* s_tau = smem + L.tau;
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_slot = smem + L.slots;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * T;
    const int valid = (int)min((int64_t)T, args.batch - tile_start);
    const bool vec_ok = args.aligned;
    const bool bulk = args.aligned && ((valid & 3) == 0);

    if (bulk) {
        if (tid == 0) {
            mbar_init(&mbar, 1);
            fence_mbar_init();
            const uint32_t bytes = (uint32_t)valid * n * 4u;
            mbar_arrive_expect_tx(&mbar, 3u * bytes);
            bulk_g2s(s_q, args.q + tile_start * n, bytes, &mbar);
            bulk_g2s(s_qd, args.qd + tile_start * n, bytes, &mbar);
            bulk_g2s(s_qdd, args.qdd + tile_start * n, bytes, &mbar);
        }
    } else {
        coop_copy(s_q, args.q + tile_start * n, valid * n, vec_ok);
        coop_copy(s_qd, args.qd + tile_start * n, valid * n, vec_ok);
        coop_copy(s_qdd, args.qdd + tile_start * n, valid * n, vec_ok);
    }
    if (FOLD) {
        if (fold.n_full == 0) {        // args.table already holds the folded canonical rows (drmb200_fold_link_table): plain copy
            for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += T) s_tab[i] = __ldg(args.table + i);
        } else {
            stage_folded_table(s_tab, s_link, args.table, fold, prog, T);      // s_link: scratch until the walk starts
        }
    } else {
        stage_canonical_table(s_tab, args.table, prog, T);
    }
    __syncthreads();
    if (bulk) mbar_wait(&mbar, 0);

    if (tid < valid) {
        // explicit 32-bit shared-window addresses (see smem_addr_opaque in drm_common.cuh)
        const uint32_t a_q = smem_addr_opaque(s_q + tid * n), a_qd = smem_addr_opaque(s_qd + tid * n);
        const uint32_t a_qdd = smem_addr_opaque(s_qdd + tid * n), a_tau = smem_addr_opaque(s_tau + tid * n);
        const uint32_t a_tab = smem_addr_opaque(s_tab);
        const uint32_t a_link = smem_addr_opaque(s_link + tid), a_slot = smem_addr_opaque(s_slot + tid);
        constexpr uint32_t E = 4u * T;                      // byte stride between elements of a slot-major vector
        auto ldv_s = [](uint32_t a) { return v3(lds_f32(a), lds_f32(a + E), lds_f32(a + 2 * E)); };
        auto stv_s = [](uint32_t a, V3 x) { sts_f32(a, x.x); sts_f32(a + E, x.y); sts_f32(a + 2 * E, x.z); };
        const float g = (args.flags & DRMB200_GRAVITY) ? GRAVITY : 0.f;
        const bool damp = (args.flags & DRMB200_DAMPING) != 0;
        const int64_t B = args.batch;
        const int64_t b = tile_start + tid;
        auto dump6 = [&](float* base, int link, V3 ang, V3 lin) {        // natural link frame, [n_links, 6, B]
            if (base == nullptr) return;
            const int code = prog.axis[link];
            const V3 x = rnea_unpermute(ang, code), y = rnea_unpermute(lin, code);
            float* o = base + ((int64_t)link * 6) * B + b;
            o[0] = x.x; o[B] = x.y; o[2 * B] = x.z; o[3 * B] = y.x; o[4 * B] = y.y; o[5 * B] = y.z;
        };

        // ---- pass 1: root -> leaves, motion state + body wrench ------------------------------------
        // f32x2 pair arithmetic (drm_common.cuh): the velocity-level and the acceleration-level quantities obey the
        // same linear maps, so they travel as PAIRS -- W = (w | al), V = (v | a) -- and every 3x3 product, cross
        // product with r and spatial-inertia product is written once for both.
        const V3 zero = v3(0.f, 0.f, 0.f);
        V3P W = pk3(zero, zero), V = W;                     // state of the previously processed link
        if (DUMP) {                                         // the root: zero velocity, base acceleration, wrench accumulator
            stv_s(a_link, zero); stv_s(a_link + 3 * E, zero);
            dump6(args.vels, 0, zero, zero); dump6(args.accs, 0, zero, v3(0.f, 0.f, g));
        }
        for (int i = 1; i < N; ++i) {
            if (PACKED) {
                const uint32_t row = a_tab + i * (DRMB200_TABLE_STRIDE * 4);
                LinkRow C;
                load_Fr_s(row, C.F, C.r);
                {
                    const float4 d = lds_f32x4(row + 48), e = lds_f32x4(row + 64), f = lds_f32x4(row + 80), gg = lds_f32x4(row + 96);
                    C.Io.a00 = d.x; C.Io.a01 = d.y; C.Io.a02 = d.z; C.Io.a10 = d.w; C.Io.a11 = e.x; C.Io.a12 = e.y;
                    C.Io.a20 = e.z; C.Io.a21 = e.w; C.Io.a22 = f.x;
                    C.mc = v3(f.y, f.z, f.w);
                    C.m = gg.x; C.d = gg.y;
                }
                const int src = prog.psrc[i];
                V3P Wp, Vp;
                if (src == 0) { Wp = W; Vp = V; }
                else if (src < 0) { Wp = pk3(zero, zero); Vp = pk3(zero, v3(0.f, 0.f, g)); }
                else {
                    const uint32_t sl = a_slot + (src - 1) * 12 * E;
                    Wp = pk3(ldv_s(sl), ldv_s(sl + 6 * E)); Vp = pk3(ldv_s(sl + 3 * E), ldv_s(sl + 9 * E));
                }
                // E x = Rz^T (F~^T x): velocities (robot_model.py:183-193), accelerations (robot_model.py:269-277)
                W = mulT_p(C.F, Wp);
                V = mulT_p(C.F, cross_add_p(Wp, C.r, Vp));
                const int c = prog.dof[i];
                float cs = 1.f, sn = 0.f, qd_k = 0.f, qdd_k = 0.f;
                if (c >= 0) {
                    qd_k = lds_f32(a_qd + 4u * c); qdd_k = lds_f32(a_qdd + 4u * c);
                    sincos_pi2(lds_f32(a_q + 4u * c), sn, cs);
                }
                // one code path for fixed links too (cs = 1, sn = 0, zero rates are exact no-ops): only four scalars
                // cross the branch above, the packed state is never shuffled at a join
                W = rotzT_p(W, cs, sn);
                V = rotzT_p(V, cs, sn);
                V3 w, al, v, a;
                upk3(W, w, al); upk3(V, v, a);
                w.z += qd_k;
                al.x = fmaf(w.y, qd_k, al.x); al.y = fmaf(-w.x, qd_k, al.y); al.z += qdd_k;         // + w x (0,0,qd) + (0,0,qdd)
                a.x = fmaf(v.y, qd_k, a.x); a.y = fmaf(-v.x, qd_k, a.y);                            // + v x (0,0,qd)
                W = pk3(w, al); V = pk3(v, a);
                if (DUMP) { dump6(args.vels, i, w, v); dump6(args.accs, i, al, a); }
                // body wrench (robot_model.py:289-293; spatial_vector_algebra.py:321-338), both lanes at once
                V3 hl_v, hl_a, ha_v, ha_a;
                upk3(inertia_lin_p(C.m, C.mc, W, V), hl_v, hl_a);
                upk3(inertia_ang_p(C.Io, C.mc, W, V), ha_v, ha_a);
                const V3 f = cross_add(w, hl_v, hl_a);
                const V3 nn = cross_add(w, ha_v, cross_add(v, hl_v, ha_a));
                const uint32_t lk = a_link + i * 8 * E;
                stv_s(lk, f); stv_s(lk + 3 * E, nn);
                sts_f32(lk + 6 * E, cs); sts_f32(lk + 7 * E, sn);
                const int sv = prog.save[i];
                if (sv >= 0) {
                    const uint32_t sl = a_slot + sv * 12 * E;
                    stv_s(sl, w); stv_s(sl + 3 * E, v); stv_s(sl + 6 * E, al); stv_s(sl + 9 * E, a);
                }
                continue;
            }
            V3 w, al, v, a;
            upk3(W, w, al); upk3(V, v, a);
            const uint32_t row = a_tab + i * (DRMB200_TABLE_STRIDE * 4);
            LinkRow C;
            load_Fr_s(row, C.F, C.r);
            {
                const float4 d = lds_f32x4(row + 48), e = lds_f32x4(row + 64), f = lds_f32x4(row + 80), gg = lds_f32x4(row + 96);
                C.Io.a00 = d.x; C.Io.a01 = d.y; C.Io.a02 = d.z; C.Io.a10 = d.w; C.Io.a11 = e.x; C.Io.a12 = e.y;
                C.Io.a20 = e.z; C.Io.a21 = e.w; C.Io.a22 = f.x;
                C.mc = v3(f.y, f.z, f.w);
                C.m = gg.x; C.d = gg.y;
            }
            const int src = prog.psrc[i];
            V3 wp, vp, alp, ap;
            if (src == 0) { wp = w; vp = v; alp = al; ap = a; }
            else if (src < 0) { wp = vp = alp = v3(0.f, 0.f, 0.f); ap = v3(0.f, 0.f, g); }
            else {
                const uint32_t sl = a_slot + (src - 1) * 12 * E;
                wp = ldv_s(sl); vp = ldv_s(sl + 3 * E); alp = ldv_s(sl + 6 * E); ap = ldv_s(sl + 9 * E);
            }
            M3 M = C.F;
            const int c = prog.dof[i];
            float cs = 1.f, sn = 0.f, qd_k = 0.f, qdd_k = 0.f;
            if (c >= 0) {
                qd_k = lds_f32(a_qd + 4u * c);
                qdd_k = lds_f32(a_qdd + 4u * c);
                sincos_pi2(lds_f32(a_q + 4u * c), sn, cs);
                rotate_z(M, cs, sn);
            }
            // velocities (robot_model.py:183-193), accelerations (robot_model.py:269-277)
            w = mulT(M, wp); w.z += qd_k;
            v = mulT(M, cross_add(wp, C.r, vp));
            al = mulT(M, alp) + cross_z(w, qd_k); al.z += qdd_k;
            a = mulT(M, cross_add(alp, C.r, ap)) + cross_z(v, qd_k);
            if (DUMP) { dump6(args.vels, i, w, v); dump6(args.accs, i, al, a); }
            // body wrench (robot_model.py:289-293; spatial_vector_algebra.py:321-338)
            const V3 hl_a = C.m * a - cross(C.mc, al);
            const V3 ha_a = mul_add(C.Io, al, cross(C.mc, a));
            const V3 hl_v = C.m * v - cross(C.mc, w);
            const V3 ha_v = mul_add(C.Io, w, cross(C.mc, v));
            const V3 f = cross_add(w, hl_v, hl_a);
            const V3 nn = cross_add(w, ha_v, cross_add(v, hl_v, ha_a));
            const uint32_t lk = a_link + i * 8 * E;
            stv_s(lk, f); stv_s(lk + 3 * E, nn);
            sts_f32(lk + 6 * E, cs); sts_f32(lk + 7 * E, sn);
            const int sv = prog.save[i];
            if (sv >= 0) {
                const uint32_t sl = a_slot + sv * 12 * E;
                stv_s(sl, w); stv_s(sl + 3 * E, v); stv_s(sl + 6 * E, al); stv_s(sl + 9 * E, a);
            }
            W = pk3(w, al); V = pk3(v, a);
        }

        // ---- pass 2: leaves -> root, wrench propagation + joint torques (robot_model.py:284-301, 353-373)
        // The wrench a link hands to its parent travels in REGISTERS when the parent is the link processed next
        // (parent == i - 1: always, on a chain); only children of far branch points accumulate into their parent's
        // shared-memory slot.  prog.tip[i] < 0 says that link i + 1 is a child of i, i.e. `carry` is meant for link i.
        V3 carry_f = zero, carry_n = zero;
        for (int i = N - 1; i >= 1; --i) {
            const uint32_t lk = a_link + i * 8 * E;
            V3 f = ldv_s(lk);
            V3 nn = ldv_s(lk + 3 * E);
            if (i + 1 < N && prog.tip[i] < 0) { f = f + carry_f; nn = nn + carry_n; }
            if (DUMP) dump6(args.forces, i, nn, f);
            const int c = prog.dof[i];
            const uint32_t row = a_tab + i * (DRMB200_TABLE_STRIDE * 4);
            if (c >= 0) {
                float t = nn.z;
                if (damp) t = fmaf(lds_f32(row + 100), lds_f32(a_qd + 4u * c), t);
                sts_f32(a_tau + 4u * c, t);
            }
            const int p = prog.parent[i];
            if (p > 0 || (DUMP && p == 0)) {                // the fused kernel never needs the wrench on the root
                M3 F; V3 r;
                load_Fr_s(row, F, r);
                const float cs = lds_f32(lk + 6 * E), sn = lds_f32(lk + 7 * E);
                V3 fp, np;
                if (PACKED) {                                       // (M f | M n) = F~ (Rz (f | n))  (sva:281-291)
                    upk3(mul_pv(F, rotz_p(pk3(f, nn), cs, sn)), fp, np);
                    np = cross_add(r, fp, np);
                } else {
                    fp = mul(F, rotz(f, cs, sn));
                    np = cross_add(r, fp, mul(F, rotz(nn, cs, sn)));
                }
                if (p == i - 1) {
                    carry_f = fp; carry_n = np;
                } else {
                    const uint32_t pk = a_link + p * 8 * E;
                    stv_s(pk, ldv_s(pk) + fp);
                    stv_s(pk + 3 * E, ldv_s(pk + 3 * E) + np);
                }
            }
        }
        if (DUMP) dump6(args.forces, 0, ldv_s(a_link + 3 * E) + carry_n, ldv_s(a_link) + carry_f);     // link 1 is a child of the root
    }

    if (args.tau == nullptr) return;
    if (bulk) {
        fence_proxy_async();
        __syncthreads();
        if (tid == 0) {
            bulk_s2g(args.tau + tile_start * n, s_tau, (uint32_t)valid * n * 4u);
            bulk_commit();
            bulk_wait_read<0>();
        }
    } else {
        __syncthreads();
        coop_copy(args.tau + tile_start * n, s_tau, valid * n, vec_ok);
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
int build_tree_program(const drmb200_topology_t* topo, TreeProgram* prog) {
    if (topo == nullptr) { set_error("topology is null"); return DRMB200_EINVAL; }
    const int N = topo->n_links;
    if (N < 1 || N > DRMB200_MAX_LINKS) { set_error("n_links=%d outside [1, %d]", N, DRMB200_MAX_LINKS); return DRMB200_ELIMIT; }
    if (topo->n_dofs < 0 || topo->n_dofs > N) { set_error("n_dofs=%d inconsistent with n_links=%d", topo->n_dofs, N); return DRMB200_EINVAL; }
    prog->n_links = N;
    prog->n_dofs = topo->n_dofs;
    int last_far_child[DRMB200_MAX_LINKS];      // last child c of i with c != i+1, or -1
    for (int i = 0; i < N; ++i) last_far_child[i] = -1;
    for (int i = 1; i < N; ++i) {
        const int p = topo->parent[i];
        if (p < 0 || p >= i) { set_error("link %d: parent %d violates topological order", i, p); return DRMB200_EINVAL; }
        const int ax = topo->axis[i];
        if (ax < -3 || ax > 3) { set_error("link %d: bad axis code %d", i, ax); return DRMB200_EINVAL; }
        if (ax != 0 && (topo->dof[i] < 0 || topo->dof[i] >= topo->n_dofs)) { set_error("link %d: bad dof %d", i, (int)topo->dof[i]); return DRMB200_EINVAL; }
        prog->parent[i] = (int8_t)p;
        prog->axis[i] = (int8_t)ax;
        prog->dof[i] = (ax != 0) ? topo->dof[i] : (int8_t)-1;
        if (p != i - 1 && p != 0) last_far_child[p] = i;
    }
    prog->parent[0] = -1; prog->axis[0] = 0; prog->dof[0] = -1; prog->psrc[0] = -1; prog->save[0] = -1; prog->accw[0] = 0;
    int slot_of[DRMB200_MAX_LINKS];
    int slot_free_after[DRM_MAX_SLOTS];
    for (int s = 0; s < DRM_MAX_SLOTS; ++s) slot_free_after[s] = -1;
    int n_slots = 0;
    for (int i = 1; i < N; ++i) {
        const int p = topo->parent[i];
        prog->psrc[i] = (p == 0) ? -1 : (p == i - 1 ? 0 : (int8_t)(1 + slot_of[p]));
        prog->save[i] = -1;
        prog->accw[i] = (p == 0 || p == i - 1) ? 0 : (last_far_child[p] == i ? 2 : 1);
        if (last_far_child[i] >= 0) {
            int s = 0;
            while (s < DRM_MAX_SLOTS && slot_free_after[s] >= i) ++s;
            if (s == DRM_MAX_SLOTS) { set_error("tree needs more than %d live branch points", DRM_MAX_SLOTS); return DRMB200_ELIMIT; }
            slot_of[i] = s;
            slot_free_after[s] = last_far_child[i];
            prog->save[i] = (int8_t)s;
            if (s + 1 > n_slots) n_slots = s + 1;
        }
    }
    prog->n_slots = n_slots;
    int n_tips = 0;
    prog->tip[0] = -1;
    for (int i = 1; i < N; ++i) prog->tip[i] = (i + 1 < N && topo->parent[i + 1] == i) ? (int8_t)-1 : (int8_t)n_tips++;
    prog->n_tips = n_tips;
    return DRMB200_OK;
}

template <int T, bool PACKED, bool DUMP, bool FOLD>
static int launch_rnea(const TreeProgram& prog, const FoldProgram& fold, const RneaArgs& args, cudaStream_t stream) {
    const size_t smem_bytes = (size_t)RneaSmemLayout(T, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float);
    if (smem_bytes > SMEM_CTA_MAX) { set_error("model needs %zu B of shared memory per CTA (> 227 KB)", smem_bytes); return DRMB200_ELIMIT; }
    return launch_kernel<rnea_kernel<T, PACKED, DUMP, FOLD>>((args.batch + T - 1) / T, T, smem_bytes, stream, false, "rnea", prog,
                                                             fold, args);
}

// the tree program (and the folded one) depend only on the topology: keep the last two per thread

static int build_fold(const drmb200_topology_t* topo, TreeProgram* red, FoldProgram* fold, bool* foldable) {
    const int N = topo->n_links;
    memset(fold, 0, sizeof(*fold));
    fold->n_full = N;
    drmb200_topology_t rt;
    memset(&rt, 0, sizeof(rt));
    int n_red = 1, n_fixed = 0;
    fold->full_of[0] = 0; fold->red_of[0] = 0; fold->parent[0] = -1; fold->axis[0] = 0;
    rt.parent[0] = -1; rt.axis[0] = 0; rt.dof[0] = -1;
    for (int l = 1; l < N; ++l) {
        fold->parent[l] = topo->parent[l];
        fold->axis[l] = topo->axis[l];
        if (topo->axis[l] != 0) {
            const int j = n_red++;
            fold->full_of[j] = (int8_t)l;
            fold->red_of[l] = (int8_t)j;
            rt.parent[j] = fold->red_of[topo->parent[l]];          // anchor of the parent: nearest movable ancestor, or the root
            rt.axis[j] = topo->axis[l];
            rt.dof[j] = topo->dof[l];
        } else {
            fold->red_of[l] = fold->red_of[topo->parent[l]];
            ++n_fixed;
        }
    }
    fold->n_red = n_red;
    int e = 0;
    for (int j = 0; j < n_red; ++j) {
        fold->carry_start[j] = (int8_t)e;
        if (j == 0) continue;                              // links fixed to the root load no joint
        for (int l = 1; l < N; ++l)
            if (topo->axis[l] == 0 && fold->red_of[l] == j) fold->carry[e++] = (int8_t)l;
    }
    fold->carry_start[n_red] = (int8_t)e;
    rt.n_links = n_red;
    rt.n_dofs = topo->n_dofs;
    // staging scratch (raw table + poses, 40 floats per original link) lives in the per-link state region (8 floats per
    // reduced link and configuration) of the smallest tile any of the tree kernels uses (32 configurations)
    *foldable = n_fixed > 0 && n_red > 1 && N * 40 <= n_red * 8 * 32;
    return build_tree_program(&rt, red);
}

const CachedPrograms* cached_programs(const drmb200_topology_t* topo, int* rc_out) {
    static thread_local CachedPrograms cache[2] = {};
    static thread_local int next = 0;
    *rc_out = DRMB200_OK;
    if (topo == nullptr) { set_error("topology is null"); *rc_out = DRMB200_EINVAL; return nullptr; }
    for (auto& c : cache) if (c.valid && memcmp(&c.topo, topo, sizeof(*topo)) == 0) return &c;
    CachedPrograms& c = cache[next];
    c.valid = false;
    *rc_out = build_tree_program(topo, &c.full);
    if (*rc_out != DRMB200_OK) return nullptr;
    *rc_out = build_fold(topo, &c.red, &c.fold, &c.foldable);
    if (*rc_out != DRMB200_OK) return nullptr;
    c.topo = *topo; c.valid = true;
    next ^= 1;
    return &c;
}

int select_fold(const drmb200_topology_t* topo, bool prefolded, FoldChoice* out) {
    int rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);
    if (cp == nullptr) return rc;
    if (prefolded && !cp->foldable) { set_error("this topology has no link behind a fixed joint to fold"); return DRMB200_EINVAL; }
    out->folded = prefolded || (cp->foldable && get_option(11) != 0);      // "rnea_fold"
    out->prog = out->folded ? &cp->red : &cp->full;
    out->fold = cp->fold;
    if (!out->folded) out->fold.n_red = 0;
    if (prefolded) out->fold.n_full = 0;
    return DRMB200_OK;
}

// The folded canonical table of a link table, once, for callers whose table does not change between launches (constant
// models): folding it while staging costs every CTA a noticeable share of the inverse-dynamics kernel, a plain copy of
// n_red x 28 floats costs nothing.  Output: [n_red, 28] canonical rows (row 0 unused).
__global__ void __launch_bounds__(64)
fold_table_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold,
                  const float* __restrict__ table, float* __restrict__ folded) {
    extern __shared__ __align__(16) float fsm[];
    float* s_tab = fsm;                                                    // [n_red][28]
    float* scratch = fsm + fold.n_red * DRMB200_TABLE_STRIDE;              // [n_full][40]
    for (int i = threadIdx.x; i < DRMB200_TABLE_STRIDE; i += 64) s_tab[i] = 0.f;
    stage_folded_table(s_tab, scratch, table, fold, prog, 64);
    for (int i = threadIdx.x; i < fold.n_red * DRMB200_TABLE_STRIDE; i += 64) folded[i] = s_tab[i];
}

int64_t folded_table_rows(const drmb200_topology_t* topo) {
    FoldChoice fc;
    const int rc = select_fold(topo, false, &fc);
    if (rc != DRMB200_OK) return rc;
    return fc.folded ? fc.fold.n_red : 0;
}

int fold_table_device(const drmb200_topology_t* topo, const float* table, float* folded, cudaStream_t stream) {
    int rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);
    if (cp == nullptr) return rc;
    if (!cp->foldable) { set_error("this topology has no link behind a fixed joint to fold (drmb200_folded_table_rows() == 0)"); return DRMB200_EINVAL; }
    if (table == nullptr || folded == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    const size_t smem = (size_t)(cp->fold.n_red * DRMB200_TABLE_STRIDE + cp->fold.n_full * 40) * sizeof(float);
    return launch_kernel<fold_table_kernel>(1, 64, smem, stream, false, "fold_table", cp->red, cp->fold, table, folded);
}

// Tile: 128 amortises the table staging (heavier since it folds the fixed links) over twice the configurations (chosen by a
// Panda sweep before the H100 port; not re-measured on the H100); 64 only for batches that would leave SMs without a CTA,
// and for models whose 128-row footprint is larger than RNEA_128_MAX_BYTES.  "rnea_tile" 64 / 128 forces one (256 lost that
// sweep too).
constexpr size_t RNEA_128_MAX_BYTES = 110 * 1024;

static int rnea_tile(const TreeProgram& prog, int64_t batch) {
    int tile = (batch < 32768) ? 64 : 128;
    if (get_option(12) == 64 || get_option(12) == 128) tile = get_option(12);
    if ((size_t)RneaSmemLayout(128, prog.n_dofs, prog.n_links, prog.n_slots).total_floats * sizeof(float) > RNEA_128_MAX_BYTES) tile = 64;
    return tile;
}

template <bool FOLD>
static int launch_rnea_tile(int tile, const TreeProgram& prog, const FoldProgram& fold, const RneaArgs& args, cudaStream_t stream) {
    const bool packed = get_option(4) != 0;             // "rnea_packed": f32x2 pair arithmetic (default) vs scalar, for A/B runs
    if (tile == 64) return packed ? launch_rnea<64, true, false, FOLD>(prog, fold, args, stream) : launch_rnea<64, false, false, FOLD>(prog, fold, args, stream);
    return packed ? launch_rnea<128, true, false, FOLD>(prog, fold, args, stream) : launch_rnea<128, false, false, FOLD>(prog, fold, args, stream);
}

// prefolded: `table` holds the rows of drmb200_fold_link_table
static int inverse_dynamics_impl(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                 const float* qdd, int64_t batch, uint32_t flags, float* tau, cudaStream_t stream, bool prefolded) {
    FoldChoice fc;
    const int rc = select_fold(topo, prefolded, &fc);
    if (rc != DRMB200_OK) return rc;
    const TreeProgram& prog = *fc.prog;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || qdd == nullptr || tau == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    RneaArgs args;
    args.table = table; args.q = q; args.qd = qd; args.qdd = qdd; args.tau = tau; args.batch = batch; args.flags = flags;
    args.vels = args.accs = args.forces = nullptr;
    args.aligned = aligned16(q, qd, qdd, tau);
    const int tile = rnea_tile(prog, batch);
    return fc.folded ? launch_rnea_tile<true>(tile, prog, fc.fold, args, stream) : launch_rnea_tile<false>(tile, prog, fc.fold, args, stream);
}

int inverse_dynamics_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                            const float* qdd, int64_t batch, uint32_t flags, float* tau, cudaStream_t stream) {
    return inverse_dynamics_impl(topo, table, q, qd, qdd, batch, flags, tau, stream, false);
}
int inverse_dynamics_prefolded_device(const drmb200_topology_t* topo, const float* folded, const float* q, const float* qd,
                                      const float* qdd, int64_t batch, uint32_t flags, float* tau, cudaStream_t stream) {
    return inverse_dynamics_impl(topo, folded, q, qd, qdd, batch, flags, tau, stream, true);
}

// inverse dynamics + the per-link state of the reference's bodies (vel, acc, force), see rnea_kernel<.., DUMP>
int dynamic_state_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                         const float* qdd, int64_t batch, uint32_t flags, float* tau, float* vels, float* accs,
                         float* forces, cudaStream_t stream) {
    int rc;
    const CachedPrograms* cp = cached_programs(topo, &rc);
    if (cp == nullptr) return rc;
    const TreeProgram* prog = &cp->full;                  // every link reports its state: no folding here
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || qdd == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    RneaArgs args;
    args.table = table; args.q = q; args.qd = qd; args.qdd = qdd; args.tau = tau; args.batch = batch; args.flags = flags;
    args.vels = vels; args.accs = accs; args.forces = forces;
    args.aligned = aligned16(q, qd, qdd, tau);
    return launch_rnea<64, true, true, false>(*prog, cp->fold, args, stream);
}

}  // namespace drm
