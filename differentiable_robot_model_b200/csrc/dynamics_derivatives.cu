// dynamics_derivatives.cu -- batched Jacobians of the dynamics (sm_90a):
//   inverse dynamics   dtau/dq, dtau/dqd                    [B, n, n]   (tangent RNEA)
//   forward dynamics   dqdd/dq, dqdd/dqd, dqdd/df           [B, n, n]   (tangent articulated-body algorithm, aba_tangent.cuh)
// out[b, i, j] = d y_i / d x_j of exactly what drmb200_inverse_dynamics / drmb200_forward_dynamics evaluate, for any
// link table (non-symmetric inertia matrices included: the forward-dynamics Jacobians differentiate the reference's
// articulated-body arithmetic itself, which is not the inverse of its RNEA when an inertia is non-symmetric).
//
// Forward mode, one THREAD per (configuration, column j).  The thread carries the primal recursion and two tangent lanes,
// dq = e_j and dqd = e_j (forward dynamics: a third, df = e_j), through every link step in the canonical +z joint frames of
// drm_common.cuh.  A joint's own angle enters only its own link step, through the rotation derivatives
//   d(M^T x)/dq = (M^T x) x e_z,   d(M x)/dq = M (e_z x x)          (M = F~ Rz(q))
// Inverse dynamics, link i (closed form of rnea.cu, tangents marked d):
//   dw  = E dw_p + [own] Ew_p x e_z + (0,0,dqd)          dv = E (dv_p + dw_p x r) + [own] E(v_p + w_p x r) x e_z
//   dal = E dal_p + [own] E al_p x e_z + dw x (0,0,qd) + w x (0,0,dqd)
//   da  = E (da_p + dal_p x r) + [own] E(a_p + al_p x r) x e_z + dv x (0,0,qd) + v x (0,0,dqd)
//   df, dn: the bilinear wrench terms differentiated; the leaves -> root sum through M with [own] M (e_z x .)
//   dtau_k = dn_k.z + d_k dqd_k
//
// Mapping: a CTA owns TC configurations x all n columns (TC * n threads), so its output is one contiguous range of each
// matrix ([TC, n, n]); it is staged in shared memory and leaves with one TMA bulk copy per matrix (cooperative copies for
// ragged or unaligned tiles).  Per link and thread the kernel keeps the primal and tangent state it needs on the way back
// in shared memory, slot-major with stride TC * n; branch points use the tree program's slots like rnea.cu / aba.cu.
// TC is the largest count (<= 128 / n) whose footprint stays under ~113 KB (two CTAs per SM); a model that needs more than
// 227 KB per CTA even at TC = 1 is refused with DRMB200_ELIMIT (about 50 DoF for inverse dynamics and 38 for forward
// dynamics on a serial chain, fewer for trees with live branch points).
//
// Algorithmic HBM bytes per configuration: 12n in, 8n^2 (ID) / 12n^2 (FD) out.  Every thread repeats its configuration's
// primal recursion (n times per configuration): the arithmetic, not the bytes, bounds the kernel.
#include "aba_tangent.cuh"
#include "launch.cuh"

namespace drm {

constexpr int IDD_LINK = 20;     // per link: f, n, cs, sn, (df, dn) lane 0, (df, dn) lane 1
constexpr int IDD_SLOT = 36;     // per branch slot: w, v, al, a and their two tangents

struct DerivArgs {
    const float* __restrict__ table;
    const float* __restrict__ q;
    const float* __restrict__ qd;
    const float* __restrict__ x3;        // qdd (inverse dynamics) or f (forward dynamics)
    float* out[3];                       // ID: dtau_dq, dtau_dqd; FD: dqdd_dq, dqdd_dqd, dqdd_df; each may be null
    int64_t batch;
    uint32_t flags;
    int32_t aligned;
    int32_t tc;                          // configurations per CTA
};

struct DerivSmemLayout {
    int in[3], out[3], table, link, slots, total_floats;
    __host__ __device__ static int up4(int x) { return (x + 3) & ~3; }       // 16-byte aligned regions
    __host__ __device__ DerivSmemLayout(int tc, int n, int n_links, int n_slots, int fold_scratch_links, bool fd) {
        const int S = tc * n;
        int o = 0;
        for (int k = 0; k < 3; ++k) { in[k] = o; o += up4(S); }
        for (int k = 0; k < 3; ++k) { out[k] = o; if (k < (fd ? 3 : 2)) o += up4(S * n); }
        table = o; o += n_links * DRMB200_TABLE_STRIDE;
        link = o;
        const int lf = n_links * (fd ? FDD_LINK : IDD_LINK) * S, scratch = fold_scratch_links * 40;   // folding scratch (rnea.cu)
        o += up4(lf > scratch ? lf : scratch);
        slots = o; o += n_slots * (fd ? FDD_SLOT : IDD_SLOT) * S;
        total_floats = o;
    }
};

// Inverse dynamics: one thread, configuration rows qrow / qdrow / qddrow, column j; outputs element (c, j) at o[c * n].
__device__ __forceinline__ void rnea_tangent_body(const TreeProgram& prog, const float* s_tab, const float* qrow,
                                                  const float* qdrow, const float* qddrow, int j, int n, float* o_q,
                                                  float* o_qd, float* lk0, float* sl0, int S, uint32_t flags) {
    const int N = prog.n_links;
    const float g = (flags & DRMB200_GRAVITY) ? 9.81f : 0.f;      // robot_model.py:347
    const bool damp = (flags & DRMB200_DAMPING) != 0;
    const V3 zero = v3(0.f, 0.f, 0.f);

    // ---- pass 1: root -> leaves, motion state, body wrench and their tangents -----------------------------------------
    V3 w = zero, v = zero, al = zero, a = zero;
    V3 tw0 = zero, tv0 = zero, tal0 = zero, ta0 = zero, tw1 = zero, tv1 = zero, tal1 = zero, ta1 = zero;
    for (int i = 1; i < N; ++i) {
        const LinkRow C = load_row(s_tab + i * DRMB200_TABLE_STRIDE);
        const int src = prog.psrc[i];
        V3 wp, vp, alp, ap, twp0, tvp0, talp0, tap0, twp1, tvp1, talp1, tap1;
        if (src == 0) {
            wp = w; vp = v; alp = al; ap = a;
            twp0 = tw0; tvp0 = tv0; talp0 = tal0; tap0 = ta0; twp1 = tw1; tvp1 = tv1; talp1 = tal1; tap1 = ta1;
        } else if (src < 0) {
            wp = vp = alp = twp0 = tvp0 = talp0 = tap0 = twp1 = tvp1 = talp1 = tap1 = zero;
            ap = v3(0.f, 0.f, g);
        } else {
            const float* sl = sl0 + (src - 1) * IDD_SLOT * S;
            wp = ldv(sl, S); vp = ldv(sl + 3 * S, S); alp = ldv(sl + 6 * S, S); ap = ldv(sl + 9 * S, S);
            twp0 = ldv(sl + 12 * S, S); tvp0 = ldv(sl + 15 * S, S); talp0 = ldv(sl + 18 * S, S); tap0 = ldv(sl + 21 * S, S);
            twp1 = ldv(sl + 24 * S, S); tvp1 = ldv(sl + 27 * S, S); talp1 = ldv(sl + 30 * S, S); tap1 = ldv(sl + 33 * S, S);
        }
        M3 M = C.F;
        const int c = prog.dof[i];
        float cs = 1.f, sn = 0.f, qd_k = 0.f, qdd_k = 0.f;
        if (c >= 0) {
            qd_k = qdrow[c];
            qdd_k = qddrow[c];
            sincos_pi2(qrow[c], sn, cs);
            rotate_z(M, cs, sn);
        }
        const bool own = (c == j);
        const float dqd1 = own ? 1.f : 0.f;
        const V3 Ew = mulT(M, wp), Ev = mulT(M, cross_add(wp, C.r, vp));
        const V3 Eal = mulT(M, alp), Ea = mulT(M, cross_add(alp, C.r, ap));
        w = Ew; w.z += qd_k;
        v = Ev;
        al = Eal + cross_z(w, qd_k); al.z += qdd_k;
        a = Ea + cross_z(v, qd_k);
        // lane 0: dq_j
        tw0 = mulT(M, twp0); tv0 = mulT(M, cross_add(twp0, C.r, tvp0));
        tal0 = mulT(M, talp0); ta0 = mulT(M, cross_add(talp0, C.r, tap0));
        if (own) { tw0 = tw0 + zc1(Ew); tv0 = tv0 + zc1(Ev); tal0 = tal0 + zc1(Eal); ta0 = ta0 + zc1(Ea); }
        tal0 = tal0 + cross_z(tw0, qd_k);
        ta0 = ta0 + cross_z(tv0, qd_k);
        // lane 1: dqd_j
        tw1 = mulT(M, twp1); tw1.z += dqd1;
        tv1 = mulT(M, cross_add(twp1, C.r, tvp1));
        tal1 = mulT(M, talp1) + cross_z(tw1, qd_k) + cross_z(w, dqd1);
        ta1 = mulT(M, cross_add(talp1, C.r, tap1)) + cross_z(tv1, qd_k) + cross_z(v, dqd1);
        // body wrench (rnea.cu) and its tangents
        const V3 hl_v = C.m * v - cross(C.mc, w), ha_v = mul_add(C.Io, w, cross(C.mc, v));
        const V3 hl_a = C.m * a - cross(C.mc, al), ha_a = mul_add(C.Io, al, cross(C.mc, a));
        const V3 f = cross_add(w, hl_v, hl_a);
        const V3 nn = cross_add(w, ha_v, cross_add(v, hl_v, ha_a));
        auto dwrench = [&](V3 tw, V3 tv, V3 tal, V3 ta, V3& df, V3& dn) {
            const V3 dhl_v = C.m * tv - cross(C.mc, tw), dha_v = mul_add(C.Io, tw, cross(C.mc, tv));
            const V3 dhl_a = C.m * ta - cross(C.mc, tal), dha_a = mul_add(C.Io, tal, cross(C.mc, ta));
            df = dhl_a + cross(tw, hl_v) + cross(w, dhl_v);
            dn = dha_a + cross(tw, ha_v) + cross(w, dha_v) + cross(tv, hl_v) + cross(v, dhl_v);
        };
        V3 df0, dn0, df1, dn1;
        dwrench(tw0, tv0, tal0, ta0, df0, dn0);
        dwrench(tw1, tv1, tal1, ta1, df1, dn1);
        float* lk = lk0 + i * IDD_LINK * S;
        stv(lk, S, f); stv(lk + 3 * S, S, nn); lk[6 * S] = cs; lk[7 * S] = sn;
        stv(lk + 8 * S, S, df0); stv(lk + 11 * S, S, dn0); stv(lk + 14 * S, S, df1); stv(lk + 17 * S, S, dn1);
        const int sv = prog.save[i];
        if (sv >= 0) {
            float* sl = sl0 + sv * IDD_SLOT * S;
            stv(sl, S, w); stv(sl + 3 * S, S, v); stv(sl + 6 * S, S, al); stv(sl + 9 * S, S, a);
            stv(sl + 12 * S, S, tw0); stv(sl + 15 * S, S, tv0); stv(sl + 18 * S, S, tal0); stv(sl + 21 * S, S, ta0);
            stv(sl + 24 * S, S, tw1); stv(sl + 27 * S, S, tv1); stv(sl + 30 * S, S, tal1); stv(sl + 33 * S, S, ta1);
        }
    }

    // ---- pass 2: leaves -> root, wrenches (children accumulate into their parent's link entry) and joint torques ------
    for (int i = N - 1; i >= 1; --i) {
        const float* lk = lk0 + i * IDD_LINK * S;
        const int c = prog.dof[i];
        const float* row = s_tab + i * DRMB200_TABLE_STRIDE;
        if (c >= 0) {
            if (o_q) o_q[c * n] = lk[13 * S];                                          // dn.z, lane 0
            if (o_qd) o_qd[c * n] = (damp && c == j) ? lk[19 * S] + row[25] : lk[19 * S];
        }
        const int p = prog.parent[i];
        if (p > 0) {
            M3 F; V3 r;
            load_Fr(row, F, r);
            const float cs = lk[6 * S], sn = lk[7 * S];
            const V3 Rf = rotz(ldv(lk, S), cs, sn), Rn = rotz(ldv(lk + 3 * S, S), cs, sn);
            V3 Rdf0 = rotz(ldv(lk + 8 * S, S), cs, sn), Rdn0 = rotz(ldv(lk + 11 * S, S), cs, sn);
            const V3 Rdf1 = rotz(ldv(lk + 14 * S, S), cs, sn), Rdn1 = rotz(ldv(lk + 17 * S, S), cs, sn);
            if (c == j) { Rdf0 = Rdf0 + ezx(Rf); Rdn0 = Rdn0 + ezx(Rn); }
            const V3 fp = mul(F, Rf), df0 = mul(F, Rdf0), df1 = mul(F, Rdf1);
            const V3 np = cross_add(r, fp, mul(F, Rn)), dn0 = cross_add(r, df0, mul(F, Rdn0)), dn1 = cross_add(r, df1, mul(F, Rdn1));
            float* pk = lk0 + p * IDD_LINK * S;
            stv(pk, S, ldv(pk, S) + fp); stv(pk + 3 * S, S, ldv(pk + 3 * S, S) + np);
            stv(pk + 8 * S, S, ldv(pk + 8 * S, S) + df0); stv(pk + 11 * S, S, ldv(pk + 11 * S, S) + dn0);
            stv(pk + 14 * S, S, ldv(pk + 14 * S, S) + df1); stv(pk + 17 * S, S, ldv(pk + 17 * S, S) + dn1);
        }
    }
}

template <bool FD>
__global__ void dynamics_derivatives_kernel(const __grid_constant__ TreeProgram prog, const __grid_constant__ FoldProgram fold,
                                            const DerivArgs args) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;

    const int n = prog.n_dofs;
    const int N = prog.n_links;
    const int TC = args.tc, S = TC * n;
    const bool staging_fold = fold.n_red > 0 && fold.n_full > 0;
    const DerivSmemLayout L(TC, n, N, prog.n_slots, staging_fold ? fold.n_full : 0, FD);
    float* s_in0 = smem + L.in[0];
    float* s_in1 = smem + L.in[1];
    float* s_in2 = smem + L.in[2];
    float* s_tab = smem + L.table;
    float* s_link = smem + L.link;
    float* s_slot = smem + L.slots;

    const int tid = threadIdx.x;
    const int64_t tile_start = (int64_t)blockIdx.x * TC;
    const int valid = (int)min((int64_t)TC, args.batch - tile_start);
    // TC * n need not be a multiple of 4: each tile checks the 16-byte alignment of its own global ranges
    const bool vec_in = args.aligned && ((tile_start * n) & 3) == 0;
    const bool bulk_in = vec_in && ((valid * n) & 3) == 0;
    const int64_t out_off = tile_start * n * n;
    const int out_floats = valid * n * n;
    const bool vec_out = args.aligned && (out_off & 3) == 0;
    const bool bulk_out = vec_out && (out_floats & 3) == 0;

    if (bulk_in) {
        if (tid == 0) {
            mbar_init(&mbar, 1);
            fence_mbar_init();
            const uint32_t bytes = (uint32_t)valid * n * 4u;
            mbar_arrive_expect_tx(&mbar, 3u * bytes);
            bulk_g2s(s_in0, args.q + tile_start * n, bytes, &mbar);
            bulk_g2s(s_in1, args.qd + tile_start * n, bytes, &mbar);
            bulk_g2s(s_in2, args.x3 + tile_start * n, bytes, &mbar);
        }
    } else {
        coop_copy(s_in0, args.q + tile_start * n, valid * n, vec_in);
        coop_copy(s_in1, args.qd + tile_start * n, valid * n, vec_in);
        coop_copy(s_in2, args.x3 + tile_start * n, valid * n, vec_in);
    }
    if (fold.n_red > 0 && fold.n_full == 0) {                // rows folded beforehand (drmb200_fold_link_table)
        for (int i = tid; i < N * DRMB200_TABLE_STRIDE; i += blockDim.x) s_tab[i] = __ldg(args.table + i);
    } else if (staging_fold) {
        stage_folded_table(s_tab, s_link, args.table, fold, prog, blockDim.x);
    } else {
        stage_canonical_table(s_tab, args.table, prog, blockDim.x);
    }
    __syncthreads();
    if (bulk_in) mbar_wait(&mbar, 0);

    const int lc = tid / n, j = tid - lc * n;
    if (lc < valid) {
        const int row = lc * n;
        float* o0 = args.out[0] ? smem + L.out[0] + lc * n * n + j : nullptr;
        float* o1 = args.out[1] ? smem + L.out[1] + lc * n * n + j : nullptr;
        if (FD) {
            float* o2 = args.out[2] ? smem + L.out[2] + lc * n * n + j : nullptr;
            aba_tangent_body(prog, s_tab, s_in0 + row, s_in1 + row, s_in2 + row, j, n, o0, o1, o2, s_link + tid, s_slot + tid, S,
                             args.flags);
        } else {
            rnea_tangent_body(prog, s_tab, s_in0 + row, s_in1 + row, s_in2 + row, j, n, o0, o1, s_link + tid, s_slot + tid, S,
                              args.flags);
        }
    }

    constexpr int N_OUT = FD ? 3 : 2;
    if (bulk_out) {
        fence_proxy_async();
        __syncthreads();
        if (tid == 0) {
            for (int k = 0; k < N_OUT; ++k)
                if (args.out[k]) bulk_s2g(args.out[k] + out_off, smem + L.out[k], (uint32_t)out_floats * 4u);
            bulk_commit();
            bulk_wait_read<0>();
        }
    } else {
        __syncthreads();
        for (int k = 0; k < N_OUT; ++k)
            if (args.out[k]) coop_copy(args.out[k] + out_off, smem + L.out[k], out_floats, vec_out);
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// ~128 threads per CTA: TC = 128 / n configurations, fewer while the footprint would leave a single CTA per SM.  fold_full:
// the full link count when the kernel folds the table while staging it (folding scratch), else 0.
static TileChoice deriv_tile(const TreeProgram& prog, int fold_full, bool fd, size_t static_bytes) {
    const int n = prog.n_dofs;
    return tile_count_down(n >= 128 ? 1 : 128 / n, [&](int tc) {
        return (size_t)DerivSmemLayout(tc, n, prog.n_links, prog.n_slots, fold_full, fd).total_floats * sizeof(float);
    }, static_bytes);
}

template <bool FD>
static int derivatives_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd, const float* x3,
                              int64_t batch, uint32_t flags, float* o0, float* o1, float* o2, cudaStream_t stream, bool prefolded) {
    FoldChoice fc;
    int rc = select_fold(topo, prefolded, &fc);
    if (rc != DRMB200_OK) return rc;
    const TreeProgram& prog = *fc.prog;
    if (batch < 0) { set_error("batch=%lld < 0", (long long)batch); return DRMB200_EINVAL; }
    if (batch == 0 || prog.n_dofs == 0 || (o0 == nullptr && o1 == nullptr && o2 == nullptr)) return DRMB200_OK;
    if (table == nullptr || q == nullptr || qd == nullptr || x3 == nullptr) { set_error("null pointer argument"); return DRMB200_EINVAL; }
    DerivArgs args;
    args.table = table; args.q = q; args.qd = qd; args.x3 = x3;
    args.out[0] = o0; args.out[1] = o1; args.out[2] = o2;
    args.batch = batch; args.flags = flags & (DRMB200_GRAVITY | DRMB200_DAMPING);
    args.aligned = aligned16(q, qd, x3, o0, o1, o2);

    constexpr auto kern = dynamics_derivatives_kernel<FD>;
    size_t static_bytes;
    rc = static_smem_bytes<kern>(&static_bytes);
    if (rc != DRMB200_OK) return rc;
    const bool staging_fold = fc.fold.n_red > 0 && fc.fold.n_full > 0;
    const TileChoice c = deriv_tile(prog, staging_fold ? fc.fold.n_full : 0, FD, static_bytes);
    if (c.bytes + static_bytes > SMEM_CTA_MAX) {
        set_error("model needs %zu B of shared memory per CTA (> 227 KB) for its %s derivatives", c.bytes + static_bytes,
                  FD ? "forward-dynamics" : "inverse-dynamics");
        return DRMB200_ELIMIT;
    }
    args.tc = c.tile;
    return launch_kernel<kern>((batch + c.tile - 1) / c.tile, c.tile * prog.n_dofs, c.bytes, stream, false, "dynamics derivatives", prog,
                               fc.fold, args);
}

int inverse_dynamics_derivatives_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                        const float* qdd, int64_t batch, uint32_t flags, float* dtau_dq, float* dtau_dqd,
                                        cudaStream_t stream, bool prefolded) {
    return derivatives_device<false>(topo, table, q, qd, qdd, batch, flags, dtau_dq, dtau_dqd, nullptr, stream, prefolded);
}

int forward_dynamics_derivatives_device(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                                        const float* f, int64_t batch, uint32_t flags, float* dqdd_dq, float* dqdd_dqd,
                                        float* dqdd_df, cudaStream_t stream, bool prefolded) {
    return derivatives_device<true>(topo, table, q, qd, f, batch, flags, dqdd_dq, dqdd_dqd, dqdd_df, stream, prefolded);
}

}  // namespace drm
