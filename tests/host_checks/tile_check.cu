// Host-side check (no GPU needed): the tile each of four kernels picks for a model, from the real program builders, the real
// fold selection and the real tile choosers of the kernels' host code:
//
//   dynamics_derivatives.cu     select_fold -> deriv_tile (DerivSmemLayout, TC = 128 / n lowered to fit)
//   inverse_kinematics.cu       build_path_program -> ik_tile (IkSmemLayout, T = 64 or 32)
//   inverse_kinematics_multi.cu build_union_program -> ikm_tile (IkmSmemLayout, T = 64, 32, ..., 1)
//   operational_space.cu        build_union_program + cached_programs (full tree) -> osd_tile (OsdSmemLayout, T = 64, ..., 1)
//
// The static shared bytes the kernels add are the `-Xptxas -v` values (the GPU tests read them back from the device).
// tests/test_tile_choice.py compares every line with the Python mirrors of tests/tile_mirrors.py.
//
// stdin: one case per line: N, N-1 parents, N-1 axis codes (0 = fixed), n_ee, n_ee link indices.
// stdout: one line per case, eleven "tile bytes" pairs: derivatives ID / FD with folding, ID / FD without folding (the
// "rnea_fold" = 0 program), ID / FD on prefolded rows, IK of the first link (pose; position mode uses the same layout),
// multi-link IK pose / position, operational-space pose / position.  tile = 0: refused for its shared memory (bytes is what
// the ELIMIT message names); tile = rc < 0, bytes = 0: the program builder refused the model
// (-1000: no movable joint, nothing to launch).
#include <cstdio>
#include <vector>
#include "rnea.cu"
#include "fk_jacobian.cu"
#include "fk_tree.cu"
#include "dynamics_derivatives.cu"
#include "inverse_kinematics.cu"
#include "inverse_kinematics_multi.cu"
#include "operational_space.cu"

static int g_rnea_fold = 0;

namespace drm {
void set_error(const char*, ...) {}
void count_launch(int) {}
int get_option(int which) { return which == 11 ? g_rnea_fold : 0; }       // "rnea_fold"
}  // namespace drm

using namespace drm;

static constexpr size_t STATIC_DERIV = 128, STATIC_IK = 0, STATIC_IKM = 0, STATIC_OSD = 128;

// a choice as the ELIMIT message states it: dynamic + static bytes, tile 0 when refused
static void put(TileChoice c, size_t stat) {
    const size_t b = c.bytes + stat;
    std::printf(" %d %zu", b > SMEM_CTA_MAX ? 0 : c.tile, b);
}
static void put(int tile, size_t bytes) { std::printf(" %d %zu", tile, bytes); }

static void deriv(const drmb200_topology_t* topo, bool fold, bool prefolded, bool fd) {
    g_rnea_fold = fold ? 1 : 0;
    FoldChoice fc;
    const int rc = select_fold(topo, prefolded, &fc);
    if (rc != DRMB200_OK) { put(rc, 0); return; }
    if (fc.prog->n_dofs == 0) { put(-1000, 0); return; }        // nothing to launch
    const bool staging_fold = fc.fold.n_red > 0 && fc.fold.n_full > 0;
    put(deriv_tile(*fc.prog, staging_fold ? fc.fold.n_full : 0, fd, STATIC_DERIV), STATIC_DERIV);
}

int main() {
    int N, count = 0;
    while (std::scanf("%d", &N) == 1) {
        std::vector<int> par(N, -1), axis(N, 0);
        for (int i = 1; i < N; ++i) if (std::scanf("%d", &par[i]) != 1) return 2;
        for (int i = 1; i < N; ++i) if (std::scanf("%d", &axis[i]) != 1) return 2;
        int n_ee = 0;
        if (std::scanf("%d", &n_ee) != 1 || n_ee < 1 || n_ee > MT_MAX_EE) return 2;
        int32_t links[MT_MAX_EE];
        for (int e = 0; e < n_ee; ++e) if (std::scanf("%d", &links[e]) != 1) return 2;
        drmb200_topology_t topo;
        std::memset(&topo, 0, sizeof(topo));
        topo.n_links = N;
        topo.parent[0] = -1;
        int n_dofs = 0;
        for (int i = 1; i < N; ++i) {
            topo.parent[i] = (int8_t)par[i];
            topo.axis[i] = (int8_t)axis[i];
            topo.dof[i] = axis[i] != 0 ? (int8_t)n_dofs++ : (int8_t)-1;
        }
        topo.n_dofs = n_dofs;

        for (int k = 0; k < 6; ++k) deriv(&topo, k < 2, k >= 4, k & 1);

        PathProgram path;
        int rc = build_path_program(&topo, links[0], &path);
        if (rc != DRMB200_OK) put(rc, 0);
        else put(ik_tile(path, STATIC_IK), STATIC_IK);

        UnionProgram P;
        rc = build_union_program(&topo, n_ee, links, &P);
        for (int pose = 1; pose >= 0; --pose) {
            if (rc != DRMB200_OK) put(rc, 0);
            else put(ikm_tile(P, pose, STATIC_IKM), STATIC_IKM);
        }
        int rc_cp = 0;
        const CachedPrograms* cp = cached_programs(&topo, &rc_cp);
        for (int pose = 1; pose >= 0; --pose) {
            if (rc != DRMB200_OK || cp == nullptr) put(rc != DRMB200_OK ? rc : rc_cp, 0);
            else put(osd_tile(cp->full, P, (pose ? 6 : 3) * n_ee, STATIC_OSD), STATIC_OSD);
        }
        std::printf("\n");
        ++count;
    }
    std::fprintf(stderr, "checked %d cases\n", count);
    return 0;
}
