// Host-side check (no GPU needed): the tile each of four kernels picks for a model, from the real program builders and the
// real __host__ __device__ shared-memory layout structs.
//
//   dynamics_derivatives.cu     cached_programs -> tree / fold program -> DerivSmemLayout, TC = 128 / n lowered to fit
//   inverse_kinematics.cu       build_path_program -> IkSmemLayout, T = 64 or 32
//   inverse_kinematics_multi.cu build_multi_program -> IkmSmemLayout, T = 64, 32, ..., 1
//   operational_space.cu        build_multi_program + cached_programs (full tree) -> OsdSmemLayout, T = 64, 32, ..., 1
//
// The choosers live inside the launch functions, next to the launch, so the loops below restate them over the real
// structs; the static shared bytes the kernels add are the `-Xptxas -v` values (the GPU tests read them back from the
// device).  tests/test_tile_choice.py compares every line with the Python mirrors of tests/tile_mirrors.py.
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

namespace drm {
void set_error(const char*, ...) {}
void count_launch(int) {}
int get_option(int) { return 0; }
}  // namespace drm

using namespace drm;

static constexpr size_t TWO_CTAS = 113 * 1024, CAP = 227 * 1024;
static constexpr size_t STATIC_DERIV = 128, STATIC_IK = 0, STATIC_IKM = 0, STATIC_OSD = 128;

static void put(int tile, size_t bytes) { std::printf(" %d %zu", tile, bytes); }

static void deriv(const CachedPrograms* cp, bool fold, bool prefolded, bool fd) {
    const bool folded = prefolded || (cp->foldable && fold);
    if (prefolded && !cp->foldable) { put(DRMB200_EINVAL, 0); return; }
    const TreeProgram& prog = folded ? cp->red : cp->full;
    const int fold_full = (folded && !prefolded) ? cp->fold.n_full : 0;
    const int n = prog.n_dofs;
    if (n == 0) { put(-1000, 0); return; }          // nothing to launch
    auto bytes_of = [&](int tc) {
        return (size_t)DerivSmemLayout(tc, n, prog.n_links, prog.n_slots, fold_full, fd).total_floats * 4 + STATIC_DERIV;
    };
    int tc = n >= 128 ? 1 : 128 / n;
    while (tc > 1 && bytes_of(tc) > TWO_CTAS) --tc;
    put(bytes_of(tc) > CAP ? 0 : tc, bytes_of(tc));
}

template <typename F>
static void ladder(F floats_of, size_t stat) {
    int T = 64;
    while (T > 1 && (size_t)floats_of(T) * 4 + stat > TWO_CTAS) T >>= 1;
    const size_t b = (size_t)floats_of(T) * 4 + stat;
    put(b > CAP ? 0 : T, b);
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

        int rc_cp = 0, rc = 0;
        const CachedPrograms* cp = cached_programs(&topo, &rc_cp);
        for (int k = 0; k < 6; ++k) {
            if (cp == nullptr) { put(rc_cp, 0); continue; }
            deriv(cp, k < 2, k >= 4, k & 1);
        }

        PathProgram path;
        rc = build_path_program(&topo, links[0], &path);
        if (rc != DRMB200_OK) put(rc, 0);
        else {
            auto bytes_of = [&](int T) { return (size_t)IkSmemLayout(T, path.n_dofs, path.len).total_floats * 4 + STATIC_IK; };
            const int T = bytes_of(64) <= TWO_CTAS ? 64 : 32;
            put(bytes_of(T) > CAP ? 0 : T, bytes_of(T));
        }

        MultiProgram W;
        rc = build_multi_program(&topo, n_ee, links, &W);
        int n_u = 0;
        if (rc == DRMB200_OK)
            for (int k = 0; k < W.n_steps; ++k) n_u += W.dof[k] >= 0;
        for (int pose = 1; pose >= 0; --pose) {
            if (rc != DRMB200_OK) { put(rc, 0); continue; }
            ladder([&](int T) { return IkmSmemLayout(T, W.n_dofs, n_u, n_ee, pose, W.n_steps, W.n_jslots, W.n_state_slots).total_floats; },
                   STATIC_IKM);
        }
        for (int pose = 1; pose >= 0; --pose) {
            if (rc != DRMB200_OK || cp == nullptr) { put(rc != DRMB200_OK ? rc : rc_cp, 0); continue; }
            OsdProgram P;
            P.walk = W;
            P.n_u = n_u;
            const int M = (pose ? 6 : 3) * n_ee;
            ladder([&](int T) { return OsdSmemLayout(T, cp->full, P, M).total_floats; }, STATIC_OSD);
        }
        std::printf("\n");
        ++count;
    }
    std::fprintf(stderr, "checked %d cases\n", count);
    return 0;
}
