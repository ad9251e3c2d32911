// Host-side check (no GPU needed): the tree programs (build_tree_program) and fold programs (build_fold) of arbitrary
// parents-first topologies, interpreted symbolically the way the kernels use them.
//
// stdin: one topology per line: N, then N-1 parents (links 1..N-1), then N-1 axis codes (0 = fixed).
// stdout: one line per topology: "<rc_full> <n_slots> <rc_red> <n_red_slots> <foldable>", then one "ERR ..." line per
// violated rule.  The caller compares rc / slots / foldable with its own mirror of the builders.
//
// Rules checked, forward (rnea.cu, mass_matrix.cu, aba_body.cuh, kinematic_state.cu):
//   * psrc[i] names where link i reads its parent's state: -1 parent is the root, 0 the register (holds link i-1),
//     k > 0 slot k-1, which must still hold the parent's state (the last save to it was the parent's);
//   * no slot is overwritten while a later link still has to read the previous occupant from it.
// Backward (backward_rnea.cu pass 2, the ABA adjoint in aba_body.cuh), leaves -> root:
//   * tip[i] >= 0 (a distinct index < n_tips) exactly when link i+1 is not a child of i; otherwise link i's state is
//     re-derived from child i+1;
//   * a child hands its adjoint to a parent p != i-1, p != 0 through slot save[p]: accw 2 stores (it must be the first
//     writer of that accumulator in the backward sweep and must not clobber an accumulator still to be read), accw 1
//     adds (the slot must hold p's accumulator); accw 0 exactly for children of the root and of link i-1;
//   * when the sweep reaches a branch point, its slot holds the sum over exactly its far children.
// Fold (build_fold, stage_folded_table): red_of / full_of are inverse on the movable links, every fixed link maps to
// its parent's anchor, the carry CSR partitions the fixed links not anchored at the root, the reduced tree is
// parents-first with each movable link hung from its nearest movable ancestor, and its program passes the same checks.
#include <cstdio>
#include <set>
#include <string>
#include <vector>
#include "rnea.cu"

namespace drm {
void set_error(const char*, ...) {}
void count_launch(int) {}
int get_option(int) { return 0; }
}  // namespace drm

using namespace drm;

static int n_err = 0;
#define ERR(...) do { ++n_err; std::printf("ERR "); std::printf(__VA_ARGS__); std::printf("\n"); } while (0)

static void check_program(const char* what, const TreeProgram& P, const std::vector<int>& par) {
    const int N = (int)par.size();
    if (P.n_links != N) ERR("%s: n_links %d != %d", what, P.n_links, N);
    if (P.n_slots < 0 || P.n_slots > DRM_MAX_SLOTS) ERR("%s: n_slots %d", what, P.n_slots);
    std::vector<std::vector<int>> far(N);                  // far children: children other than i+1 (root excluded)
    for (int i = 1; i < N; ++i) {
        if (P.parent[i] != par[i]) ERR("%s: parent[%d] %d != %d", what, i, P.parent[i], par[i]);
        if (par[i] != 0 && par[i] != i - 1) far[par[i]].push_back(i);
    }
    // forward sweep
    int holder[DRM_MAX_SLOTS];
    for (int s = 0; s < DRM_MAX_SLOTS; ++s) holder[s] = -1;
    for (int i = 1; i < N; ++i) {
        const int p = par[i], src = P.psrc[i];
        if (p == 0) { if (src != -1) ERR("%s: link %d (child of the root) psrc %d", what, i, src); }
        else if (src == 0) { if (p != i - 1) ERR("%s: link %d reads the register (link %d) for parent %d", what, i, i - 1, p); }
        else if (src < 1 || src > P.n_slots) ERR("%s: link %d psrc %d outside [1, %d]", what, i, src, P.n_slots);
        else if (holder[src - 1] != p) ERR("%s: link %d reads slot %d holding link %d, parent is %d", what, i, src - 1, holder[src - 1], p);
        const int sv = P.save[i];
        if (sv >= 0) {
            if (sv >= P.n_slots) { ERR("%s: link %d saves to slot %d >= n_slots %d", what, i, sv, P.n_slots); continue; }
            const int h = holder[sv];
            if (h >= 0)
                for (int j = i + 1; j < N; ++j)
                    if (par[j] == h && P.psrc[j] > 0) ERR("%s: link %d overwrites slot %d, link %d still reads link %d from it", what, i, sv, j, h);
            holder[sv] = i;
        } else if (!far[i].empty()) {
            ERR("%s: branch point %d saves no state", what, i);
        }
    }
    // backward sweep
    std::set<int> tips;
    int acc_owner[DRM_MAX_SLOTS];
    std::set<int> acc_from[DRM_MAX_SLOTS];
    for (int s = 0; s < DRM_MAX_SLOTS; ++s) acc_owner[s] = -1;
    for (int i = N - 1; i >= 1; --i) {
        const bool next_is_child = i + 1 < N && par[i + 1] == i;
        const int tp = P.tip[i];
        if ((tp < 0) != next_is_child) ERR("%s: tip[%d] = %d but link %d %s a child", what, i, tp, i + 1, next_is_child ? "is" : "is not");
        if (tp >= 0 && (tp >= P.n_tips || !tips.insert(tp).second)) ERR("%s: tip[%d] = %d reused or >= n_tips %d", what, i, tp, P.n_tips);
        if (P.save[i] >= 0 && P.save[i] < DRM_MAX_SLOTS) {           // the sweep reaches a branch point: consume its accumulator
            const int s = P.save[i];
            std::set<int> want(far[i].begin(), far[i].end());
            if (acc_owner[s] != i || acc_from[s] != want) ERR("%s: branch point %d finds slot %d owned by %d with %zu of %zu far children", what, i, s, acc_owner[s], acc_from[s].size(), want.size());
            acc_owner[s] = -1;
            acc_from[s].clear();
        }
        const int p = par[i], w = P.accw[i];
        if (p == 0 || p == i - 1) { if (w != 0) ERR("%s: link %d (parent %d) accw %d", what, i, p, w); continue; }
        const int s = P.save[p];
        if (s < 0 || s >= DRM_MAX_SLOTS) { ERR("%s: far parent %d of link %d has no slot", what, p, i); continue; }
        if (w == 2) {
            if (acc_owner[s] >= 0) ERR("%s: link %d stores into slot %d over the live accumulator of %d", what, i, s, acc_owner[s]);
            acc_owner[s] = p;
            acc_from[s] = {i};
        } else if (w == 1) {
            if (acc_owner[s] != p) ERR("%s: link %d adds into slot %d owned by %d, not its parent %d", what, i, s, acc_owner[s], p);
            acc_from[s].insert(i);
        } else {
            ERR("%s: link %d has far parent %d but accw %d", what, i, p, w);
        }
    }
    if ((int)tips.size() != P.n_tips) ERR("%s: %zu tips used, n_tips %d", what, tips.size(), P.n_tips);
    for (int s = 0; s < DRM_MAX_SLOTS; ++s) if (acc_owner[s] >= 0) ERR("%s: accumulator of %d in slot %d never read", what, acc_owner[s], s);
}

static void check_fold(const FoldProgram& F, const TreeProgram& red, const std::vector<int>& par, const std::vector<int>& axis) {
    const int N = (int)par.size();
    int n_mov = 0;
    for (int l = 1; l < N; ++l) n_mov += axis[l] != 0;
    if (F.n_full != N || F.n_red != 1 + n_mov) { ERR("fold: n_full %d n_red %d for N %d with %d movable", F.n_full, F.n_red, N, n_mov); return; }
    if (F.red_of[0] != 0 || F.full_of[0] != 0) ERR("fold: root maps to %d / %d", F.red_of[0], F.full_of[0]);
    int prev = 0;
    for (int j = 1; j < F.n_red; ++j) {
        const int l = F.full_of[j];
        if (l <= prev || l >= N || axis[l] == 0 || F.red_of[l] != j) ERR("fold: full_of[%d] = %d", j, l);
        prev = l;
    }
    std::vector<int> red_par(F.n_red, -1);
    for (int l = 1; l < N; ++l) {
        if (F.parent[l] != par[l] || F.axis[l] != axis[l]) ERR("fold: link %d parent/axis copy", l);
        if (axis[l] != 0) {
            const int j = F.red_of[l];
            if (j < 1 || j >= F.n_red || F.full_of[j] != l) ERR("fold: red_of[%d] = %d", l, j);
            else red_par[j] = F.red_of[par[l]];
        } else if (F.red_of[l] != F.red_of[par[l]]) {
            ERR("fold: fixed link %d maps to %d, its parent to %d", l, F.red_of[l], F.red_of[par[l]]);
        }
    }
    if (F.carry_start[0] != 0 || (F.n_red > 1 && F.carry_start[1] != 0)) ERR("fold: links carried by the root");
    std::vector<int> seen(N, 0);
    for (int j = 0; j < F.n_red; ++j) {
        if (F.carry_start[j + 1] < F.carry_start[j]) ERR("fold: carry_start not monotone at %d", j);
        for (int e = F.carry_start[j]; e < F.carry_start[j + 1]; ++e) {
            const int l = F.carry[e];
            if (l < 1 || l >= N || axis[l] != 0 || F.red_of[l] != j) ERR("fold: carry[%d] = %d in bucket %d", e, l, j);
            else ++seen[l];
        }
    }
    for (int l = 1; l < N; ++l) {
        const int want = (axis[l] == 0 && F.red_of[l] != 0) ? 1 : 0;
        if (seen[l] != want) ERR("fold: fixed link %d carried %d times, want %d", l, seen[l], want);
    }
    for (int j = 1; j < F.n_red; ++j) if (red_par[j] < 0 || red_par[j] >= j) ERR("fold: reduced link %d parent %d", j, red_par[j]);
    for (int j = 1; j < F.n_red; ++j) if (red.axis[j] != axis[F.full_of[j]]) ERR("fold: reduced link %d axis", j);
    check_program("red", red, red_par);
}

int main() {
    int N, count = 0;
    while (std::scanf("%d", &N) == 1) {
        std::vector<int> par(N, -1), axis(N, 0);
        for (int i = 1; i < N; ++i) if (std::scanf("%d", &par[i]) != 1) return 2;
        for (int i = 1; i < N; ++i) if (std::scanf("%d", &axis[i]) != 1) return 2;
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
        TreeProgram full, red;
        FoldProgram fold;
        bool fo = false;
        const int rc_full = build_tree_program(&topo, &full);
        const int rc_red = build_fold(&topo, &red, &fold, &fo);
        std::printf("%d %d %d %d %d\n", rc_full, rc_full == 0 ? full.n_slots : -1, rc_red, rc_red == 0 ? red.n_slots : -1, fo ? 1 : 0);
        if (rc_full == 0) check_program("full", full, par);
        if (rc_red == 0) check_fold(fold, red, par, axis);
        ++count;
    }
    std::printf("checked %d topologies, %d errors\n", count, n_err);
    return n_err ? 1 : 0;
}
