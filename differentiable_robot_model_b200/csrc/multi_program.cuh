// multi_program.cuh -- the depth-first walk of the union of several root -> link paths, compiled on the host by
// build_multi_program (fk_tree.cu).  Shared by the multi-link FK kernel (fk_tree.cu) and the multi-link inverse kinematics
// (inverse_kinematics_multi.cu), so both walk the tree in the same order with the same signed table gather.
#pragma once
#include "drm_common.cuh"

namespace drm {

constexpr int MT_MAX_EE = 8;

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

// DRMB200_ELIMIT for n_ee outside [1, MT_MAX_EE] or too many live branch points, DRMB200_EINVAL for a bad topology, a link
// index out of range or a link requested twice.
int build_multi_program(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, MultiProgram* prog);

// The walk as the solver kernels (multi-link inverse kinematics, operational-space dynamics) use it, with U: the movable
// joints on the union of the paths, which span the columns of their stacked Jacobian.
struct UnionProgram {
    MultiProgram walk;
    int32_t n_u;                           // movable joints on the union of the paths
    int8_t u_dof[DRMB200_MAX_LINKS];       // U column -> q / dof column, in walk order
};

// build_multi_program, then U (fk_tree.cu)
int build_union_program(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, UnionProgram* prog);

// Link l's rows of a stacked Jacobian J [MR n_ee][n_u] (one row's slot-major slots, rows n_u T apart): J_lin = z x p_e -
// z x p_j over J_ang = z (MR = 6 only), from the walk's joint scratch jscr (z, z x p_j per path depth) and the link's
// position p_e.  Columns of joints off the link's path are left as they are (zero).
__device__ __forceinline__ void link_jacobian(const UnionProgram& P, int l, int MR, V3 p, const float* jscr, float* J, int T) {
    const int n_u = P.n_u;
    const int rs = n_u * T;
    float* Jl = J + MR * l * rs;
    for (int u = 0; u < n_u; ++u) {
        const int s = P.walk.cslot[l][P.u_dof[u]];
        if (s < 0) continue;
        const float* js = jscr + s * 6 * T;
        const V3 z = ldv(js, T), m = ldv(js + 3 * T, T);
        const V3 j = cross_add(z, p, v3(-m.x, -m.y, -m.z));
        float* col = Jl + u * T;
        col[0] = j.x; col[rs] = j.y; col[2 * rs] = j.z;
        if (MR == 6) { col[3 * rs] = z.x; col[4 * rs] = z.y; col[5 * rs] = z.z; }
    }
}

}  // namespace drm
