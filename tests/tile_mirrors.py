"""Python mirrors of the host-side tile choosers of four kernels, and of the shared-memory layouts they size tiles by:

  * dynamics_derivatives.cu  deriv_tile: TC = 128 / n configurations per CTA, lowered one by one while the CTA
                             (DerivSmemLayout) exceeds 113 KB; ELIMIT when TC = 1 still exceeds 227 KB;
  * inverse_kinematics.cu    ik_tile: T = 64 rows per CTA if IkSmemLayout(64) fits 113 KB, else 32;
  * inverse_kinematics_multi.cu  ikm_tile: T = 64, 32, ..., 1 (IkmSmemLayout), first that fits 113 KB;
  * operational_space.cu     osd_tile: the same ladder over OsdSmemLayout (one template instantiation per rung).

Every chooser adds the kernel's static shared memory (STATIC_SMEM, what `-Xptxas -v` reports) to the dynamic bytes.
tests/host_checks/tile_check.cu evaluates the real layout structs on the real programs; tests/test_tile_choice.py pins
these mirrors to it.  A choice is (tile, bytes): bytes is the CTA's dynamic + static shared memory, the number an ELIMIT
message names; tile is None for a refusal.

Test helper module (not a conftest).
"""
from typing import Optional, Tuple

import synthetic_robots as S

TWO_CTAS = 113 * 1024          # a CTA at most this large leaves room for a second one on the SM
SMEM_CAP = 227 * 1024          # the most shared memory one CTA may have
TABLE_STRIDE = 28              # DRMB200_TABLE_STRIDE
STATIC_SMEM = {"deriv": 128, "ik": 0, "ikm": 0, "osd": 128}     # static shared bytes per kernel (-Xptxas -v)
LADDER = (64, 32, 16, 8, 4, 2, 1)                                # IKM / OSD tile sizes, largest first

Choice = Tuple[Optional[int], int]


def up4(x):
    return (x + 3) & ~3


# ------------------------------------------------------------------------------------------------
# dynamics derivatives
# ------------------------------------------------------------------------------------------------
def deriv_floats(tc, n, n_links, n_slots, fold_full, fd):
    """DerivSmemLayout(tc, n, n_links, n_slots, fold_full, fd).total_floats."""
    s = tc * n
    o = 3 * up4(s) + (3 if fd else 2) * up4(s * n) + n_links * TABLE_STRIDE
    o += up4(max(n_links * (32 if fd else 20) * s, fold_full * 40))
    return o + n_slots * (96 if fd else 36) * s


def deriv_choice(n, n_links, n_slots, fold_full, fd) -> Choice:
    """deriv_tile's tile for a program of n_links links (n movable) and n_slots branch slots; fold_full is the
    full link count when the kernel folds while staging, else 0."""
    static = STATIC_SMEM["deriv"]
    tc = 1 if n >= 128 else 128 // n
    while tc > 1 and 4 * deriv_floats(tc, n, n_links, n_slots, fold_full, fd) + static > TWO_CTAS:
        tc -= 1
    need = 4 * deriv_floats(tc, n, n_links, n_slots, fold_full, fd) + static
    return (tc if need <= SMEM_CAP else None), need


def deriv_program(parents, movable, fold=True, prefolded=False):
    """(n, n_links, n_slots, fold_full) of the program derivatives_device runs: the folded tree when the model is foldable
    and the "rnea_fold" option is on (folding while staging unless the rows are folded already), else the full tree."""
    n = sum(movable[1:])
    if S.foldable(parents, movable) and (fold or prefolded):
        return n, 1 + n, S.live_slots(S.reduced_parents(parents, movable)), 0 if prefolded else len(parents)
    return n, len(parents), S.live_slots(parents), 0


# ------------------------------------------------------------------------------------------------
# single-link inverse kinematics
# ------------------------------------------------------------------------------------------------
def ik_floats(T, n, path_len):
    """IkSmemLayout(T, n, path_len).total_floats."""
    return path_len * 12 + 2 * n + 2 * n * T + 12 * n * T + 7 * T


def ik_choice(n, path_len) -> Choice:
    static = STATIC_SMEM["ik"]
    T = 64 if 4 * ik_floats(64, n, path_len) + static <= TWO_CTAS else 32
    need = 4 * ik_floats(T, n, path_len) + static
    return (T if need <= SMEM_CAP else None), need


def path_len(parents, link):
    k = 0
    while link > 0:
        link, k = parents[link], k + 1
    return k


# ------------------------------------------------------------------------------------------------
# the depth-first walk of several links (build_multi_program, fk_tree.cu)
# ------------------------------------------------------------------------------------------------
def multi_program(parents, movable, links):
    """(n_steps, n_u, n_jslots, n_state_slots) of build_multi_program's walk of the union of the root -> link paths;
    n_state_slots is uncapped (> MAX_SLOTS: the builder refuses)."""
    N = len(parents)
    marked = [False] * N
    for l in links:
        while l > 0:
            marked[l] = True
            l = parents[l]
    n_children = [0] * N
    for i in range(1, N):
        if marked[i]:
            n_children[parents[i]] += 1
    depth = [0] * N
    slot_of, remaining, busy = [0] * N, [0] * N, []
    stack = [i for i in range(N - 1, 0, -1) if marked[i] and parents[i] == 0]
    n_steps = n_u = n_jslots = n_slots = 0
    while stack:
        l = stack.pop()
        p = parents[l]
        depth[l] = depth[p] + (1 if movable[l] else 0)
        n_u += movable[l]
        n_jslots = max(n_jslots, depth[l])
        if p != 0 and n_children[p] > 1:
            remaining[p] -= 1
            if remaining[p] == 0:
                busy[slot_of[p]] = False
        if n_children[l] > 1:
            s = next((k for k, b in enumerate(busy) if not b), len(busy))
            if s == len(busy):
                busy.append(True)
            busy[s] = True
            slot_of[l], remaining[l] = s, n_children[l]
            n_slots = max(n_slots, s + 1)
        stack.extend(c for c in range(N - 1, l, -1) if marked[c] and parents[c] == l)
        n_steps += 1
    return n_steps, n_u, n_jslots, n_slots


# ------------------------------------------------------------------------------------------------
# multi-link inverse kinematics
# ------------------------------------------------------------------------------------------------
def ikm_floats(T, n, n_u, n_ee, pose, n_steps, n_jslots, n_state_slots):
    """IkmSmemLayout(T, n, n_u, n_ee, pose, n_steps, n_jslots, n_state_slots).total_floats."""
    M = (6 if pose else 3) * n_ee
    m = min(M, n_u)
    tw = 7 if pose else 3
    per_row = 2 * n + 2 * M * n_u + 2 * M + tw * n_ee + m * (m + 1) // 2 + m + 6 * n_jslots + 12 * n_state_slots
    return n_steps * 12 + 2 * n + per_row * T


def ladder(floats_of, static) -> Choice:
    """The first rung of LADDER whose CTA fits TWO_CTAS (else a one-row CTA), refused above SMEM_CAP."""
    T = next((t for t in LADDER if 4 * floats_of(t) + static <= TWO_CTAS), 1)
    need = 4 * floats_of(T) + static
    return (T if need <= SMEM_CAP else None), need


def ikm_choice(parents, movable, links, pose) -> Choice:
    n = sum(movable[1:])
    n_steps, n_u, n_jslots, n_slots = multi_program(parents, movable, links)
    return ladder(lambda T: ikm_floats(T, n, n_u, len(links), pose, n_steps, n_jslots, n_slots), STATIC_SMEM["ikm"])


# ------------------------------------------------------------------------------------------------
# operational-space dynamics
# ------------------------------------------------------------------------------------------------
def osd_floats(T, n, n_links, tree_slots, n_u, M, n_jslots, n_state_slots):
    """OsdSmemLayout(T, tree program, walk, M).total_floats (AbaSmemLayout of the full tree first)."""
    aba = 4 * T * n + n_links * TABLE_STRIDE + n_links * 14 * T + tree_slots * 42 * T
    return aba + T * (M * n_u + 6 * n_jslots + 24 * n_state_slots + 3 * M + M * M)


def osd_choice(parents, movable, links, pose) -> Choice:
    n = sum(movable[1:])
    _, n_u, n_jslots, n_slots = multi_program(parents, movable, links)
    M = (6 if pose else 3) * len(links)
    tree_slots = S.live_slots(parents)
    return ladder(lambda T: osd_floats(T, n, len(parents), tree_slots, n_u, M, n_jslots, n_slots), STATIC_SMEM["osd"])

