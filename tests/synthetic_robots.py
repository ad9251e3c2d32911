"""Seeded URDF models of topologies the shipped robots never produce, for the topology tests.

A model is an abstract tree (``parents``, ``movable``; abstract link ids, parents-first) written to a URDF in some
parents-first document ORDER.  The link and joint parameters are drawn per abstract link from the seed, so two orders of
the same tree describe the same robot: link ``l<k>`` is abstract link k in every order, and only the DoF numbering
(document order of the movable joints) differs.

Every family states what it is there to reach (live branch-point slots of the full and of the folded tree, foldability,
size) and ``build()`` asserts it with Python mirrors of the host-side program builders (``build_tree_program`` and
``build_fold`` in ``csrc/rnea.cu``), so a family cannot drift into the easy case.

Test helper module (not a conftest): imported by test_topology_programs.py and test_synthetic_topologies_gpu.py.
"""
import os
import random
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

MAX_SLOTS = 8            # DRM_MAX_SLOTS (csrc/drm_common.cuh)
MAX_LINKS = 64           # DRMB200_MAX_LINKS
AXES = ("1 0 0", "-1 0 0", "0 1 0", "0 -1 0", "0 0 1", "0 0 -1")


# ------------------------------------------------------------------------------------------------
# mirrors of the host-side program builders
# ------------------------------------------------------------------------------------------------
def live_slots(parents: Sequence[int]) -> int:
    """Shared-memory state slots build_tree_program needs for a parents-first tree (uncapped: > MAX_SLOTS means the
    builder refuses).  A link is a branch point if it has a child other than the next link (children of the root
    excluded); its slot stays busy up to and including its last such child."""
    N = len(parents)
    last_far = [-1] * N
    for i in range(1, N):
        p = parents[i]
        if p != i - 1 and p != 0:
            last_far[p] = i
    busy_until: List[int] = []          # per slot: the last link that still reads it
    peak = 0
    for i in range(1, N):
        if last_far[i] >= 0:
            s = next((k for k, until in enumerate(busy_until) if until < i), len(busy_until))
            if s == len(busy_until):
                busy_until.append(last_far[i])
            else:
                busy_until[s] = last_far[i]
            peak = max(peak, s + 1)
    return peak


def reduced_parents(parents: Sequence[int], movable: Sequence[bool]) -> List[int]:
    """Parent list of the folded tree of build_fold: the root and the movable links in document order, each movable
    link hung from its nearest movable ancestor (or the root)."""
    red_of = [0] * len(parents)
    red = [-1]
    for l in range(1, len(parents)):
        if movable[l]:
            red.append(red_of[parents[l]])
            red_of[l] = len(red) - 1
        else:
            red_of[l] = red_of[parents[l]]
    return red


def foldable(parents: Sequence[int], movable: Sequence[bool]) -> bool:
    """build_fold's rule: something to fold, a movable link to fold it into, and staging scratch (40 floats per link)
    that fits the per-link state region of the smallest tile (8 floats per reduced link x 32 configurations)."""
    N = len(parents)
    n_red = 1 + sum(1 for l in range(1, N) if movable[l])
    n_fixed = N - n_red
    return n_fixed > 0 and n_red > 1 and N * 40 <= n_red * 8 * 32


# ------------------------------------------------------------------------------------------------
# document orders of an abstract tree
# ------------------------------------------------------------------------------------------------
def _children(parents):
    ch = [[] for _ in parents]
    for i in range(1, len(parents)):
        ch[parents[i]].append(i)
    return ch


def dfs_order(parents):
    ch, out, stack = _children(parents), [], [0]
    while stack:
        l = stack.pop()
        out.append(l)
        stack.extend(reversed(ch[l]))
    return out


def bfs_order(parents):
    ch, out = _children(parents), [0]
    for l in out:
        out.extend(ch[l])
    return out


def random_order(parents, seed):
    """A uniformly drawn parents-first order: repeatedly emit a random link whose parent is already placed."""
    rnd = random.Random(seed)
    ch, out, ready = _children(parents), [0], list(_children(parents)[0])
    while ready:
        l = ready.pop(rnd.randrange(len(ready)))
        out.append(l)
        ready.extend(ch[l])
    return out


def reorder(parents, movable, order):
    """(parents, movable) of the tree in document order `order` (order[k] = abstract id of document link k)."""
    pos = {a: k for k, a in enumerate(order)}
    return [-1] + [pos[parents[a]] for a in order[1:]], [movable[a] for a in order]


# ------------------------------------------------------------------------------------------------
# model description + URDF writer
# ------------------------------------------------------------------------------------------------
@dataclass
class Spec:
    name: str
    parents: List[int]                       # abstract tree, parents-first
    movable: List[bool]
    order: Optional[List[int]] = None        # document order (abstract ids); None = identity
    seed: int = 0
    massless: Sequence[int] = ()             # abstract links with mass 0 / inertia 0 and a zero joint origin
    axes: Dict[int, int] = field(default_factory=dict)   # abstract link -> index into AXES (else random)
    claims: Dict[str, object] = field(default_factory=dict)

    def doc(self):
        """(parents, movable) in document order."""
        return reorder(self.parents, self.movable, self.order or list(range(len(self.parents))))

    def check_claims(self):
        par, mov = self.doc()
        got = {"n_links": len(par), "n_dofs": sum(mov[1:]), "slots": live_slots(par),
               "red_slots": live_slots(reduced_parents(par, mov)), "foldable": foldable(par, mov)}
        for key, want in self.claims.items():
            if key.endswith("_min"):
                assert got[key[:-4]] >= want, f"{self.name}: {key[:-4]} = {got[key[:-4]]} < {want}"
            else:
                assert got[key] == want, f"{self.name}: {key} = {got[key]}, the family claims {want}"
        return got


def _params(spec):
    """Per-abstract-link parameters drawn from the seed (independent of the document order)."""
    rnd = random.Random(spec.seed)
    out = []
    for a in range(len(spec.parents)):
        m = rnd.uniform(0.2, 2.0)
        d = [m * rnd.uniform(0.002, 0.01) for _ in range(3)]
        off = [0.2 * min(d) * rnd.uniform(-1, 1) for _ in range(3)]
        p = dict(mass=m, com=[rnd.uniform(-0.05, 0.05), rnd.uniform(-0.05, 0.05), rnd.uniform(0.0, 0.1)],
                 inertia=[d[0], off[0], off[1], d[1], off[2], d[2]],
                 xyz=[rnd.uniform(-0.1, 0.1), rnd.uniform(-0.1, 0.1), rnd.uniform(0.05, 0.2)],
                 rpy=[rnd.uniform(-1, 1), rnd.uniform(-1, 1), rnd.uniform(-1, 1)],
                 axis=spec.axes.get(a, rnd.randrange(6)), damping=rnd.uniform(0.05, 0.5),
                 lower=-rnd.uniform(1.5, 2.5), upper=rnd.uniform(1.5, 2.5), velocity=rnd.uniform(1.0, 3.0))
        if a in spec.massless:
            p.update(mass=0.0, com=[0.0, 0.0, 0.0], inertia=[0.0] * 6, xyz=[0.0, 0.0, 0.0], rpy=[0.0, 0.0, 0.0])
        out.append(p)
    return out


def urdf_text(spec):
    order = spec.order or list(range(len(spec.parents)))
    prm = _params(spec)
    f = lambda v: " ".join(f"{x:.7g}" for x in v)      # noqa: E731
    lines = [f'<robot name="{spec.name}">']
    for a in order:
        p = prm[a]
        ixx, ixy, ixz, iyy, iyz, izz = p["inertia"]
        lines.append(f'  <link name="l{a}"><inertial><origin xyz="{f(p["com"])}"/><mass value="{p["mass"]:.7g}"/>'
                     f'<inertia ixx="{ixx:.7g}" ixy="{ixy:.7g}" ixz="{ixz:.7g}" iyy="{iyy:.7g}" iyz="{iyz:.7g}" '
                     f'izz="{izz:.7g}"/></inertial></link>')
    for a in order[1:]:
        p = prm[a]
        kind = "revolute" if spec.movable[a] else "fixed"
        body = f'<parent link="l{spec.parents[a]}"/><child link="l{a}"/><origin xyz="{f(p["xyz"])}" rpy="{f(p["rpy"])}"/>'
        if spec.movable[a]:
            body += (f'<axis xyz="{AXES[p["axis"]]}"/><limit effort="10" lower="{p["lower"]:.7g}" upper="{p["upper"]:.7g}" '
                     f'velocity="{p["velocity"]:.7g}"/><dynamics damping="{p["damping"]:.7g}"/>')
        lines.append(f'  <joint name="j{a}" type="{kind}">{body}</joint>')
    lines.append("</robot>")
    return "\n".join(lines) + "\n"


def build(spec, directory):
    """Check the family's claims, write `<directory>/<name>.urdf` and return its path."""
    spec.check_claims()
    path = os.path.join(directory, spec.name + ".urdf")
    with open(path, "w") as fh:
        fh.write(urdf_text(spec))
    return path


def leaves(parents):
    has_child = set(parents[1:])
    return [i for i in range(1, len(parents)) if i not in has_child]


# ------------------------------------------------------------------------------------------------
# families
# ------------------------------------------------------------------------------------------------
class _Tree:
    def __init__(self):
        self.parents, self.movable = [-1], [False]

    def add(self, parent, movable=True):
        self.parents.append(parent)
        self.movable.append(movable)
        return len(self.parents) - 1

    def chain(self, parent, n, movable=True):
        for _ in range(n):
            parent = self.add(parent, movable)
        return parent


def hand_on_arm(fingers, finger_links=4, palm_movable=True):
    """A 3-link arm, a palm and `fingers` fingers of `finger_links` links, as an abstract tree (depth-first ids)."""
    t = _Tree()
    palm = t.add(t.chain(0, 3), palm_movable)
    for _ in range(fingers):
        t.chain(palm, finger_links)
    return t


def humanoid():
    """Torso -> two 7-DoF arms each ending in a palm with 3 two-link fingers, plus a 2-DoF head; pelvis (the root) ->
    two 6-DoF legs with a fixed foot."""
    t = _Tree()
    for _ in range(2):
        t.add(t.chain(0, 6), False)
    torso = t.add(0)
    for _ in range(2):
        palm = t.add(t.chain(torso, 7), False)
        for _ in range(3):
            t.chain(palm, 2)
    t.chain(torso, 2)
    return t


def fixed_structures():
    """Runs of fixed joints, a fixed branch point with movable children, fixed leaves with mass, massive links fixed to
    the root and massless virtual links between consecutive revolute joints (a 3-axis joint)."""
    t = _Tree()
    t.chain(t.add(0, False), 1, False)              # massive links fixed to the root (a fixed run hanging off it)
    a = t.add(0)
    run = t.chain(a, 3, False)                      # three consecutive fixed joints
    b = t.add(run)
    hub = t.add(b, False)                           # fixed branch point with movable children
    c = t.add(hub)
    t.add(c, False)                                 # fixed leaf with mass
    t.chain(hub, 2)
    v1 = t.add(hub)
    v2 = t.add(v1)                                  # v2, v3: massless links of a 3-axis joint (v1 -> v2 -> v3 -> w)
    v3 = t.add(v2)
    w = t.add(v3)
    t.chain(t.add(w, False), 4, False)              # a fixed run of 4 ending in a fixed leaf
    d = t.add(run)                                  # a second movable child of the fixed run's end
    t.add(d, False)
    return t, (v2, v3), {v1: 0, v2: 2, v3: 4, w: 0}


def unfoldable():
    """Far more fixed links than movable ones: three revolute joints, each followed by a fixed run of 8 (one of them
    forking), so N * 40 > n_red * 8 * 32 and the kernels walk the full tree even with rnea_fold on."""
    t = _Tree()
    p = 0
    for k in range(3):
        p = t.add(p)
        end = t.chain(p, 8 if k != 1 else 5, False)
        if k == 1:
            t.chain(p, 3, False)
        p = end
    return t


def random_tree(n_links, seed, max_slots=MAX_SLOTS, fixed_share=0.2):
    """A random parents-first tree of `n_links` links whose tree program fits `max_slots` (rejection sampling)."""
    rnd = random.Random(seed)
    while True:
        parents, movable = [-1], [False]
        for i in range(1, n_links):
            parents.append(rnd.choice(range(max(0, i - 6), i)) if rnd.random() < 0.5 else i - 1)
            movable.append(rnd.random() >= fixed_share)
        movable[1] = True
        if live_slots(parents) <= max_slots:
            return parents, movable


def families():
    """name -> Spec for every family the tests run (the refusal models excluded: see refusal_families)."""
    out = {}
    for palm_movable, tag in ((True, "movable_palm"), (False, "fixed_palm")):
        t = hand_on_arm(7, palm_movable=palm_movable)
        n_dofs = sum(t.movable[1:])
        out[f"A_bfs_{tag}"] = Spec(f"A_bfs_{tag}", t.parents, t.movable, bfs_order(t.parents), seed=11,
                                   claims=dict(n_links=33, n_dofs=n_dofs, slots=8, red_slots=8, foldable=not palm_movable))
        out[f"B_dfs_{tag}"] = Spec(f"B_dfs_{tag}", t.parents, t.movable, dfs_order(t.parents), seed=11,
                                   claims=dict(n_links=33, n_dofs=n_dofs, slots=1, red_slots=1, foldable=not palm_movable))
    h = humanoid()
    out["C_dfs"] = Spec("C_dfs", h.parents, h.movable, dfs_order(h.parents), seed=21,
                        claims=dict(n_links=46, n_dofs=41, slots=2, red_slots=2, foldable=True))
    out["C_random"] = Spec("C_random", h.parents, h.movable, random_order(h.parents, 5), seed=21,
                           claims=dict(n_links=46, n_dofs=41, slots_min=4, red_slots_min=4, foldable=True))
    t, massless, axes = fixed_structures()
    out["D_fixed"] = Spec("D_fixed", t.parents, t.movable, seed=31, massless=massless, axes=axes,
                          claims=dict(n_links=24, n_dofs=10, slots_min=2, red_slots_min=2, foldable=True))
    t = unfoldable()
    out["E_unfoldable"] = Spec("E_unfoldable", t.parents, t.movable, seed=41,
                               claims=dict(n_links=28, n_dofs=3, slots=2, foldable=False))
    out["F_chain64"] = Spec("F_chain64", [-1] + list(range(63)), [False] + [True] * 63, seed=51,
                            claims=dict(n_links=64, n_dofs=63, slots=0, foldable=False))
    par, mov = random_tree(64, seed=7)
    out["F_tree64"] = Spec("F_tree64", par, mov, seed=61, claims=dict(n_links=64, slots_min=3, foldable=True))
    out["G_root_only"] = Spec("G_root_only", [-1], [False], seed=71, claims=dict(n_links=1, n_dofs=0))
    out["G_all_fixed"] = Spec("G_all_fixed", [-1, 0, 1, 1], [False] * 4, seed=72, claims=dict(n_links=4, n_dofs=0, foldable=False))
    out["G_one_joint"] = Spec("G_one_joint", [-1, 0], [False, True], seed=73, claims=dict(n_links=2, n_dofs=1, slots=0, foldable=False))
    return out


def refusal_families():
    t = hand_on_arm(8)
    return {
        "H_nine_slots": Spec("H_nine_slots", t.parents, t.movable, bfs_order(t.parents), seed=81,
                             claims=dict(n_links=37, slots=9)),
        "H_65_links": Spec("H_65_links", [-1] + list(range(64)), [False] + [True] * 64, seed=82, claims=dict(n_links=65)),
    }
