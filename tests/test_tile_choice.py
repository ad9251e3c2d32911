"""CPU: the tile choosers of the dynamics-derivatives, inverse-kinematics, multi-link inverse-kinematics and
operational-space kernels.

tests/host_checks/tile_check.cu, compiled for the host with nvcc, builds the real programs and evaluates the real
shared-memory layout structs; its choice (tile and bytes) must equal the Python mirrors of tests/tile_mirrors.py on every
shipped robot with its usual link sets, every synthetic family and about 500 random topologies, with 1-8 links in pose and
position mode.  The GPU tests take their expectations (tile sizes, refusals and the bytes an ELIMIT message names) from
those mirrors, so this file is what makes them trustworthy.  It also prints which model reaches each tile and asserts that
every reachable rung of every ladder is reached.
"""
import os
import random
import shutil
import subprocess
from collections import defaultdict

import pytest

from conftest import REPO, URDFS, urdf_path
import differentiable_robot_model_b200 as drm
import synthetic_robots as S
import tile_mirrors as TM
from test_topology_programs import random_topologies

ELIMIT, EINVAL, NO_DOFS = -3, -1, -1000
COLUMNS = ["deriv_id", "deriv_fd", "deriv_id_nofold", "deriv_fd_nofold", "deriv_id_prefolded", "deriv_fd_prefolded", "ik",
           "ikm_pose", "ikm_position", "osd_pose", "osd_position"]
# link sets of the shipped robots (the ones their GPU tests use)
TIPS = ["link_3.0_tip", "link_7.0_tip", "link_11.0_tip", "link_15.0_tip"]
JACO_TIPS = ["j2n6s300_link_finger_tip_1", "j2n6s300_link_finger_tip_2", "j2n6s300_link_finger_tip_3"]
SHIPPED_LINKS = {
    "2link_robot": [["endEffector"]], "iiwa7": [["iiwa_link_ee"], ["iiwa_link_ee", "iiwa_link_4"]],
    "panda_no_gripper": [["panda_virtual_ee_link"]], "panda": [["panda_virtual_ee_link"], ["panda_virtual_ee_link", "panda_link4"]],
    "allegro_hand_description_left": [["link_15.0_tip"], TIPS], "allegro_hand_description_left_small_damping": [["link_3.0_tip"]],
    "trifinger_edu": [["finger_tip_link_240"], ["finger_tip_link_0", "finger_tip_link_120", "finger_tip_link_240"]],
    "jaco_clean": [["j2n6s300_link_finger_tip_3"]], "jaco": [["j2n6s300_link_6"], JACO_TIPS, JACO_TIPS + ["j2n6s300_end_effector"]],
    "fetch_arm_no_gripper": [["virtual_ee_link"]], "fetch_arm_no_gripper_small_damping": [["virtual_ee_link"]],
    "iiwa7_allegro": [["link_15.0_tip"], TIPS],
}
# Rungs no model within 64 links can reach.  One row of the multi-link IK needs at most about 32 KB (n = n_u = 63 joints
# and 8 links in pose mode: 2 M n_u = 6 048 floats of Jacobians, the 48 x 48 triangle, ...) and one row of the
# operational-space kernel about 28 KB, so a two-row CTA always fits 113 KB and the one-row instantiation never runs.  In
# position mode (M <= 24) a row needs at most about 16 KB and 15 KB: four rows always fit, and T = 2 never runs either.
UNREACHABLE = {("ikm_pose", 1), ("ikm_position", 1), ("osd_pose", 1), ("osd_position", 1), ("ikm_position", 2),
               ("osd_position", 2)}


def deepest(parents, movable, k):
    """The k links with the most movable joints on their root path (ties: lower index)."""
    def depth(l):
        d = 0
        while l > 0:
            d, l = d + movable[l], parents[l]
        return d
    return sorted(range(1, len(parents)), key=lambda l: (-depth(l), l))[:k] or [0]


def mirror(parents, movable, links):
    """The row tile_check prints for a case, from the mirrors: eleven (tile, bytes)."""
    n = sum(movable[1:])
    tree_refused = S.live_slots(parents) > S.MAX_SLOTS or S.live_slots(S.reduced_parents(parents, movable)) > S.MAX_SLOTS
    row = []
    for fold, pre in ((True, False), (False, False), (False, True)):
        for fd in (False, True):
            if tree_refused:
                row.append((ELIMIT, 0))
            elif pre and not S.foldable(parents, movable):
                row.append((EINVAL, 0))
            elif n == 0:
                row.append((NO_DOFS, 0))
            else:
                tile, need = TM.deriv_choice(*TM.deriv_program(parents, movable, fold, pre), fd)
                row.append((tile or 0, need))
    tile, need = TM.ik_choice(n, TM.path_len(parents, links[0]))
    row.append((tile or 0, need))
    walk_refused = TM.multi_program(parents, movable, links)[3] > S.MAX_SLOTS
    for choose, refused in ((TM.ikm_choice, walk_refused), (TM.osd_choice, walk_refused or tree_refused)):
        for pose in (True, False):
            if refused:
                row.append((ELIMIT, 0))
            else:
                tile, need = choose(parents, movable, links, pose)
                row.append((tile or 0, need))
    return row


def shipped_cases():
    out = []
    for stem in sorted(URDFS):
        m = drm.DifferentiableRobotModel(urdf_path(stem), stem, device="cpu")
        t = m._topology
        par = list(t.parent[:t.n_links])
        mov = [a != 0 for a in t.axis[:t.n_links]]
        for links in SHIPPED_LINKS[stem]:
            out.append((f"{stem} {len(links)} links", par, mov, [m._name_to_idx_map[nm] for nm in links]))
    return out


def family_cases():
    out = []
    for name, spec in sorted(S.families().items()):
        par, mov = spec.doc()
        for k in range(1, 9):
            out.append((f"{name} {k} deepest", par, mov, deepest(par, mov, k)))
    par, mov = S.refusal_families()["H_nine_slots"].doc()
    out.append(("H_nine_slots 8 deepest", par, mov, deepest(par, mov, 8)))
    return out


def random_cases(count=500, seed=5):
    rnd = random.Random(seed)
    out = []
    for k, (par, axis) in enumerate(random_topologies(count, seed)):
        mov = [a != 0 for a in axis]
        E = min(rnd.randint(1, 8), len(par))
        links = deepest(par, mov, E) if k % 2 else rnd.sample(range(len(par)), E)
        out.append((f"random #{k}", par, mov, links))
    return out


@pytest.fixture(scope="module")
def tile_check(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("tile_check") / "tile_check")
    # host code is what runs: PTX for the device side is enough and skips ptxas
    subprocess.run([nvcc, "-std=c++17", "-arch=compute_90a", "-code=compute_90a", "-I",
                    os.path.join(REPO, "differentiable_robot_model_b200", "csrc"), "-o", exe,
                    os.path.join(REPO, "tests", "host_checks", "tile_check.cu")], check=True, capture_output=True)
    return exe


def run_check(exe, cases):
    text = "".join(f"{len(p)} " + " ".join(map(str, p[1:] + [(3 if m else 0) for m in mv[1:]])) + f" {len(l)} "
                   + " ".join(map(str, l)) + "\n" for _, p, mv, l in cases)
    res = subprocess.run([exe], input=text, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    rows = [[int(x) for x in line.split()] for line in res.stdout.splitlines()]
    assert len(rows) == len(cases)
    return [list(zip(r[0::2], r[1::2])) for r in rows]


def test_mirrors_match_the_host_code_and_every_rung_is_reached(tile_check):
    cases = shipped_cases() + family_cases() + random_cases()
    got = run_check(tile_check, cases)
    reached = defaultdict(list)
    for (what, par, mov, links), row in zip(cases, got):
        want = mirror(par, mov, links)
        for col, g, w in zip(COLUMNS, row, want):
            assert g == w, f"{what} links {links} {col}: host code (tile, bytes) {g}, mirror {w}"
            reached[(col, "refused" if g[0] == 0 else g[0])].append(what)
    print("\nkernel               tile     cases  first model")
    for key in sorted(reached, key=lambda k: (COLUMNS.index(k[0]), str(k[1]))):
        print(f"{key[0]:20s} {str(key[1]):8s} {len(reached[key]):5d}  {reached[key][0]}")
    for col in ("ik",):
        for T in (64, 32):
            assert reached[(col, T)], (col, T)
    for col in ("ikm_pose", "ikm_position", "osd_pose", "osd_position"):
        for T in TM.LADDER:
            if (col, T) in UNREACHABLE:
                assert not reached[(col, T)], f"{col} T={T} was thought unreachable: {reached[(col, T)][:3]}"
            else:
                assert reached[(col, T)], f"no test model reaches {col} T={T}"
    for col in COLUMNS[:6]:
        tiles = {t for (c, t) in reached if c == col and isinstance(t, int) and t > 0}
        assert 1 in tiles and 128 in tiles and len(tiles) >= 8, (col, sorted(tiles))
        assert reached[(col, "refused")] or col.endswith("prefolded"), col
