"""CPU: the synthetic topology families (tests/synthetic_robots.py) and the host-side program builders they exercise.

  * every generated URDF loads in the product loader and in the oracle with the same parent list, the one the family
    describes, and reaches what the family claims (live branch-point slots, foldability, size);
  * build_tree_program / build_fold (csrc/rnea.cu), compiled for the host with nvcc, on about 2 000 random
    parents-first topologies of up to 64 links plus every family: tests/host_checks/program_check.cu interprets each
    program symbolically (slot reads and writes, backward accumulators, tips, the fold maps), and its slot counts,
    refusals and foldability must match the Python mirrors;
  * the oracle's per-link dynamic state (drm_oracle.dynamic_state) against the reference's own `_bodies[i].vel / .acc /
    .force` (tests/golden/state_*.npz).
"""
import os
import random
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, REPO, urdf_path
import differentiable_robot_model_b200 as drm
import synthetic_robots as S
from oracle import drm_oracle as O


@pytest.fixture(scope="module")
def urdf_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("synthetic"))


ALL = {**S.families(), **S.refusal_families()}


@pytest.mark.parametrize("name", sorted(ALL))
def test_family_loads_in_product_and_oracle_with_the_described_tree(name, urdf_dir):
    spec = ALL[name]
    path = S.build(spec, urdf_dir)
    par, mov = spec.doc()
    robot = O.load_robot(path, torch.float64)
    assert robot.parent == par
    assert [d >= 0 for d in robot.dof] == mov
    if len(par) > S.MAX_LINKS:
        with pytest.raises(ValueError, match="exceed the engine limit of 64"):
            drm.DifferentiableRobotModel(path, name, device="cpu")
        return
    m = drm.DifferentiableRobotModel(path, name, device="cpu")
    assert m._parent_idx == par
    t = m._topology
    assert list(t.parent[:t.n_links]) == par and t.n_dofs == robot.n_dofs
    assert list(t.axis[:t.n_links]) == O.axis_codes(robot)
    # the same link and joint parameters in every document order: look them up by name
    table = m._link_table().double()
    ref = O.link_table(robot)
    assert float((table - ref).abs().max()) < 1e-6


def test_document_orders_describe_the_same_robot(urdf_dir):
    fam = S.families()
    for a, b in (("A_bfs_movable_palm", "B_dfs_movable_palm"), ("A_bfs_fixed_palm", "B_dfs_fixed_palm"), ("C_dfs", "C_random")):
        ra, rb = (O.load_robot(S.build(fam[k], urdf_dir), torch.float64) for k in (a, b))
        assert sorted(ra.names) == sorted(rb.names) and ra.names != rb.names
        for k, name in enumerate(ra.names):
            j = rb.index(name)
            assert (ra.parent[k] < 0 and rb.parent[j] < 0) or ra.names[ra.parent[k]] == rb.names[rb.parent[j]]
            for attr in ("trans", "rpy", "mass", "com", "inertia", "damping", "axis"):
                assert torch.equal(getattr(ra, attr)[k], getattr(rb, attr)[j]), (name, attr)


def random_topologies(count, seed):
    """Parents-first topologies of 1..64 links from several generators (uniform parents, chains with forks, breadth-first
    trees, random orders of bushy trees), with fixed links at varying density."""
    rnd = random.Random(seed)
    out = []
    for k in range(count):
        N = rnd.choice([1, 2, 3, rnd.randint(4, 16), rnd.randint(17, 63), 64, 64])
        kind = k % 4
        par = [-1]
        for i in range(1, N):
            if kind == 0:
                par.append(rnd.randrange(i))
            elif kind == 1:
                par.append(i - 1 if rnd.random() < 0.8 else rnd.randrange(i))
            else:
                par.append(rnd.randrange(max(0, i - rnd.randint(1, 12)), i))
        if kind == 2:
            par, _ = S.reorder(par, [False] * N, S.bfs_order(par))
        elif kind == 3:
            par, _ = S.reorder(par, [False] * N, S.random_order(par, rnd.randrange(1 << 30)))
        p_fixed = rnd.choice([0.0, 0.1, 0.3, 0.6, 0.9])
        axis = [0] + [0 if rnd.random() < p_fixed else rnd.choice([-3, -2, -1, 1, 2, 3]) for _ in range(N - 1)]
        out.append((par, axis))
    return out


@pytest.fixture(scope="module")
def program_check(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("program_check") / "program_check")
    subprocess.run([nvcc, "-std=c++17", "-arch=sm_90a", "-I", os.path.join(REPO, "differentiable_robot_model_b200", "csrc"),
                    "-o", exe, os.path.join(REPO, "tests", "host_checks", "program_check.cu")], check=True, capture_output=True)
    return exe


def test_tree_and_fold_programs_interpret_correctly_on_random_topologies(program_check):
    topos = random_topologies(2000, seed=1)
    for spec in list(S.families().values()) + [S.refusal_families()["H_nine_slots"]]:
        par, mov = spec.doc()
        topos.append((par, [0] + [3 if m else 0 for m in mov[1:]]))
    text = "".join(f"{len(p)} " + " ".join(map(str, p[1:] + a[1:])) + "\n" for p, a in topos)
    res = subprocess.run([program_check], input=text, capture_output=True, text=True)
    lines = res.stdout.splitlines()
    errors = [l for l in lines if l.startswith("ERR")]
    assert res.returncode == 0 and not errors, "\n".join(errors[:20]) + res.stderr
    rows = [tuple(int(x) for x in l.split()) for l in lines if not l.startswith(("ERR", "checked"))]
    assert len(rows) == len(topos)
    ELIMIT = -3
    reached = {"refused": 0, "max": 0, "red_refused": 0, "unfoldable": 0, "foldable": 0}
    for (par, axis), (rc, slots, rc_red, red_slots, fo) in zip(topos, rows):
        mov = [a != 0 for a in axis]
        want = S.live_slots(par)
        if want > S.MAX_SLOTS:
            assert (rc, slots) == (ELIMIT, -1), (par, rc)
            reached["refused"] += 1
        else:
            assert (rc, slots) == (0, want), (par, rc, slots, want)
            reached["max"] += want == S.MAX_SLOTS
        want_red = S.live_slots(S.reduced_parents(par, mov))
        if want_red > S.MAX_SLOTS:
            assert (rc_red, red_slots) == (ELIMIT, -1)
            reached["red_refused"] += 1
        else:
            assert (rc_red, red_slots) == (0, want_red)
        assert bool(fo) == S.foldable(par, mov), (par, axis)
        reached["foldable" if fo else "unfoldable"] += 1
    assert min(reached.values()) >= 5, reached           # every outcome is reached, not just the easy one


STATE = {"state_iiwa7": "iiwa7", "state_allegro_left": "allegro_hand_description_left",
         "state_iiwa7_allegro": "iiwa7_allegro", "state_trifinger_edu": "trifinger_edu"}


@pytest.mark.parametrize("stem", sorted(STATE))
def test_oracle_dynamic_state_matches_reference_bodies(stem):
    """dynamic_state against `_bodies[i].vel / .acc / .force` of the reference after compute_inverse_dynamics (fp32
    reference, so family-relative 2e-6), and inverse_dynamics is the torque of the same evaluation, bit for bit."""
    g = np.load(os.path.join(GOLDEN_DIR, stem + ".npz"))
    robot = O.load_robot(urdf_path(STATE[stem]), torch.float64)
    q, qd, qdd = (torch.tensor(g[k]).double() for k in ("q", "qd", "qdd"))
    for tag, grav in (("g1", True), ("g0", False)):
        s = O.dynamic_state(robot, q, qd, qdd, grav, True)
        assert torch.equal(s["tau"], O.inverse_dynamics(robot, q, qd, qdd, grav, True))
        for key in ("vel_ang", "vel_lin", "acc_ang", "acc_lin", "force_ang", "force_lin"):
            want = g[f"{key}.{tag}"]
            got = s[key].numpy()
            assert got.shape == want.shape, key
            err = np.abs(got - want).max() / np.abs(want).max()
            assert err <= 2e-6, f"{stem} {key}.{tag}: family-relative error {err:.2e}"
