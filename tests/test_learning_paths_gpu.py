"""GPU: parameter learning end to end -- from the ``nn.Parameter`` inside a parametrisation module to its ``.grad`` -- on
every robot family, learnable set, differentiable entry point and table path, against fp64 autograd of the oracle
(tests/learning_oracle.py).

A case is (robot, learnable set, entry point, batch); each runs on the per-module path, inside ``shared_link_table()`` and
on the fused path (``fuse_learnable_parameters``), and every check walks EVERY ``nn.Parameter`` of the model: its gradient
must match the fp64 value (rtol 1e-4, atol 2e-5 of the largest gradient magnitude of the case, as in test_backward_gpu.py),
be absent for a frozen module, and be exactly zero or absent for a module on a fixed-joint origin.  The host logic between
the modules and the kernels (which adjoint runs, whether a graph is built, which table is cached) never raises when it is
wrong -- it leaves a zero or stale gradient for some parameter, which is what these checks look for.
"""
import copy
import functools
import zlib

import pytest
import torch

from conftest import assert_close, urdf_path
import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200.rigid_body_params import (CovParameterized3DInertiaMatrixNet, PositiveScalar,
                                                                Symm3DInertiaMatrixNet, SymmPosDef3DInertiaMatrixNet,
                                                                TriangParam3DInertiaMatrixNet, UnconstrainedScalar,
                                                                UnconstrainedTensor)
import synthetic_robots as S
from learning_oracle import Learnable, gradients, learnable_robot
from rollout_oracle import forward_dynamics_rollout as oracle_rollout
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SYNTHETIC = "D_fixed"            # runs of fixed links, a fixed branch point and massless links (tests/synthetic_robots.py)
SMALL, RAGGED, LARGE = 33, 257, 70001      # one tile and a bit; a partial last tile; the persistent multi-tile adjoints
ROLLOUT_STEPS, DT = 4, 0.01
PATHS = ("per_module", "shared", "fused")


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("learning_paths"))


@functools.lru_cache(maxsize=None)
def robot_file(name, directory):
    return S.build(S.families()[name], directory) if name == SYNTHETIC else urdf_path(name)


@functools.lru_cache(maxsize=None)
def oracle_robot(name, directory):
    return O.load_robot(robot_file(name, directory), torch.float64)


# ------------------------------------------------------------------------------------------------
# learnable sets
# ------------------------------------------------------------------------------------------------
def make_set(robot, set_name, spread=1.0):
    """``(learnables, frozen)``: prototype modules (CPU, fp32) of the named set for an oracle robot, started at the URDF
    values moved by seeded perturbations (``spread`` 0: exactly at them), and the indices of the entries to freeze."""
    gen = torch.Generator().manual_seed(zlib.crc32(set_name.encode()))
    N = len(robot.names)
    links = list(range(1, N))
    movable = [i for i in links if robot.dof[i] >= 0]
    fixed = [i for i in links if robot.dof[i] < 0]
    massive = [i for i in links if float(robot.mass[i]) > 0]
    name = robot.names.__getitem__

    def rnd(*shape):
        return spread * torch.randn(*shape, generator=gen)

    def mass(ids, scale=1.1):
        m = sum(float(robot.mass[i]) for i in ids) / len(ids)
        if m > 0:
            return PositiveScalar(init_param=torch.tensor(m * (scale if spread else 1.0)))
        return UnconstrainedScalar(init_val=torch.zeros(1))               # a massless link: its mass stays 0, d/dm does not

    def com(i):
        return UnconstrainedTensor(1, 3, init_tensor=(robot.com[i].float() + 0.01 * rnd(3)).reshape(1, 3))

    def inertia(i):                                                       # inertia_mat is used as given, NOT symmetrised
        I = robot.inertia[i].float()
        return UnconstrainedTensor(3, 3, init_tensor=I + 0.02 * float(I.abs().max()) * rnd(3, 3))

    def damping(i):
        return UnconstrainedScalar(init_val=torch.tensor([float(robot.damping[i]) + (0.1 if spread else 0.0)]))

    def trans(i):
        return UnconstrainedTensor(1, 3, init_tensor=(robot.trans[i].float() + 0.01 * rnd(3)).reshape(1, 3))

    def rot(i):
        return UnconstrainedTensor(1, 3, init_tensor=(robot.rpy[i].float() + 0.05 * rnd(3)).reshape(1, 3))

    def inertial(ids):
        out = []
        for i in ids:
            out += [Learnable((name(i),), "mass", mass([i])), Learnable((name(i),), "com", com(i)),
                    Learnable((name(i),), "inertia_mat", inertia(i))]
            if robot.dof[i] >= 0:
                out.append(Learnable((name(i),), "joint_damping", damping(i)))
        return out

    def kinematic(ids):
        return [Learnable((name(i),), pname, make(i)) for i in ids for pname, make in (("trans", trans), ("rot_angles", rot))]

    frozen = ()
    if set_name == "inertial":
        out = inertial(links)
    elif set_name == "kinematic":
        out = kinematic(movable)
    elif set_name in ("both", "frozen"):
        out = inertial(links) + kinematic(movable)
        if set_name == "frozen":
            frozen = tuple(range(1, len(out), 3))
    elif set_name == "fixed_origin":
        f = fixed[0]
        out = kinematic([f]) + [Learnable((name(f),), "joint_damping", damping(f))] + inertial([f, movable[-1]]) + kinematic(movable[:1])
    elif set_name == "nets":
        # every inertia net class, started from one positive-definite matrix that satisfies the triangle inequalities
        shape = torch.tensor([[1.0, 0.1, 0.05], [0.1, 0.8, -0.07], [0.05, -0.07, 0.6]])
        nets = (SymmPosDef3DInertiaMatrixNet, CovParameterized3DInertiaMatrixNet, Symm3DInertiaMatrixNet,
                lambda init_param: TriangParam3DInertiaMatrixNet(bias=1e-9, init_param=init_param))
        out = kinematic(movable[:1])
        for i, net in zip(massive[:4], nets):
            out += [Learnable((name(i),), "inertia_mat", net(init_param=max(float(robot.inertia[i].abs().max()), 1e-4) * shape)),
                    Learnable((name(i),), "mass", mass([i]))]
    elif set_name == "tied2":
        a, b = [i for i in movable if i in massive][:2]
        pair = (name(a), name(b))
        out = [Learnable(pair, "mass", mass([a, b])), Learnable(pair, "com", com(a)), Learnable(pair, "trans", trans(b)),
               Learnable(pair, "joint_damping", damping(a))]
    elif set_name == "tied4":
        tips = [i for i in links if robot.names[i].endswith("_tip")][:4]
        four = tuple(name(i) for i in (tips if len(tips) == 4 else links[-4:]))
        joints = tuple(name(i) for i in movable[-4:])
        out = [Learnable(four, "mass", mass([robot.index(n) for n in four])),
               Learnable(four, "inertia_mat", inertia(robot.index(four[0]))), Learnable(joints, "rot_angles", rot(movable[-1])),
               Learnable(joints[:2], "trans", trans(movable[-2]))]
    else:
        raise KeyError(set_name)
    return out, frozen


def install(model, learnables, frozen=()):
    """Install a deep copy of every prototype module (one copy per entry: tied across its links); freeze; return them."""
    mods = []
    for links, pname, proto in learnables:
        mod = copy.deepcopy(proto)
        for link in links:
            model.make_link_param_learnable(link, pname, mod)
        mods.append(mod)
    for k in frozen:
        model.freeze_learnable_link_param(learnables[k].links[0], learnables[k].pname)
    return mods


# ------------------------------------------------------------------------------------------------
# entry points: one loss, written once, evaluated by the model (fp32, device) and by the oracle (fp64, CPU)
# ------------------------------------------------------------------------------------------------
class ModelApi:
    def __init__(self, model):
        self.m = model

    def fk(self, q, link):
        return self.m.compute_forward_kinematics(q, link)

    def jac(self, q, link):
        return self.m.compute_endeffector_jacobian(q, link)

    def multi(self, q, links):
        return self.m.compute_fk_and_jacobian_multi(q, list(links))

    def all_links(self, q):
        return self.m.compute_forward_kinematics_all_links(q)

    def inverse_dynamics(self, q, qd, qdd, gravity, damping):
        return self.m.compute_inverse_dynamics(q, qd, qdd, include_gravity=gravity, use_damping=damping)

    def nle(self, q, qd):
        return self.m.compute_non_linear_effects(q, qd)

    def mass_matrix(self, q):
        return self.m.compute_lagrangian_inertia_matrix(q)

    def forward_dynamics(self, q, qd, f):
        return self.m.compute_forward_dynamics(q, qd, f, include_gravity=True, use_damping=True)

    def rollout(self, q, qd, f):
        return self.m.compute_forward_dynamics_rollout(q, qd, f, DT, include_gravity=True, use_damping=True)


class OracleApi:
    def __init__(self, robot):
        self.r = robot

    def fk(self, q, link):
        return O.forward_kinematics(self.r, q, link)

    def jac(self, q, link):
        return O.jacobian(self.r, q, link)

    def multi(self, q, links):
        return {l: O.forward_kinematics(self.r, q, l) + O.jacobian(self.r, q, l) for l in links}

    def all_links(self, q):
        R, p, _, _, _ = O.kinematic_state(self.r, q)
        return {n: (p[i], O.quaternion(R[i])) for i, n in enumerate(self.r.names)}

    def inverse_dynamics(self, q, qd, qdd, gravity, damping):
        return O.inverse_dynamics(self.r, q, qd, qdd, gravity, damping)

    def nle(self, q, qd):
        return O.inverse_dynamics(self.r, q, qd, torch.zeros_like(q), True, True)

    def mass_matrix(self, q):                            # column j = ID(q, 0, e_j) without gravity and damping
        n, zero = self.r.n_dofs, torch.zeros_like(q)
        eye = torch.eye(n, dtype=q.dtype)
        return torch.stack([O.inverse_dynamics(self.r, q, zero, eye[j].expand_as(q), False, False) for j in range(n)], dim=2)

    def forward_dynamics(self, q, qd, f):
        return O.forward_dynamics(self.r, q, qd, f, True, True)

    def rollout(self, q, qd, f):
        return oracle_rollout(self.r, q, qd, f, DT, True, True)


def weights(tag, like):
    """Seeded fp32 normal weights of ``like``'s shape, on its device and in its dtype (so both sides use the same values)."""
    gen = torch.Generator().manual_seed(zlib.crc32(tag.encode()))
    return torch.randn(tuple(like.shape), generator=gen).to(device=like.device, dtype=like.dtype)


def weighted(tag, t):
    return (weights(tag, t) * t).sum()


def pose_loss(tag, pos, quat):
    """Position linearly; orientation through the even products q_i q_j, the same for either quaternion sign."""
    qq = quat.unsqueeze(2) * quat.unsqueeze(1)
    return weighted(tag + ".pos", pos) + weighted(tag + ".quat", qq)


def _fk(api, x):
    return pose_loss("fk", *api.fk(x["q"], x["ee"]))


def _jac(api, x):
    lin, ang = api.jac(x["q"], x["ee"])
    return weighted("jlin", lin) + weighted("jang", ang)


def _multi(api, x):
    out = api.multi(x["q"], x["tips"])
    return sum(pose_loss(l, out[l][0], out[l][1]) + weighted(l + ".jlin", out[l][2]) + weighted(l + ".jang", out[l][3])
               for l in x["tips"])


def _all_links(api, x):
    out = api.all_links(x["q"])
    return sum(pose_loss(l, *out[l]) for l in sorted(out))


def _id(gravity, damping):
    return lambda api, x: weighted("tau", api.inverse_dynamics(x["q"], x["qd"], x["qdd"], gravity, damping))


def _rollout(api, x):
    q, qd, qdd = api.rollout(x["q"], x["qd"], x["fT"])
    return weighted("roll.q", q) + weighted("roll.qd", qd) + weighted("roll.qdd", qdd)


# name -> the losses of the entry point; more than one loss = one backward() each, gradients accumulating
ENTRY = {
    "fk": (_fk,),
    "jacobian": (_jac,),
    "fk_multi": (_multi,),
    "fk_all_links": (_all_links,),
    "id_gd": (_id(True, True),), "id_g": (_id(True, False),), "id_d": (_id(False, True),), "id": (_id(False, False),),
    "nle": (lambda api, x: weighted("nle", api.nle(x["q"], x["qd"])),),
    "mass_matrix": (lambda api, x: weighted("H", api.mass_matrix(x["q"])),),
    "forward_dynamics": (lambda api, x: weighted("qdd", api.forward_dynamics(x["q"], x["qd"], x["f"])),),
    "rollout": (_rollout,),
    "combined": (lambda api, x: _fk(api, x) + _jac(api, x) + _id(True, True)(api, x),),
    "two_backwards": (_fk, _id(True, True)),
}
ENTRY_ALL = tuple(ENTRY)
ENTRY_CORE = ("fk", "fk_all_links", "id_gd", "forward_dynamics", "combined")


def inputs(robot, batch):
    """fp32 values (held in fp64 for the oracle): q, qd, qdd from the joint limits, joint forces, end effector, tips."""
    q, qd, qdd = (t.float() for t in O.sample_inputs(robot, batch, seed=batch, dtype=torch.float64))
    gen = torch.Generator().manual_seed(batch + 1)
    parents = set(robot.parent)
    tips = [n for n in robot.names if n.endswith("_tip")] or [n for i, n in enumerate(robot.names) if i and i not in parents]
    return dict(q=q, qd=qd, qdd=qdd, f=0.5 * torch.randn(batch, robot.n_dofs, generator=gen),
                fT=0.5 * torch.randn(ROLLOUT_STEPS, batch, robot.n_dofs, generator=gen), ee=robot.names[-1], tips=tuple(tips[:4]))


def cast(x, **kw):
    return {k: (v.to(**kw) if isinstance(v, torch.Tensor) else v) for k, v in x.items()}


@functools.lru_cache(maxsize=None)
def reference(robot_name, set_name, entry, batch, directory):
    """fp64 gradients of the case, once for all paths: (learnables, frozen, per entry {parameter name: gradient})."""
    robot = oracle_robot(robot_name, directory)
    learnables, frozen = make_set(robot, set_name)
    learned, leaves = learnable_robot(robot, learnables)
    x = cast(inputs(robot, batch), dtype=torch.float64)
    loss = sum(fn(OracleApi(learned), x) for fn in ENTRY[entry]) / batch
    return learnables, frozen, gradients(loss, leaves)


def run_model(model, entry, x, path):
    for fn in ENTRY[entry]:
        if path == "shared":
            with model.shared_link_table():
                loss = fn(ModelApi(model), x) / x["q"].shape[0]
        else:
            loss = fn(ModelApi(model), x) / x["q"].shape[0]
        if loss.requires_grad:
            loss.backward()


def gradient_of(model, p):
    """The gradient a parameter received: its own ``.grad``, or its slice of the fused flat gradient; None if neither."""
    fused = getattr(model, "fused_link_params", None)
    if fused is not None and fused.flat.grad is not None:
        start = (p.data_ptr() - fused.flat.data_ptr()) // 4
        if 0 <= start <= fused.flat.numel() - p.numel() and p.data_ptr() >= fused.flat.data_ptr():
            assert p.grad is None
            return fused.flat.grad[start:start + p.numel()].view(p.shape)
    return p.grad


def check_gradients(model, mods, want, frozen, what, atol_scale=2e-5):
    mine = {id(p) for mod in mods for p in mod.parameters()}
    fused = getattr(model, "fused_link_params", None)
    assert {id(p) for p in model.parameters() if fused is None or p is not fused.flat} == mine, "a parameter the set does not know"
    scale = max([float(g.abs().max()) for d in want for g in d.values()])
    for k, (mod, grads) in enumerate(zip(mods, want)):
        for name, p in mod.named_parameters():
            got, tag = gradient_of(model, p), f"{what}: entry {k} {name}"
            if k in frozen:
                assert got is None, f"{tag}: a frozen parameter received a gradient"
                continue
            if got is None:                               # never entered a graph: only right where nothing depends on it
                assert float(grads[name].abs().max()) == 0.0, f"{tag}: no gradient, want {grads[name]}"
                continue
            assert_close(got.cpu().numpy(), grads[name].reshape(p.shape).numpy(), rtol=1e-4, atol=atol_scale * scale, what=tag)


def new_model(robot_name, directory):
    return drm.DifferentiableRobotModel(robot_file(robot_name, directory), robot_name, device=DEV)


# ------------------------------------------------------------------------------------------------
# the grid
# ------------------------------------------------------------------------------------------------
def _cases():
    out = []
    # every entry point with kinematic and inertial parameters learnable together: the chain, the hand and the synthetic
    # family take all of them, the deep and folded robots the core ones
    # (the rollout on the chain and the synthetic tree only: these joint forces on the hand's gram-scale fingers leave the
    # fp64 reference gradients of a rollout non-finite)
    hand = tuple(e for e in ENTRY_ALL if e != "rollout")
    for robot, entries in (("iiwa7", ENTRY_ALL), ("allegro_hand_description_left", hand), (SYNTHETIC, ENTRY_ALL),
                           ("iiwa7_allegro", ENTRY_CORE), ("fetch_arm_no_gripper", ENTRY_CORE), ("trifinger_edu", ENTRY_CORE)):
        out += [(robot, "both", e, SMALL) for e in entries]
    sets = {"inertial": ("iiwa7", "fetch_arm_no_gripper", "allegro_hand_description_left"),
            "kinematic": ("iiwa7", "trifinger_edu", "iiwa7_allegro"),
            "fixed_origin": ("iiwa7", "fetch_arm_no_gripper", SYNTHETIC),
            "nets": ("iiwa7", "allegro_hand_description_left"),
            "tied2": ("iiwa7", "trifinger_edu"),
            "tied4": ("allegro_hand_description_left", "iiwa7_allegro", SYNTHETIC),
            "frozen": ("iiwa7", "allegro_hand_description_left")}
    for set_name, robots in sets.items():
        for robot in robots:
            # kinematics do not depend on an inertial-only set (see test_inertial_only_set_builds_no_graph_for_kinematics)
            last = "mass_matrix" if set_name == "inertial" else "fk_multi"
            out += [(robot, set_name, e, RAGGED) for e in ("id_gd", "forward_dynamics", "combined", last)]
    # the persistent multi-tile adjoints, chain and tree: the full adjoint, the inertial single sweep and the FK adjoint
    for robot in ("iiwa7", "allegro_hand_description_left"):
        out += [(robot, "both", "id_gd", LARGE), (robot, "inertial", "id_gd", LARGE), (robot, "kinematic", "fk", LARGE)]
    return out


CASES = _cases()


def _paths(set_name, entry):
    paths = PATHS if set_name != "nets" else PATHS[:2]               # the inertia nets cannot be fused
    return [p for p in paths if not (entry == "two_backwards" and p == "shared")]     # separate graphs: no shared table


@pytest.mark.parametrize("robot_name,set_name,entry,batch,path",
                         [c + (p,) for c in CASES for p in _paths(c[1], c[2])],
                         ids=lambda v: str(v))
def test_parameter_gradients_match_fp64_oracle(robot_name, set_name, entry, batch, path, model_dir):
    learnables, frozen, want = reference(robot_name, set_name, entry, batch, model_dir)
    model = new_model(robot_name, model_dir)
    mods = install(model, learnables, frozen)
    n_values = sum(p.numel() for p in model.parameters() if p.requires_grad)
    if path == "fused":
        flat = model.fuse_learnable_parameters()
        assert flat.numel() == n_values                                # tied modules once, frozen modules not at all
    x = cast(inputs(oracle_robot(robot_name, model_dir), batch), device=DEV)
    run_model(model, entry, x, path)
    check_gradients(model, mods, want, frozen, f"{robot_name} {set_name} {entry} {path}")


@pytest.mark.parametrize("robot_name,set_name,entry,batch",
                         [c for c in CASES if c[1] != "nets" and c[2] in ("id_gd", "combined", "fk_multi", "mass_matrix", "rollout")],
                         ids=lambda v: str(v))
def test_fused_gradients_equal_per_module_gradients(robot_name, set_name, entry, batch, model_dir):
    """The fused and the per-module table are bit-identical before the first step, so their gradients differ by the
    rounding of the table adjoint's sums only (tolerance of test_fused_params_gpu.py, step 0)."""
    robot = oracle_robot(robot_name, model_dir)
    learnables, frozen = make_set(robot, set_name)
    x = cast(inputs(robot, batch), device=DEV)
    plain, fused = new_model(robot_name, model_dir), new_model(robot_name, model_dir)
    mods_p, mods_f = install(plain, learnables, frozen), install(fused, learnables, frozen)
    fused.fuse_learnable_parameters()
    assert torch.equal(plain._link_table().detach(), fused._link_table().detach())
    run_model(plain, entry, x, "per_module")
    run_model(fused, entry, x, "fused")
    for k, (mp, mf) in enumerate(zip(mods_p, mods_f)):
        for (name, pp), (_, pf) in zip(mp.named_parameters(), mf.named_parameters()):
            want, got = gradient_of(plain, pp), gradient_of(fused, pf)
            if k in frozen:
                assert want is None and got is None
                continue
            want = torch.zeros_like(got) if want is None else want           # a fixed-joint origin: no graph vs zero
            assert_close(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-5, atol=1e-6 * max(1.0, float(want.abs().max())),
                         what=f"{robot_name} {set_name} {entry}: entry {k} {name}")


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("robot_name", ["iiwa7", "allegro_hand_description_left"])
def test_inertial_only_set_builds_no_graph_for_kinematics(robot_name, path, model_dir):
    """Kinematics read the F / r columns only: with nothing but inertial parameters learnable, FK and the Jacobian return
    the constant model's values bit for bit, carry no graph and leave every gradient None."""
    robot = oracle_robot(robot_name, model_dir)
    learnables, _ = make_set(robot, "inertial")
    const, model = new_model(robot_name, model_dir), new_model(robot_name, model_dir)
    install(model, learnables)
    if path == "fused":
        model.fuse_learnable_parameters()
    x = cast(inputs(robot, SMALL), device=DEV)

    def outputs(m):
        return m.compute_forward_kinematics(x["q"], x["ee"]) + m.compute_endeffector_jacobian(x["q"], x["ee"]) \
            + m.compute_fk_and_jacobian(x["q"], x["ee"])

    if path == "shared":
        with model.shared_link_table():
            got = outputs(model)
    else:
        got = outputs(model)
    for a, b in zip(got, outputs(const)):
        assert not a.requires_grad and torch.equal(a, b)
    assert all(p.grad is None for p in model.parameters())


# ------------------------------------------------------------------------------------------------
# state transitions of one model (host logic: which table is cached, which adjoint runs)
# ------------------------------------------------------------------------------------------------
def test_learnable_state_transitions_leave_no_stale_table_or_gradient(model_dir):
    robot = oracle_robot("iiwa7", model_dir)
    learnables, _ = make_set(robot, "both", spread=0.0)       # every module starts at its URDF value (l * l: to one rounding)
    kin = [k for k, l in enumerate(learnables) if l.pname in ("trans", "rot_angles")]
    x, x64 = cast(inputs(robot, SMALL), device=DEV), cast(inputs(robot, SMALL), dtype=torch.float64)
    const, model = new_model("iiwa7", model_dir), new_model("iiwa7", model_dir)

    def values(m):
        return (m.compute_inverse_dynamics(x["q"], x["qd"], x["qdd"]),) + tuple(m.compute_forward_kinematics(x["q"], x["ee"])) \
            + (m.compute_lagrangian_inertia_matrix(x["q"]), m.compute_forward_dynamics(x["q"], x["qd"], x["f"]))

    def step(what, frozen=()):
        for p in model.parameters():
            p.grad = None
        run_model(model, "combined", x, "per_module")
        protos = [Learnable(l.links, l.pname, mod) for l, mod in zip(learnables, mods)]       # the modules' current values
        learned, leaves = learnable_robot(robot, protos)
        want = gradients(sum(fn(OracleApi(learned), x64) for fn in ENTRY["combined"]) / SMALL, leaves)
        check_gradients(model, mods, want, frozen, what)

    # a constant model is called first (table, folded table and the learnable flag are cached), then becomes learnable
    before = values(model)
    assert model._table_cache is not None and model._has_learnable is False
    mods = install(model, learnables)
    assert model._kinematic_params_learnable()
    after = values(model)
    assert all(t.requires_grad for t in after)
    step("made learnable after a constant call")
    # freeze every kinematic module: the inertial gradients stay right, the frozen modules get none
    for k in kin:
        model.freeze_learnable_link_param(learnables[k].links[0], learnables[k].pname)
    assert not model._kinematic_params_learnable()
    step("kinematic modules frozen", frozen=kin)
    for k in kin:
        model.unfreeze_learnable_link_param(learnables[k].links[0], learnables[k].pname)
    assert model._kinematic_params_learnable()
    step("kinematic modules unfrozen")
    # nothing requires grad: the constant model's values, no graph
    for p in model.parameters():
        p.requires_grad_(False)
    for got, want_, first in zip(values(model), values(const), before):
        assert not got.requires_grad
        # the constant model folds its fixed link into the table once, this one per CTA: the same sums in another order,
        # which forward dynamics divides by the articulated inertia
        assert_close(got.cpu().numpy(), want_.cpu().numpy(), rtol=1e-5, atol=2e-5 * float(want_.abs().max()), what="all frozen")
        assert torch.equal(first, want_)
    # an in-place edit is seen by the next call
    for p in model.parameters():
        p.requires_grad_(True)
    with torch.no_grad():
        mods[0].l.data.copy_(mods[0].l.data * 1.5)                      # the first link's mass
        mods[kin[0]].param.data.copy_(mods[kin[0]].param.data + 0.05)
    edited = values(model)
    assert not torch.equal(edited[0], after[0]) and not torch.equal(edited[1], after[1])
    step("after in-place edits")


def test_freezing_and_the_fused_path(model_dir):
    """A module frozen before fusing is a constant of the fused table: no optimiser step moves it -- not even one that
    moves parameters whose gradient is zero (weight decay) -- and freezing or unfreezing after fusing raises instead of
    silently doing nothing."""
    robot = oracle_robot("iiwa7", model_dir)
    learnables, frozen = make_set(robot, "frozen")
    model = new_model("iiwa7", model_dir)
    mods = install(model, learnables, frozen)
    held = {k: [p.detach().clone() for p in mods[k].parameters()] for k in frozen}
    flat = model.fuse_learnable_parameters()
    x = cast(inputs(robot, SMALL), device=DEV)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2, weight_decay=0.1)
    start = flat.detach().clone()
    for _ in range(2):
        opt.zero_grad()
        run_model(model, "combined", x, "fused")
        opt.step()
    assert not torch.equal(flat.detach(), start)
    for k, was in held.items():
        for p, w in zip(mods[k].parameters(), was):
            assert torch.equal(p.detach(), w) and p.grad is None
    link, pname = learnables[frozen[0]].links[0], learnables[frozen[0]].pname
    with pytest.raises(RuntimeError, match="after fuse"):
        model.unfreeze_learnable_link_param(link, pname)
    with pytest.raises(RuntimeError, match="after fuse"):
        model.freeze_learnable_link_param(learnables[0].links[0], learnables[0].pname)
    with pytest.raises(RuntimeError, match="already fused"):
        model.fuse_learnable_parameters()
