"""
Model compiler: per-link host objects -> flat tables for the CUDA kernels
==========================================================================
Two products (SURVEY.md Appendix A; layout documented in ``include/drm_b200.h``):

* ``Topology`` -- immutable integers (parent index, joint-axis code, DoF column per link), resolved
  ONCE at model construction.  The reference re-resolves parents by *name* with an O(#joints) scan
  inside every per-link loop (``robot_model.py:176,264,297,563,606,664``).
* ``build_link_table`` -- the differentiable float table ``[n_links, 28]`` on the model's device,
  built with ordinary (batched) torch ops from whatever the six per-link parameter callables
  return, so autograd carries the kernels' ``d table`` back to any user parametrisation module
  (``robot_model.py:682-689``).  Contents per link: ``F = Rz(yaw) Ry(pitch) Rx(roll)``
  (``rigid_body.py:138-143``), ``r = trans``, ``I_o = I_c + m S(c) S(c)^T`` and ``mc = m c``
  (``spatial_vector_algebra.py:323-327``; ``inertia_mat`` is used as given, NOT symmetrised),
  ``m``, ``damping``.  The reference recomputes all of these for every link on every call.
"""
import ctypes

import torch

MAX_LINKS = 64        # DRMB200_MAX_LINKS
TABLE_STRIDE = 28     # DRMB200_TABLE_STRIDE


class Topology(ctypes.Structure):
    """ctypes mirror of ``drmb200_topology_t`` (include/drm_b200.h)."""

    _fields_ = [
        ("n_links", ctypes.c_int32),
        ("n_dofs", ctypes.c_int32),
        ("parent", ctypes.c_int8 * MAX_LINKS),
        ("axis", ctypes.c_int8 * MAX_LINKS),
        ("dof", ctypes.c_int8 * MAX_LINKS),
    ]


def axis_code(joint_axis, joint_name=""):
    """Signed axis code (+-1/+-2/+-3 = +-x/+-y/+-z) of a movable joint.

    The reference dispatches on ``|axis[k]| == 1`` (``rigid_body.py:149-154``) and is inconsistent for
    anything else (FK silently falls through to z, inverse dynamics raises, ``robot_model.py:357``);
    every shipped URDF uses signed coordinate axes, so anything else is rejected here.
    """
    a = [float(x) for x in joint_axis.reshape(-1).tolist()]
    nz = [k for k in range(3) if a[k] != 0.0]
    if len(nz) != 1 or abs(a[nz[0]]) != 1.0:
        raise ValueError(
            f"joint {joint_name!r}: axis {a} is not a signed coordinate axis; only +-x / +-y / +-z "
            "joint axes are supported (the reference is inconsistent for other axes)"
        )
    k = nz[0]
    return (k + 1) if a[k] > 0 else -(k + 1)


def compile_topology(bodies, parent_idx):
    n_links = len(bodies)
    if n_links > MAX_LINKS:
        raise ValueError(f"{n_links} links exceed the engine limit of {MAX_LINKS}")
    topo = Topology()
    topo.n_links = n_links
    n_dofs = 0
    for i, body in enumerate(bodies):
        p = parent_idx[i]
        if i == 0:
            p = -1
        elif not (0 <= p < i):
            raise ValueError(
                f"link {body.name!r} (index {i}) has parent index {p}: links must be listed parents-first "
                "(true for every shipped URDF; the reference assumes link 0 is the root)"
            )
        topo.parent[i] = p
        if body.joint_idx is not None:
            topo.axis[i] = axis_code(body.joint_axis, body.name)
            topo.dof[i] = body.joint_idx
            n_dofs += 1
        else:
            topo.axis[i] = 0
            topo.dof[i] = -1
    topo.n_dofs = n_dofs
    return topo


def _rpy_to_matrix(rpy):
    """Batched ``Rz(yaw) @ Ry(pitch) @ Rx(roll)`` for rpy ``[N,3]`` (rigid_body.py:138-143)."""
    cr, sr = torch.cos(rpy[:, 0]), torch.sin(rpy[:, 0])
    cp, sp = torch.cos(rpy[:, 1]), torch.sin(rpy[:, 1])
    cy, sy = torch.cos(rpy[:, 2]), torch.sin(rpy[:, 2])
    rows = [
        cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr,
        sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr,
        -sp, cp * sr, cp * cr,
    ]
    return torch.stack(rows, dim=1)          # [N, 9] row-major


RAW_STRIDE = 20       # DRMB200_RAW_STRIDE
# (owner attribute, parameter name, offset in the raw row, size); trans / rot_angles / damping of FIXED joints are
# frozen at their construction-time values (reference quirk, rigid_body.py:64-67)
_RAW_FIELDS = (("body", "rot_angles", 0, 3), ("body", "trans", 3, 3), ("inertia", "mass", 6, 1),
               ("inertia", "com", 7, 3), ("inertia", "inertia_mat", 10, 9), ("body", "joint_damping", 19, 1))


def _raw_layout(bodies, device):
    """Constant part of the raw block + where the learnable modules' outputs go.  Link parameters that are plain
    constants (lambdas over the URDF tensors) are evaluated once; only ``torch.nn.Module`` parametrisations are
    re-evaluated per call.  Cached per (ModuleList, set of learnable modules)."""
    f32 = dict(dtype=torch.float32, device=device)
    learnable, const_rows = [], []
    for i, body in enumerate(bodies):
        movable = body.joint_idx is not None
        row = torch.zeros(RAW_STRIDE, **f32)
        for owner_name, pname, off, size in _RAW_FIELDS:
            owner = body if owner_name == "body" else body.inertia
            if owner_name == "body" and not movable:
                if pname == "rot_angles":
                    row[off:off + size] = body._ctor_rot_angles.reshape(3).to(**f32)
                elif pname == "trans":
                    row[off:off + size] = body._ctor_trans.reshape(3).to(**f32)
                continue                                      # damping of a fixed joint stays 0
            attr = getattr(owner, pname)
            if isinstance(attr, torch.nn.Module):
                learnable.append((attr, i * RAW_STRIDE + off, size))
            else:
                val = attr()
                if val is not None:
                    row[off:off + size] = val.detach().reshape(size).to(**f32)
        const_rows.append(row)
    const = torch.stack(const_rows).reshape(-1)
    index = torch.tensor([o + k for _, o, s in learnable for k in range(s)], dtype=torch.long, device=device)
    return const, learnable, index


def gather_raw_parameters(bodies, device):
    """``[n_links, 20]`` = rpy(3) | trans(3) | mass | com(3) | inertia_mat(9) | damping per link, differentiable
    w.r.t. the learnable parametrisation modules: one ``torch.cat`` of their outputs + one ``index_copy`` into the
    cached constant block (two launches, independent of the number of links)."""
    sig = (str(device),) + tuple(id(getattr(b if o == "body" else b.inertia, p)) for b in bodies for o, p, _, _ in _RAW_FIELDS)
    cached = getattr(bodies, "_drm_gather_cache", None)
    if cached is None or cached[0] != sig:
        cached = (sig,) + _raw_layout(bodies, device)
        object.__setattr__(bodies, "_drm_gather_cache", cached)        # plain attribute on the ModuleList
    _, const, learnable, index = cached
    if not learnable:
        return const.reshape(len(bodies), RAW_STRIDE)
    vals = torch.cat([m().reshape(s).to(dtype=torch.float32, device=device) for m, _, s in learnable])
    return const.index_copy(0, index, vals).reshape(len(bodies), RAW_STRIDE)


class FusedLinkParameters(torch.nn.Module):
    """All learnable link parameters of a model in ONE flat ``nn.Parameter`` (BASELINE config 5: 21 modules -> one
    tensor, one table-build launch, one AccumulateGrad node, one fused optimiser launch).

    Built by ``DifferentiableRobotModel.fuse_learnable_parameters()`` from the parametrisation modules that are
    installed at that moment.  Supported: ``UnconstrainedScalar`` / ``UnconstrainedTensor`` (identity) and
    ``PositiveScalar`` (``l^2 + min_val``) -- the ones the reference's examples use
    (``examples/learn_dynamics_iiwa.py:57-65``); anything else raises and the model stays on the per-module path.
    The modules' own Parameters are re-pointed at slices of the flat storage, so ``print_learnable_params`` /
    ``state_dict`` keep showing the live values; only the flat vector receives gradients.

    * Tied parameters: a module installed on several links owns ONE slice of ``flat`` that every one of its raw entries
      reads; its gradient is the sum over those entries, as autograd gives on the per-module path.  So
      ``flat.numel()`` is the number of parameter values that required grad before fusing.
    * Frozen modules (no parameter requires grad when fusing, ``freeze_learnable_link_param``): their current output is
      written into the constant block and they stay out of ``flat`` -- no gradient, no optimiser update, whatever the
      optimiser does with zero gradients.  The value is fixed from then on; freezing is decided before fusing."""

    def __init__(self, bodies, device):
        super().__init__()
        from .rigid_body_params import PositiveScalar, UnconstrainedScalar, UnconstrainedTensor
        const, learnable, _ = _raw_layout(bodies, device)
        n_raw = const.numel()
        src = torch.full((n_raw,), -1, dtype=torch.int32)
        kind = torch.zeros(n_raw, dtype=torch.int32)
        off = torch.zeros(n_raw, dtype=torch.float32)
        chunks, owners, cursor = [], {}, 0                # owners: id(param) -> (param, start of its slice of flat)

        def claim(param, size, module):
            nonlocal cursor
            if param.numel() != size:
                raise ValueError(f"{type(module).__name__}: {param.numel()} values for a link parameter of {size}")
            if id(param) not in owners:                   # a tied module is claimed once, by its first link
                chunks.append(param.detach().reshape(-1).to(dtype=torch.float32, device=device))
                owners[id(param)] = (param, cursor)
                cursor += size
            return owners[id(param)][1]

        def frozen(module):
            return not any(p_.requires_grad for p_ in module.parameters())

        seen = set()
        for module, raw_offset, size in learnable:
            seen.add(id(module))
            if frozen(module):
                with torch.no_grad():
                    const[raw_offset:raw_offset + size] = module().reshape(size).to(dtype=torch.float32, device=device)
                continue
            if isinstance(module, PositiveScalar):
                param, k, o = module.l, 1, float(module._min_val)
            elif isinstance(module, (UnconstrainedScalar, UnconstrainedTensor)):
                param, k, o = module.param, 0, 0.0
            else:
                raise ValueError(f"cannot fuse a {type(module).__name__} parametrisation (supported: UnconstrainedScalar, "
                                 "UnconstrainedTensor, PositiveScalar); the model keeps evaluating its modules one by one")
            start = claim(param, size, module)
            src[raw_offset:raw_offset + size] = torch.arange(start, start + size, dtype=torch.int32)
            kind[raw_offset:raw_offset + size] = k
            off[raw_offset:raw_offset + size] = o
        # modules on fixed-joint origins feed nothing (reference quirk, rigid_body.py:64-67) but stay parameters
        for body in bodies:
            for owner, names in ((body, ("trans", "rot_angles", "joint_damping")), (body.inertia, ("mass", "com", "inertia_mat"))):
                for name in names:
                    module = getattr(owner, name)
                    if isinstance(module, torch.nn.Module) and id(module) not in seen:
                        for p_ in module.parameters():
                            if p_.requires_grad:
                                claim(p_, p_.numel(), module)
        # the inverse of src for the backward: per flat entry, the list of the raw entries that read it, ascending
        first_reader = torch.full((cursor,), -1, dtype=torch.int32)
        next_reader = torch.full((n_raw,), -1, dtype=torch.int32)
        for k in reversed(torch.nonzero(src >= 0).flatten().tolist()):
            next_reader[k] = first_reader[src[k]]
            first_reader[src[k]] = k
        # does `flat` feed a joint origin (rpy | trans of a movable link)?  If not, kinematics need no parameter gradient
        self.feeds_kinematics = bool((src.reshape(-1, RAW_STRIDE)[:, :6] >= 0).any())
        self.flat = torch.nn.Parameter(torch.cat(chunks) if chunks else torch.zeros(0, device=device))
        self.register_buffer("const_raw", const.reshape(len(bodies), RAW_STRIDE).contiguous(), persistent=False)
        self.register_buffer("src", src.to(device), persistent=False)
        self.register_buffer("kind", kind.to(device), persistent=False)
        self.register_buffer("off", off.to(device), persistent=False)
        self.register_buffer("first_reader", first_reader.to(device), persistent=False)
        self.register_buffer("next_reader", next_reader.to(device), persistent=False)
        for param, start in owners.values():             # the modules' Parameters become views of the flat storage
            param.data = self.flat.data[start:start + param.numel()].view(param.shape)
            param.requires_grad_(False)                   # gradients (and optimiser updates) go through `flat` only

    def table(self):
        from . import engine
        return engine.FusedTableFunction.apply(self.flat, self.const_raw, self.src, self.kind, self.off, self.first_reader,
                                               self.next_reader)


def build_link_table(bodies, device):
    """Evaluate every link's parameter callables into the ``[n_links, 28]`` fp32 device table.

    On a CUDA device: one ``torch.cat`` + one kernel (``engine.BuildLinkTableFunction`` -> ``csrc/table.cu``), with an
    analytic backward kernel.  On the CPU (host-side introspection / tests only; compute entry points refuse CPU
    tensors) the same table is assembled with batched torch ops below."""
    if torch.device(device).type == "cuda":
        from . import engine
        return engine.BuildLinkTableFunction.apply(gather_raw_parameters(bodies, device))
    f32 = dict(dtype=torch.float32, device=device)
    trans, rpy, mass, com, inertia, damping = [], [], [], [], [], []
    for i, body in enumerate(bodies):
        movable = body.joint_idx is not None
        # fixed joints keep their construction-time origin (reference quirk, rigid_body.py:64-67)
        trans.append((body.trans() if movable else body._ctor_trans).reshape(3))
        rpy.append((body.rot_angles() if movable else body._ctor_rot_angles).reshape(3))
        m, c, inert = body.inertia._get_parameter_values()
        mass.append(m.reshape(()))
        com.append(c.reshape(3))
        inertia.append(inert.reshape(9))
        d = body.joint_damping() if movable else None
        damping.append(d.reshape(()) if d is not None else torch.zeros((), **f32))
    trans = torch.stack(trans).to(**f32)
    rpy = torch.stack(rpy).to(**f32)
    mass = torch.stack(mass).to(**f32)
    com = torch.stack(com).to(**f32)
    inertia = torch.stack(inertia).to(**f32)
    damping = torch.stack(damping).to(**f32)

    F = _rpy_to_matrix(rpy)
    cx, cy, cz = com[:, 0], com[:, 1], com[:, 2]
    # S(c) S(c)^T = |c|^2 I - c c^T
    ssT = torch.stack(
        [cy * cy + cz * cz, -cx * cy, -cx * cz,
         -cx * cy, cx * cx + cz * cz, -cy * cz,
         -cx * cz, -cy * cz, cx * cx + cy * cy], dim=1)
    Io = inertia + mass[:, None] * ssT
    mc = mass[:, None] * com
    pad = torch.zeros((len(bodies), 2), **f32)
    table = torch.cat([F, trans, Io, mc, mass[:, None], damping[:, None], pad], dim=1)
    assert table.shape == (len(bodies), TABLE_STRIDE)
    return table.contiguous()
