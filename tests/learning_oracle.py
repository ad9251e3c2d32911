"""fp64 parameter gradients of the oracle (oracle/drm_oracle.py), for the parameter-learning tests.

Test helper module (not a conftest): imported by test_learning_paths_gpu.py.  A learnable set is a list of
``Learnable(links, pname, module)``: one parametrisation module (``rigid_body_params``) installed as ``pname`` of every
link in ``links`` (more than one link = tied parameters).  ``learnable_robot`` returns an oracle ``Robot`` whose ``rpy``,
``trans``, ``mass``, ``com``, ``inertia`` and ``damping`` rows are float64 functions of leaf tensors, one leaf per
``nn.Parameter`` of every module; ``O.forward_kinematics``, ``O.jacobian``, ``O.kinematic_state``, ``O.inverse_dynamics``,
``O.forward_dynamics`` and the rollout oracle then give the parameter gradients by plain autograd.  ``O.load_robot``
derives nothing from these fields (every oracle function reads them on each call), so replacing the six tensors is enough.

* The three fusible parametrisations are restated here: UnconstrainedScalar and UnconstrainedTensor are the identity,
  PositiveScalar is ``l * l + min_val``.  The inertia nets are the ``rigid_body_params`` classes evaluated in double
  precision (a deep copy with float64 parameters); test_params.py pins those classes to the reference's golden vectors.
* Reference quirk kept: ``trans``, ``rot_angles`` and ``joint_damping`` of a link behind a FIXED joint are frozen at their
  construction-time values, so a module installed there feeds nothing and its leaves get an exactly zero gradient.
* Orientation: the reference's quaternion autograd treats ``0.5 / sqrt(t)`` as a constant while the kernels use the exact
  derivative.  The losses of the tests use the oracle's ``O.quaternion``, which is differentiated exactly, and only
  through even functions of the quaternion (``q_i q_j``), which are the same on every branch and for either sign.
"""
import copy
from typing import Dict, List, NamedTuple, Tuple

import torch

from differentiable_robot_model_b200.rigid_body_params import PositiveScalar, UnconstrainedScalar, UnconstrainedTensor
from oracle import drm_oracle as O

# parameter name -> (Robot field, shape of one link's row); the first three belong to the joint and are frozen on fixed links
FIELDS = {"rot_angles": ("rpy", (3,)), "trans": ("trans", (3,)), "joint_damping": ("damping", ()),
          "mass": ("mass", ()), "com": ("com", (3,)), "inertia_mat": ("inertia", (3, 3))}
JOINT_PARAMS = ("rot_angles", "trans", "joint_damping")


class Learnable(NamedTuple):
    links: Tuple[str, ...]
    pname: str
    module: torch.nn.Module


def _evaluate(module):
    """(value, {parameter name: float64 leaf}) of one parametrisation module at its current parameter values."""
    def leaf(p):
        return p.detach().cpu().double().clone().requires_grad_(True)

    if isinstance(module, PositiveScalar):
        l = leaf(module.l)
        return l * l + module._min_val, {"l": l}
    if isinstance(module, (UnconstrainedScalar, UnconstrainedTensor)):
        param = leaf(module.param)
        return param, {"param": param}
    twin = copy.deepcopy(module).cpu().double()
    return twin(), dict(twin.named_parameters())


def learnable_robot(robot, learnables: List[Learnable]):
    """``(robot', leaves)``: the float64 oracle robot with the learnable set applied, and per entry of ``learnables`` the
    dict ``{parameter name: leaf}`` (names as in ``module.named_parameters()``)."""
    assert robot.trans.dtype == torch.float64
    rows = {field: [getattr(robot, field)[i] for i in range(len(robot.names))] for field, _ in FIELDS.values()}
    leaves = []
    for links, pname, module in learnables:
        value, module_leaves = _evaluate(module)
        leaves.append(module_leaves)
        field, shape = FIELDS[pname]
        for link in links:
            i = robot.index(link)
            if pname in JOINT_PARAMS and robot.dof[i] < 0:
                continue                                          # fixed joint: the construction-time value stays
            rows[field][i] = value.reshape(shape)
    fields = {field: torch.stack(r) for field, r in rows.items()}
    out = O.Robot(robot.names, robot.parent, robot.dof, robot.joint_type, robot.limits, axis=robot.axis,
                  n_dofs=robot.n_dofs, controlled=robot.controlled, **fields)
    return out, leaves


def gradients(loss, leaves: List[Dict[str, torch.Tensor]]) -> List[Dict[str, torch.Tensor]]:
    """d loss / d leaf in the structure of ``leaves``; a leaf the loss does not depend on gets zeros."""
    flat = [t for d in leaves for t in d.values()]
    grads = torch.autograd.grad(loss, flat, allow_unused=True) if loss.requires_grad else [None] * len(flat)
    it = iter(grads)
    return [{name: (torch.zeros_like(t) if g is None else g) for (name, t), g in zip(d.items(), it)} for d in leaves]
