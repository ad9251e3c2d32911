"""
Differentiable robot model -- CUDA engine behind the reference's API
=====================================================================
Drop-in for ``differentiable_robot_model.robot_model`` (reference ``robot_model.py``): same class and
wrapper names, constructor, method names, keyword arguments, return-tuple order, squeeze behaviour
for 1-D inputs and exception types.  The difference is *where the arithmetic happens*: the
reference walks a Python list of per-link ``nn.Module``s issuing dozens of tiny ``[B,3,3]`` torch ops
per link (``robot_model.py:173-193, 262-301``); here a call is

    argument checks -> link table (cached, or rebuilt differentiably when parameters are learnable)
    -> ONE hand-written sm_90a kernel through the C ABI (``engine.py`` / ``include/drm_b200.h``)

on the caller's current CUDA stream, with analytic backward kernels registered through
``torch.autograd.Function`` so the parameter-learning examples still train.

Deliberate deviations from the reference (see DESIGN.md):
  * compute entry points need a CUDA model and CUDA fp32 tensors -- there is no CPU path;
  * per-body state ``_bodies[i].pose / vel`` is refreshed only by ``update_kinematic_state`` (one
    all-links launch), not as a side effect of every call; ``acc / force`` are not materialised
    (the fused kernels write nothing per link to HBM);
  * ``recursive=True`` FK returns the same (correct) result as the non-recursive path; the
    reference's recursive variant depends on stale per-body state (``rigid_body.py:119``);
  * joint axes must be signed coordinate axes (true for every shipped URDF).
"""
import contextlib
import os
import weakref
from dataclasses import dataclass
from typing import Dict, List, NamedTuple, Optional, Tuple, Union

import torch

from . import engine
from .link_table import FusedLinkParameters, build_link_table, compile_topology
from .rigid_body import DifferentiableRigidBody
from .urdf_utils import URDFRobotModel

robot_description_folder = os.path.join(os.path.dirname(os.path.abspath(__file__)), "robot_data")


def tensor_check(function):
    """Argument validation with the semantics of the reference decorator (``robot_model.py:25-84``):
    every Tensor argument must live on the model's device type, have ndim 1 or 2 and share the batch
    shape of the first one; 1-D inputs are promoted to ``[1, n]`` and Tensor outputs squeezed back.
    Violations raise ``AssertionError`` like the reference's ``assert``s."""

    @dataclass
    class BatchInfo:
        shape: torch.Size = torch.Size([])
        init: bool = False

    def pre(arg, model, info):
        if type(arg) is not torch.Tensor:
            return arg
        assert arg.device.type == model._device.type, f"Input argument of different device as module: {arg}"
        assert arg.ndim in (1, 2), "Input tensors must have ndim of 1 or 2."
        if info.init:
            assert info.shape == arg.shape[:-1], "Batch size mismatch between input tensors."
        else:
            info.init, info.shape = True, arg.shape[:-1]
        return arg.unsqueeze(0) if len(info.shape) == 0 else arg

    def post(ret, info):
        if type(ret) is torch.Tensor and info.init and len(info.shape) == 0:
            return ret[0, ...]
        return ret

    def wrapper(self, *args, **kwargs):
        info = BatchInfo()
        args = [pre(a, self, info) for a in args]
        kwargs = {k: pre(v, self, info) for k, v in kwargs.items()}
        ret = function(self, *args, **kwargs)
        if type(ret) is torch.Tensor:
            return post(ret, info)
        if type(ret) is tuple:
            return tuple(post(r, info) for r in ret)
        return ret

    wrapper.__name__ = function.__name__
    wrapper.__doc__ = function.__doc__
    return wrapper


class InverseKinematicsResult(NamedTuple):
    """What :meth:`DifferentiableRobotModel.compute_inverse_kinematics` returns, per row: the joint angles, the position
    and orientation errors at them (metres / radians; orientation 0 for position-only solves), whether both are within
    tolerance, and the final Levenberg-Marquardt damping (pass it back as ``damping`` to continue a solve).
    :meth:`DifferentiableRobotModel.compute_inverse_kinematics_multi` returns the same with the errors per link,
    [n_links x batch_size]."""
    q: torch.Tensor
    pos_error: torch.Tensor
    rot_error: torch.Tensor
    converged: torch.Tensor
    damping: torch.Tensor


class OperationalSpaceDynamics(NamedTuple):
    """What :meth:`DifferentiableRobotModel.compute_operational_space_dynamics` returns, per row, with M = 6 rows per link
    (linear over angular) or 3 for position only, links stacked in the order requested: the inverse operational-space
    inertia ``J G J^T`` [M x M], the true world-frame acceleration ``J qdd + Jdot qd`` [M], the velocity ``J qd`` [M] and
    the bias acceleration ``Jdot qd`` [M]."""
    inv_inertia: torch.Tensor
    acceleration: torch.Tensor
    velocity: torch.Tensor
    bias_acceleration: torch.Tensor


class ContactDynamics(NamedTuple):
    """What :meth:`DifferentiableRobotModel.compute_contact_dynamics` returns, per row: the joint accelerations under the
    contacts [n_dofs], the contact forces ``lambda`` [M] (world frame, at each link origin; 6 per link, force over torque, or
    3 for position only, links stacked in the order requested) and whether the row's contact system was solved (bool; an
    unsolved row has NaN in both)."""
    qdd: torch.Tensor
    force: torch.Tensor
    solved: torch.Tensor


class ContactImpulse(NamedTuple):
    """What :meth:`DifferentiableRobotModel.compute_contact_impulse` returns, per row: the joint velocities just after the
    impact [n_dofs], the contact impulses ``Lambda`` [M] (laid out like :class:`ContactDynamics`'s force) and whether the
    row's contact system was solved."""
    qd_plus: torch.Tensor
    impulse: torch.Tensor
    solved: torch.Tensor


class EnergyAndMomentum(NamedTuple):
    """What :meth:`DifferentiableRobotModel.compute_energy_and_momentum` returns, per row: the kinetic and potential energy
    [J], the generalized momentum ``H(q) qd`` [n_dofs], the centre of mass [3] and its velocity [3] in the world frame, and
    the CoM Jacobian [3 x n_dofs].  The three velocity-dependent fields are None when no ``qd`` was given."""
    kinetic_energy: Optional[torch.Tensor]
    potential_energy: torch.Tensor
    momentum: Optional[torch.Tensor]
    com: torch.Tensor
    com_velocity: Optional[torch.Tensor]
    com_jacobian: torch.Tensor


class ControlledRollout(NamedTuple):
    """What :meth:`DifferentiableRobotModel.compute_pd_controlled_rollout` returns, time-major [T x batch_size x n_dofs]
    (or [T x n_dofs]): the joint angles, velocities and accelerations after each step (as
    :meth:`DifferentiableRobotModel.compute_forward_dynamics_rollout`) and the joint torques the controller applied."""
    q: torch.Tensor
    qd: torch.Tensor
    qdd: torch.Tensor
    tau: torch.Tensor


class ContactRollout(NamedTuple):
    """What :meth:`DifferentiableRobotModel.compute_contact_rollout` returns, time-major: the joint angles, velocities and
    accelerations after each step [T x batch_size x n_dofs] (as :meth:`DifferentiableRobotModel.compute_forward_dynamics_rollout`),
    the contact forces of each step [T x batch_size x M] (laid out like :class:`ContactDynamics`'s force) and whether every
    step of the row was solved [batch_size]."""
    q: torch.Tensor
    qd: torch.Tensor
    qdd: torch.Tensor
    force: torch.Tensor
    solved: torch.Tensor


class DifferentiableRobotModel(torch.nn.Module):
    """Batched rigid-body kinematics / dynamics of a URDF robot on one GPU (H100, sm_90a)."""

    def __init__(self, urdf_path: str, name="", device=None):
        super().__init__()
        self.name = name
        # device=None: the reference defaults to the CPU and computes there (robot_model.py:100-104).  This engine has
        # no CPU path, so a default-constructed model lives on the current CUDA device whenever one is present (and
        # computes, like the reference's default-constructed model does); without a GPU it is a host-side model
        # (URDF, topology, parameters, joint limits) whose compute entry points raise.  An explicit device is honoured.
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        self._device = torch.device(device)
        if self._device.type == "cuda" and self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())

        self._urdf_model = URDFRobotModel(urdf_path=urdf_path, device=self._device)
        self._bodies = torch.nn.ModuleList()
        self._n_dofs = 0
        self._controlled_joints = []
        self._name_to_idx_map = dict()

        # links in URDF document order; the joint is part of its child link (robot_model.py:114-130)
        for i, link in enumerate(self._urdf_model.robot.links):
            params = self._urdf_model.get_body_parameters_from_urdf(i, link)
            body = DifferentiableRigidBody(rigid_body_params=params, device=self._device)
            if params["joint_type"] != "fixed":
                body.joint_idx = self._n_dofs
                self._n_dofs += 1
                self._controlled_joints.append(i)
            self._bodies.append(body)
            self._name_to_idx_map[body.name] = i

        # resolve parents ONCE (robot_model.py:133-137 does the same; the reference's hot loops re-scan)
        self._parent_idx = [-1] * len(self._bodies)
        for i, body in enumerate(self._bodies):
            if i == 0:
                continue
            parent_idx = self._name_to_idx_map[self._urdf_model.get_name_of_parent_body(body.name)]
            self._parent_idx[i] = parent_idx
            body.set_parent(self._bodies[parent_idx])
            self._bodies[parent_idx].add_child(body)

        for body in self._bodies:
            body._bind_model(self)
        self._topology = compile_topology(self._bodies, self._parent_idx)
        self._kin_state = None
        self._table_cache = None
        self._folded_cache = None
        self._has_learnable = None          # any of the six per-link attributes replaced by a torch.nn.Module

    # ------------------------------------------------------------------------------------------
    # link table
    # ------------------------------------------------------------------------------------------
    @contextlib.contextmanager
    def shared_link_table(self):
        """Opt-in: every compute call inside the block uses ONE (differentiable) link table, built on entry.

        By default each call of a model with learnable link parameters rebuilds the table, exactly like each call of
        the reference rebuilds its per-link graph, so that separate ``backward()`` calls stay independent.  A training
        step that evaluates several quantities before a single ``backward()`` (e.g. FK + Jacobian + inverse dynamics,
        BASELINE config 5) can share the table and save the repeated parametrisation -> table work."""
        self._shared_table = self._link_table()
        try:
            yield self._shared_table
        finally:
            self._shared_table = None

    def invalidate_link_table(self) -> None:
        """Drop the cached link table (call after editing a constant link parameter tensor in place)."""
        self._table_cache = None
        self._folded_cache = None
        self._has_learnable = None

    def _folded_table(self):
        """Constant models only: the link table with the links behind fixed joints folded into their movable ancestors
        (``drmb200_fold_link_table``), computed once; the inverse-dynamics kernel then skips its per-CTA folding."""
        if self._any_learnable_module() or getattr(self, "_shared_table", None) is not None:
            return None
        if getattr(self, "_folded_cache", None) is None:
            folded = engine.fold_link_table(self._topology, self._link_table())
            self._folded_cache = folded if folded is not None else False
        return self._folded_cache if self._folded_cache is not False else None

    def _any_learnable_module(self) -> bool:
        if self._has_learnable is None:
            self._has_learnable = any(
                isinstance(getattr(owner, name), torch.nn.Module)
                for body in self._bodies
                for owner, names in ((body, ("trans", "rot_angles", "joint_damping")), (body.inertia, ("mass", "com", "inertia_mat")))
                for name in names)
        return self._has_learnable

    def _link_table(self) -> torch.Tensor:
        """The ``[n_links, 28]`` device table.  A model whose link parameters are all URDF constants builds it once.
        As soon as any link parameter is a parametrisation module the table is re-evaluated on EVERY call (one
        ``torch.cat`` + one kernel), exactly like the reference re-evaluates its per-link callables on every call --
        in-place edits of parameters (``p.data.copy_``), buffers or frozen modules can never leave a stale table behind;
        the result carries an autograd graph when grad mode is on and a parameter requires grad."""
        if getattr(self, "_shared_table", None) is not None:
            return self._shared_table
        if getattr(self, "fused_link_params", None) is not None:
            return self.fused_link_params.table()
        if self._any_learnable_module():
            return build_link_table(self._bodies, self._device)
        if self._table_cache is None:
            with torch.no_grad():
                self._table_cache = build_link_table(self._bodies, self._device)
        return self._table_cache

    def fuse_learnable_parameters(self) -> torch.nn.Parameter:
        """Gather every learnable link parameter into ONE flat ``nn.Parameter`` (returned; also
        ``model.fused_link_params.flat``): the link table is then built from it by one kernel, the backward leaves one
        gradient tensor and ``torch.optim.Adam(model.parameters(), fused=True)`` updates everything in one launch.  Call
        once, after the last ``make_link_param_learnable``; values and gradients are the same as on the per-module path
        (the modules' own Parameters become views of the flat storage and stop requiring grad):

        * a module installed on several links (tied parameters) owns one slice of the flat vector and receives the sum
          of the gradients of all its links;
        * a module that is frozen (``freeze_learnable_link_param``) when this is called stays out of the flat vector:
          its current value becomes a constant of the table, so it gets no gradient and no optimiser can move it.
          Freezing is decided before fusing -- afterwards ``freeze_`` / ``unfreeze_learnable_link_param``,
          ``make_link_param_learnable`` and a second ``fuse_learnable_parameters`` raise ``RuntimeError``.

        Raises ``ValueError`` for (unfrozen) parametrisations other than UnconstrainedScalar / UnconstrainedTensor /
        PositiveScalar; the model then stays on the per-module path."""
        if self._device.type != "cuda":
            raise RuntimeError("fuse_learnable_parameters needs a CUDA model")
        if getattr(self, "fused_link_params", None) is not None:
            raise RuntimeError("fuse_learnable_parameters() called twice: the model is already fused")
        self.fused_link_params = FusedLinkParameters(self._bodies, self._device)
        return self.fused_link_params.flat

    def _kinematic_params_learnable(self) -> bool:
        """True if any joint origin (``trans`` / ``rot_angles`` of a movable link) is a learnable module with a
        parameter that requires grad -- then the backward kernels must produce the F / r columns of the table
        gradient; otherwise the RNEA backward can take the single-sweep inertial path."""
        fused = getattr(self, "fused_link_params", None)
        if fused is not None:                                  # the flat vector carries everything that can learn
            return fused.feeds_kinematics and fused.flat.requires_grad
        for body in self._bodies:
            if body.joint_idx is None:
                continue
            for name in ("trans", "rot_angles"):
                attr = getattr(body, name)
                if isinstance(attr, torch.nn.Module):
                    params = list(attr.parameters())
                    if not params or any(p.requires_grad for p in params):      # parameter-free modules: be safe
                        return True
        return False

    def _check_q(self, *tensors):
        for t in tensors:
            assert t.ndim == 2
            assert t.shape[1] == self._n_dofs

    # ------------------------------------------------------------------------------------------
    # kinematics
    # ------------------------------------------------------------------------------------------
    def _fk_jacobian(self, q, link_name, want_pos, want_quat, want_jac):
        link_idx = self._name_to_idx_map[link_name]          # KeyError for unknown links (robot_model.py:245)
        table = self._link_table()
        # kinematics depend on the (F, r) columns only: with nothing but inertial parameters learnable there is no graph
        if torch.is_grad_enabled() and (q.requires_grad or (table.requires_grad and self._kinematic_params_learnable())):
            return engine.FkJacobianFunction.apply(table, q, self._topology, link_idx, want_pos, want_quat, want_jac)
        return engine.fk_jacobian_raw(self._topology, link_idx, table.detach(), q, want_pos, want_quat, want_jac)

    @tensor_check
    def compute_forward_kinematics(
        self, q: torch.Tensor, link_name: str, recursive: bool = False
    ) -> Tuple[torch.Tensor, torch.Tensor]:
        r"""
        Args:
            q: joint angles [batch_size x n_dofs]
            link_name: name of link
        Returns: translation [batch_size x 3] and xyzw quaternion [batch_size x 4] of the link frame
        """
        self._check_q(q)
        pos, quat, _, _ = self._fk_jacobian(q, link_name, True, True, False)
        return pos, quat

    @tensor_check
    def compute_endeffector_jacobian(self, q: torch.Tensor, link_name: str) -> Tuple[torch.Tensor, torch.Tensor]:
        r"""
        Args:
            q: joint angles [batch_size x n_dofs]
            link_name: name of link for the jacobian
        Returns: linear and angular jacobian, each [batch_size x 3 x n_dofs]
        """
        self._check_q(q)
        _, _, jlin, jang = self._fk_jacobian(q, link_name, False, False, True)
        return jlin, jang

    @tensor_check
    def compute_fk_and_jacobian(
        self, q: torch.Tensor, link_name: str
    ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        r"""Fused op (one launch): ``(pos, quat, lin_jac, ang_jac)`` of ``link_name``.  The reference
        computes all four inside ``compute_endeffector_jacobian`` and discards the pose."""
        self._check_q(q)
        return self._fk_jacobian(q, link_name, True, True, True)

    def _fk_jacobian_multi(self, q, link_names, want_pos, want_quat, want_jac):
        links = [self._name_to_idx_map[name] for name in link_names]      # KeyError for unknown links
        assert len(set(links)) == len(links), "link names must be distinct"
        table = self._link_table()
        if torch.is_grad_enabled() and (q.requires_grad or table.requires_grad):
            return engine.FkJacobianMultiFunction.apply(table, q, self._topology, links, want_pos, want_quat, want_jac)
        return engine.fk_jacobian_multi_raw(self._topology, links, table, q, want_pos, want_quat, want_jac)

    @tensor_check
    def compute_fk_and_jacobian_multi(
        self, q: torch.Tensor, link_names: List[str]
    ) -> Dict[str, Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]]:
        r"""``{link_name: (pos, quat, lin_jac, ang_jac)}`` of several links (at most 8, distinct) from ONE launch that walks
        the union of their root paths once per configuration (``csrc/fk_tree.cu``) -- e.g. the four fingertips of a hand.
        Every entry equals what ``compute_forward_kinematics`` / ``compute_endeffector_jacobian`` return for that link
        (the reference runs its whole per-link pass once per end effector, ``robot_model.py:641``).  Differentiable.
        Like ``compute_forward_kinematics_all_links``, 1-D inputs give un-squeezed ``[1, .]`` values."""
        self._check_q(q)
        pos, quat, jlin, jang = self._fk_jacobian_multi(q, link_names, True, True, True)
        return {name: (pos[e], quat[e], jlin[e], jang[e]) for e, name in enumerate(link_names)}

    @tensor_check
    def compute_endeffector_jacobians(
        self, q: torch.Tensor, link_names: List[str]
    ) -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
        r"""``{link_name: (lin_jac, ang_jac)}`` of several links from one launch (see ``compute_fk_and_jacobian_multi``)."""
        self._check_q(q)
        _, _, jlin, jang = self._fk_jacobian_multi(q, link_names, False, False, True)
        return {name: (jlin[e], jang[e]) for e, name in enumerate(link_names)}

    # ------------------------------------------------------------------------------------------
    # dynamics
    # ------------------------------------------------------------------------------------------
    @tensor_check
    def compute_inverse_dynamics(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        qdd_des: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = True,
    ) -> torch.Tensor:
        r"""
        Args:
            q, qd, qdd_des: joint angles / velocities / desired accelerations [batch_size x n_dofs]
            include_gravity: when False, gravity compensation is assumed to be taken care of
            use_damping: add ``damping * qd``
        Returns: joint torques [batch_size x n_dofs] that achieve the desired accelerations
        """
        self._check_q(q, qd, qdd_des)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        self._remember_dynamic_inputs(q, qd, qdd_des, flags)       # for the lazy `_bodies[i].acc / .force`
        table = self._link_table()
        if not self._kinematic_params_learnable():
            flags |= engine.INERTIAL_GRADS_ONLY     # backward hint: only (I_o, mc, m, damping) columns can matter
        folded = self._folded_table()                  # constant model: folded once instead of once per CTA
        if torch.is_grad_enabled() and (
            table.requires_grad or q.requires_grad or qd.requires_grad or qdd_des.requires_grad
        ):
            return engine.InverseDynamicsFunction.apply(table, q, qd, qdd_des, self._topology, flags, folded)
        return engine.inverse_dynamics_raw(self._topology, table, q, qd, qdd_des, flags, folded=folded)

    @tensor_check
    def compute_non_linear_effects(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = True,
    ) -> torch.Tensor:
        r"""Coriolis, centrifugal, gravitational and damping torques = inverse dynamics at qdd = 0
        (robot_model.py:378-400)."""
        return self.compute_inverse_dynamics(q, qd, q.new_zeros(q.shape), include_gravity, use_damping)

    # ------------------------------------------------------------------------------------------
    # callers either side of the hot path (SURVEY.md section 8f "next" rows): mass matrix, forward dynamics and
    # all-links kinematics each have their own kernel; non-linear effects is the RNEA kernel with qdd = 0
    # ------------------------------------------------------------------------------------------
    @tensor_check
    def compute_lagrangian_inertia_matrix(
        self,
        q: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = True,
    ) -> torch.Tensor:
        r"""Joint-space mass matrix ``H(q)`` ``[batch_size x n_dofs x n_dofs]`` in ONE launch (``csrc/mass_matrix.cu``).
        The reference builds it from n + 1 inverse-dynamics evaluations (``robot_model.py:403-450``: column j =
        ID(q, 0, e_j) - ID(q, 0, 0)); the subtraction cancels gravity and damping (qd = 0), so the kernel evaluates the n
        unit-acceleration columns directly for zero velocity and zero gravity -- ``include_gravity`` / ``use_damping``
        therefore do not change the result, exactly as in the reference up to its fp32 cancellation noise.
        Differentiable w.r.t. q and every learnable link parameter (RNEA adjoint kernel over the stacked columns)."""
        assert q.shape[1] == self._n_dofs
        return engine.MassMatrixFunction.apply(self._link_table(), q, self._topology, self._folded_table())

    @tensor_check
    def compute_lagrangian_inertia_matrix_stacked(
        self,
        q: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = True,
    ) -> torch.Tensor:
        r"""The reference's construction verbatim (column j = ID(q, 0, e_j) - ID(q, 0, 0)) as ONE RNEA launch over a
        ``(n_dofs + 1) x batch`` stacked batch; kept as an independent cross-check of the mass-matrix kernel."""
        assert q.shape[1] == self._n_dofs
        B, n = q.shape
        zero = q.new_zeros((n + 1) * B, n)
        qdd = zero.clone().view(n + 1, B, n)
        idx = torch.arange(n, device=q.device)
        qdd[idx, :, idx] = 1.0                                  # slab j: unit acceleration of joint j; slab n: zero
        tau = self.compute_inverse_dynamics(q.repeat(n + 1, 1), zero, qdd.view(-1, n), include_gravity, use_damping)
        tau = tau.view(n + 1, B, n)
        return (tau[:n] - tau[n:]).permute(1, 2, 0).contiguous()

    @tensor_check
    def compute_forward_dynamics(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        f: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
        implicit_damping_dt: Optional[float] = None,
    ) -> torch.Tensor:
        r"""Joint accelerations under applied joint forces ``f``: the articulated-body algorithm of
        ``robot_model.py:488-624`` in ONE launch (``csrc/aba.cu``), with the reference's arithmetic (general 6x6
        articulated inertias -- ``inertia_mat`` is never symmetrised --, ``+1e-37`` regularisers).  Differentiable
        w.r.t. q, qd, f and every learnable link parameter through the analytic adjoint kernel.  Unlike the reference
        this does not overwrite the caller's ``f`` when ``use_damping`` is set (``robot_model.py:521``).

        ``implicit_damping_dt = h`` (needs ``use_damping``) treats the joint damping implicitly for a step of length ``h``:
        every joint's articulated-body pivot ``d`` becomes ``d + h * damping``, which for symmetric inertias gives
        ``(H + h diag(damping))^-1 (f - nle(q, qd))``, the acceleration of a semi-implicit Euler step whose damping torque
        is taken at the end-of-step velocity ``qd + h qdd``.  Such a step is stable at any ``h``, however strongly damped
        and light the links (``include/drm_b200.h``: ``drmb200_forward_dynamics_implicit_damping``).  ``h`` is not
        differentiated."""
        self._check_q(q, qd, f)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        if implicit_damping_dt is not None:
            h = self._implicit_damping_step(True, use_damping, implicit_damping_dt)
            return engine.ForwardDynamicsFunction.apply(self._link_table(), q, qd, f, self._topology, flags, None, h)
        return engine.ForwardDynamicsFunction.apply(self._link_table(), q, qd, f, self._topology, flags, self._folded_table())

    @tensor_check
    def compute_inverse_dynamics_derivatives(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        qdd_des: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = True,
    ) -> Tuple[torch.Tensor, torch.Tensor]:
        r"""Jacobians of :meth:`compute_inverse_dynamics` in ONE launch (``csrc/dynamics_derivatives.cu``, forward-mode RNEA).

        Args:
            q, qd, qdd_des: joint angles / velocities / desired accelerations [batch_size x n_dofs]
            include_gravity, use_damping: as for :meth:`compute_inverse_dynamics`
        Returns: ``(dtau_dq, dtau_dqd)``, each [batch_size x n_dofs x n_dofs] (``[n_dofs x n_dofs]`` for 1-D inputs) with
        ``out[b, i, j] = d tau_i / d x_j``.  The outputs carry no autograd graph: they use the current values of the link
        parameters (learnable and fused ones included) but are not differentiable themselves."""
        self._check_q(q, qd, qdd_des)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        table = self._link_table().detach()
        return engine.inverse_dynamics_derivatives_raw(self._topology, table, q.detach(), qd.detach(), qdd_des.detach(), flags,
                                                       folded=self._folded_table())

    @tensor_check
    def compute_forward_dynamics_derivatives(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        f: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
    ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        r"""Jacobians of :meth:`compute_forward_dynamics` in ONE launch (``csrc/dynamics_derivatives.cu``, forward-mode
        articulated-body algorithm).

        Args:
            q, qd, f: joint angles / velocities / applied joint forces [batch_size x n_dofs]
            include_gravity, use_damping: as for :meth:`compute_forward_dynamics`
        Returns: ``(dqdd_dq, dqdd_dqd, dqdd_df)``, each [batch_size x n_dofs x n_dofs] (``[n_dofs x n_dofs]`` for 1-D
        inputs) with ``out[b, i, j] = d qdd_i / d x_j``.  They differentiate the articulated-body arithmetic itself, so they
        are exact for non-symmetric ``inertia_mat`` too, where ``-H^-1 dtau`` is not.  The outputs carry no autograd graph:
        they use the current values of the link parameters (learnable and fused ones included) but are not differentiable
        themselves."""
        self._check_q(q, qd, f)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        table = self._link_table().detach()
        return engine.forward_dynamics_derivatives_raw(self._topology, table, q.detach(), qd.detach(), f.detach(), flags,
                                                       folded=self._folded_table())

    @tensor_check
    def compute_dynamics_regressor(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        qdd_des: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = True,
    ) -> torch.Tensor:
        r"""The joint-torque regressor of the inertial parameters in ONE launch (``csrc/dynamics_regressor.cu``).

        Args:
            q, qd, qdd_des: joint angles / velocities / desired accelerations [batch_size x n_dofs]
            include_gravity, use_damping: as for :meth:`compute_inverse_dynamics`
        Returns: ``Y`` [batch_size x n_dofs x n_links x 14] (``[n_dofs x n_links x 14]`` for 1-D inputs) with
        ``Y[b, i, l, k] = d tau_i / d pi[l, k]``, ``pi = inertial_parameters()``, so that
        ``einsum("bilk,lk->bi", Y, pi)`` is :meth:`compute_inverse_dynamics` of the same inputs.  The output carries no
        autograd graph: it uses the current values of the link parameters (learnable and fused ones included) and, being
        linear in them, does not depend on the inertial ones at all."""
        self._check_q(q, qd, qdd_des)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        table = self._link_table().detach()
        return engine.dynamics_regressor_raw(self._topology, table, q.detach(), qd.detach(), qdd_des.detach(), flags)

    def inertial_parameters(self) -> torch.Tensor:
        r"""Every link's inertial parameters and damping, ``[n_links x 14]`` in URDF link order (the root first): the link
        table's columns 12:26,

            ``I_o`` (9, row-major) | ``m c`` (3) | ``m`` | joint damping,

        with ``I_o = I_c + m S(c) S(c)^T`` the rotational inertia about the link frame's origin.  Differentiable when link
        parameters are learnable.  For every configuration

            ``einsum("bilk,lk->bi", compute_dynamics_regressor(q, qd, qdd), inertial_parameters())
            == compute_inverse_dynamics(q, qd, qdd)``

        (same ``include_gravity`` / ``use_damping``).  ``I_o`` is not symmetrised, so its nine entries are nine columns of
        the regressor.  The standard symmetric 10-parameter form per link, ``(Ixx, Ixy, Ixz, Iyy, Iyz, Izz, mcx, mcy, mcz,
        m)``, has the regressor columns of ``I_o[a, a]`` and, for ``a != b``, the sum of the ``I_o[a, b]`` and ``I_o[b, a]``
        columns."""
        return self._link_table()[:, 12:26]

    def compute_energy_and_momentum(self, q: torch.Tensor, qd: Optional[torch.Tensor] = None) -> EnergyAndMomentum:
        r"""Whole-body quantities of every configuration in ONE launch (``csrc/energy_momentum.cu``; the definitions are
        stated in ``include/drm_b200.h``): kinetic energy ``1/2 sum_i <V_i, I_i V_i>``, potential energy in gravity
        ``(0, 0, -9.81)`` (zero at z = 0), generalized momentum, centre of mass ``com`` (zeros for a massless model), its
        world-frame velocity and its Jacobian.  For every configuration, up to rounding,
            ``momentum = H qd`` with ``H = compute_lagrangian_inertia_matrix(q)``,
            ``kinetic_energy = 1/2 qd . momentum``,
            ``d potential_energy / dq = compute_inverse_dynamics(q, 0, 0, include_gravity=True, use_damping=False)
            = 9.81 M com_jacobian[2]`` (M the total mass),
            ``com_jacobian = d com / dq`` and ``com_velocity = com_jacobian qd``.

        Args:
            q: joint angles [batch_size x n_dofs]
            qd: joint velocities [batch_size x n_dofs], or None: ``kinetic_energy``, ``momentum`` and ``com_velocity`` are
                then None (the other fields are bit-identical to a call with qd)
        Returns: :class:`EnergyAndMomentum` with shapes [batch_size], [batch_size], [batch_size x n_dofs], [batch_size x 3],
        [batch_size x 3], [batch_size x 3 x n_dofs], squeezed for 1-D inputs.  The outputs carry no autograd graph: they use
        the current values of the link parameters (learnable and fused ones included) but are not differentiable."""
        return EnergyAndMomentum(*self._energy_and_momentum(q, qd))

    @tensor_check
    def _energy_and_momentum(self, q, qd):
        given = [t for t in (q, qd) if t is not None]
        self._check_q(*given)
        assert all(t.dtype == torch.float32 for t in given), "the engine is fp32-only"
        table = self._link_table().detach()
        return engine.energy_momentum_raw(self._topology, table, q.detach(), None if qd is None else qd.detach())

    def compute_operational_space_dynamics(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        f: torch.Tensor,
        link_names: List[str],
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
        position_only: bool = False,
    ) -> OperationalSpaceDynamics:
        r"""Operational-space dynamics of several links (at most 8, distinct) in ONE launch (``csrc/operational_space.cu``;
        the definition is stated in ``include/drm_b200.h``).  With ``J`` the links' geometric Jacobians stacked (as
        :meth:`compute_endeffector_jacobian` returns them, linear rows over angular rows; linear rows only with
        ``position_only``), ``qdd`` what :meth:`compute_forward_dynamics` returns and ``G`` the ``dqdd_df`` of
        :meth:`compute_forward_dynamics_derivatives` (``H^-1`` for symmetric inertias):

        * ``inv_inertia = J G J^T``: maps a stacked force / wrench ``F`` applied at the links to their acceleration change,
          ``acceleration(f + J^T F) = acceleration(f) + inv_inertia F``; invert it (regularised as you see fit) for the
          operational-space inertia, or use the position-only version of several fingertips as a contact-space inverse
          inertia;
        * ``velocity = J qd``, ``bias_acceleration = Jdot qd`` and ``acceleration = J qdd + Jdot qd``.

        Args:
            q, qd, f: joint angles / velocities / applied joint forces [batch_size x n_dofs]
            link_names: the links, stacked in this order; the root and links with no movable joint on their root path get
                zero rows and columns
            include_gravity, use_damping: as for :meth:`compute_forward_dynamics`
            position_only: 3 rows per link (the linear ones) instead of 6
        Returns: :class:`OperationalSpaceDynamics` with shapes [batch_size x M x M] and [batch_size x M] (``[M x M]`` and
        ``[M]`` for 1-D inputs), M = 6 or 3 per link.  The outputs carry no autograd graph: they use the current values of
        the link parameters (learnable and fused ones included) but are not differentiable."""
        links = [self._name_to_idx_map[name] for name in link_names]      # KeyError for unknown links
        assert len(set(links)) == len(links), "link names must be distinct"
        return OperationalSpaceDynamics(*self._operational_space_dynamics(q, qd, f, links=links, include_gravity=include_gravity,
                                                                          use_damping=use_damping, position_only=position_only))

    @tensor_check
    def _operational_space_dynamics(self, q, qd, f, links, include_gravity, use_damping, position_only):
        self._check_q(q, qd, f)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        table = self._link_table().detach()
        return engine.operational_space_dynamics_raw(self._topology, links, table, q.detach(), qd.detach(), f.detach(), flags,
                                                     position_only=bool(position_only))

    def compute_contact_dynamics(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        f: torch.Tensor,
        link_names: List[str],
        accel_ref: Optional[torch.Tensor] = None,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
        position_only: bool = False,
        regularization: float = 0.0,
        differentiable: bool = False,
    ) -> ContactDynamics:
        r"""Forward dynamics with the links held by bilateral rigid contacts (at most 8, distinct), in ONE launch
        (``csrc/contact_dynamics.cu``; the definition and the solve are stated in ``include/drm_b200.h``).  With ``J``, ``G``,
        ``qdd_free`` and ``Jdot qd`` as in :meth:`compute_operational_space_dynamics` and ``mu = regularization``:

        * ``A = J G J^T + mu I`` and ``lambda`` solves ``A lambda = accel_ref - (J qdd_free + Jdot qd)``;
        * ``qdd = qdd_free + G J^T lambda``, which is :meth:`compute_forward_dynamics` at ``f + J^T lambda``;
        * ``force = lambda``: the world-frame force (and torque, in pose mode) applied at each link origin;
        * hence ``J qdd + Jdot qd = accel_ref - mu lambda``: the links move with the requested acceleration when ``mu = 0``.
          For symmetric inertias this is Gauss's principle, ``H (qdd - qdd_free) = J^T lambda``.

        Args:
            q, qd, f: joint angles / velocities / applied joint forces [batch_size x n_dofs]
            link_names: the held links, stacked in this order; each needs a movable joint on its root path
            accel_ref: the desired constraint-space acceleration [batch_size x M] (e.g. Baumgarte terms); None: 0
            include_gravity, use_damping: as for :meth:`compute_forward_dynamics`
            position_only: hold the link origins only (3 rows per link) instead of the full pose (6)
            regularization: ``mu >= 0``; redundant constraint sets (more rows than the joints can satisfy) need ``mu > 0``
            differentiable: make ``qdd`` and ``force`` differentiable (see below); off by default
        Returns: :class:`ContactDynamics` ``(qdd, force, solved)``, squeezed for 1-D inputs.  A row whose equilibrated system
        has a pivot of magnitude <= 1e-5 is not solved: ``solved`` is False and its outputs are NaN.  By default the outputs
        carry no autograd graph: they use the current values of the link parameters (learnable and fused ones included) but
        are not differentiable.

        With ``differentiable=True``, grad mode on and any of q, qd, f, accel_ref or a learnable link parameter requiring
        grad, ``qdd`` and ``force`` are differentiable w.r.t. all of them (fused parameters included) through the analytic
        adjoint (``csrc/contact_backward.cu``, stated in ``include/drm_b200.h``): for upstream gradients ``g_qdd``,
        ``g_force``, ``nu`` solves ``A^T nu = g_force + J G^T g_qdd``, ``accel_ref`` receives ``nu``, and q, qd, f and the link
        parameters receive the forward-dynamics adjoint at ``(q, qd, f + J^T lambda)`` for ``g_qdd - J^T nu`` plus the
        derivatives of ``lambda^T J f_grad - nu^T (J qdd + Jdot qd)``.  Unsolved rows receive exactly zero gradients,
        whatever their upstream gradient.  ``regularization`` is not differentiated, ``solved`` carries no graph, and the
        gradients are first-order only.  The forward is the same single launch with the same outputs, bit for bit."""
        links = self._contact_links(link_names)
        out = self._contact_dynamics(q, qd, f, accel_ref, links=links, include_gravity=include_gravity,
                                     use_damping=use_damping, position_only=bool(position_only),
                                     regularization=float(regularization), differentiable=bool(differentiable))
        return ContactDynamics(*out)

    def compute_contact_impulse(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        link_names: List[str],
        velocity_ref: Optional[torch.Tensor] = None,
        position_only: bool = False,
        regularization: float = 0.0,
        differentiable: bool = False,
    ) -> ContactImpulse:
        r"""The joint velocities after an instantaneous impact at the links (at most 8, distinct), in ONE launch
        (``csrc/contact_dynamics.cu``; stated in ``include/drm_b200.h``).  With ``J`` and ``G`` as in
        :meth:`compute_operational_space_dynamics` and ``mu = regularization``:

        * ``Lambda`` solves ``(J G J^T + mu I) Lambda = velocity_ref - J qd``;
        * ``qd_plus = qd + G J^T Lambda`` and ``impulse = Lambda``, so ``J qd_plus = velocity_ref - mu Lambda``.

        Gravity, damping and applied forces do not act during the impulse.  ``velocity_ref = None`` (0) is a perfectly
        inelastic impact, which does not increase the kinetic energy; ``velocity_ref = -e J qd`` is restitution ``e``, and
        ``e = 1`` with ``mu = 0`` keeps the kinetic energy (symmetric inertias).

        Args:
            q, qd: joint angles / velocities before the impact [batch_size x n_dofs]
            link_names, position_only, regularization: as for :meth:`compute_contact_dynamics`
            velocity_ref: the desired constraint-space velocity after the impact [batch_size x M]; None: 0
            differentiable: make ``qd_plus`` and ``impulse`` differentiable (see below); off by default
        Returns: :class:`ContactImpulse` ``(qd_plus, impulse, solved)``, squeezed for 1-D inputs; unsolved rows as in
        :meth:`compute_contact_dynamics`.  By default no autograd graph, current link parameters.

        With ``differentiable=True``, grad mode on and any of q, qd, velocity_ref or a learnable link parameter requiring
        grad, ``qd_plus`` and ``impulse`` are differentiable w.r.t. all of them: as for :meth:`compute_contact_dynamics`,
        with ``nu`` solving ``A^T nu = g_impulse + J G^T g_qd_plus``, ``velocity_ref`` receiving ``nu``, qd receiving
        ``g_qd_plus - J^T nu``, and q and the link parameters the forward-dynamics adjoint at ``(q, 0, J^T Lambda)`` plus the
        derivatives of ``Lambda^T J tau - nu^T J qd_plus``.  Unsolved rows receive exactly zero gradients; ``regularization``
        is not differentiated; ``solved`` carries no graph; first-order only; the forward is the same launch, bit for bit."""
        links = self._contact_links(link_names)
        out = self._contact_impulse(q, qd, velocity_ref, links=links, position_only=bool(position_only),
                                    regularization=float(regularization), differentiable=bool(differentiable))
        return ContactImpulse(*out)

    def _contact_links(self, link_names):
        links = [self._name_to_idx_map[name] for name in link_names]      # KeyError for unknown links
        assert len(set(links)) == len(links), "link names must be distinct"
        return links

    @tensor_check
    def _contact_dynamics(self, q, qd, f, accel_ref, links, include_gravity, use_damping, position_only, regularization,
                          differentiable=False):
        self._check_q(q, qd, f)
        M = (3 if position_only else 6) * len(links)
        assert accel_ref is None or tuple(accel_ref.shape) == (q.shape[0], M), f"accel_ref must be [batch_size x {M}]"
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        table = self._link_table()
        if differentiable and torch.is_grad_enabled() and any(t is not None and t.requires_grad
                                                              for t in (table, q, qd, f, accel_ref)):
            return engine.ContactDynamicsFunction.apply(table, q, qd, f, accel_ref, self._topology, links, flags, position_only,
                                                        regularization)
        table = table.detach()
        return engine.contact_dynamics_raw(self._topology, links, table, q.detach(), qd.detach(), f.detach(), flags,
                                           None if accel_ref is None else accel_ref.detach(), position_only, regularization)

    @tensor_check
    def _contact_impulse(self, q, qd, velocity_ref, links, position_only, regularization, differentiable=False):
        self._check_q(q, qd)
        M = (3 if position_only else 6) * len(links)
        assert velocity_ref is None or tuple(velocity_ref.shape) == (q.shape[0], M), f"velocity_ref must be [batch_size x {M}]"
        table = self._link_table()
        if differentiable and torch.is_grad_enabled() and any(t is not None and t.requires_grad
                                                              for t in (table, q, qd, velocity_ref)):
            return engine.ContactImpulseFunction.apply(table, q, qd, velocity_ref, self._topology, links, position_only,
                                                       regularization)
        table = table.detach()
        return engine.contact_impulse_raw(self._topology, links, table, q.detach(), qd.detach(),
                                          None if velocity_ref is None else velocity_ref.detach(), position_only, regularization)

    def compute_inverse_kinematics(
        self,
        q0: torch.Tensor,
        link_name: str,
        target_pos: torch.Tensor,
        target_quat: Optional[torch.Tensor] = None,
        max_iters: int = 100,
        pos_tol: float = 1e-4,
        rot_tol: float = 1e-3,
        respect_joint_limits: bool = True,
        damping: Optional[Union[float, torch.Tensor]] = None,
    ) -> InverseKinematicsResult:
        r"""Inverse kinematics of ``link_name``: up to ``max_iters`` damped least-squares (Levenberg-Marquardt) iterations
        per row, all in ONE launch (``csrc/inverse_kinematics.cu``; the algorithm is stated in ``include/drm_b200.h``).

        Args:
            q0: start joint angles [batch_size x n_dofs] (clamped to the joint limits first)
            link_name: the link whose frame should reach the target
            target_pos: target position [batch_size x 3]
            target_quat: target orientation [batch_size x 4], xyzw like :meth:`compute_forward_kinematics` (normalised
                here); None solves for the position only
            pos_tol, rot_tol: a row stops once its position error (m) and orientation error (rad) are both within these
            respect_joint_limits: clamp every iterate to :meth:`get_joint_limits`
            damping: initial damping, a float or one value per row [batch_size]; None: 1e-2
        Returns: :class:`InverseKinematicsResult` ``(q, pos_error, rot_error, converged, damping)``, squeezed for 1-D
        inputs.  Joints off the root -> link path are returned unchanged.  The outputs carry no autograd graph: they use the
        current values of the link parameters (learnable and fused ones included) but are not differentiable."""
        link_idx = self._name_to_idx_map[link_name]          # KeyError for unknown links
        damping_init = engine.IK_DAMPING_INIT
        per_row = None
        if isinstance(damping, torch.Tensor):
            per_row = damping.detach().unsqueeze(-1)          # [B, 1] (or [1] for 1-D inputs): batch-checked below
        elif damping is not None:
            damping_init = float(damping)
        out = self._inverse_kinematics(q0, target_pos, target_quat, per_row, link_idx=link_idx, max_iters=int(max_iters),
                                       damping_init=damping_init, pos_tol=float(pos_tol), rot_tol=float(rot_tol),
                                       respect_joint_limits=respect_joint_limits)
        return InverseKinematicsResult(*out)

    @tensor_check
    def _inverse_kinematics(self, q0, target_pos, target_quat, damping, link_idx, max_iters, damping_init, pos_tol, rot_tol,
                            respect_joint_limits):
        self._check_q(q0)
        assert target_pos.shape[1] == 3, "target_pos must be [batch_size x 3]"
        assert target_quat is None or target_quat.shape[1] == 4, "target_quat must be [batch_size x 4]"
        lower, upper = self._joint_limit_tensors() if respect_joint_limits else (None, None)
        table = self._link_table().detach()
        q, pos_err, rot_err, converged, damp = engine.inverse_kinematics_raw(
            self._topology, link_idx, table, q0.detach(), target_pos.detach(),
            None if target_quat is None else target_quat.detach(), lower, upper,
            None if damping is None else damping[:, 0], max_iters, damping_init, pos_tol, rot_tol)
        return q, pos_err, rot_err, converged, damp

    def compute_inverse_kinematics_multi(
        self,
        q0: torch.Tensor,
        link_names: List[str],
        target_pos: torch.Tensor,
        target_quat: Optional[torch.Tensor] = None,
        max_iters: int = 100,
        pos_tol: float = 1e-4,
        rot_tol: float = 1e-3,
        respect_joint_limits: bool = True,
        damping: Optional[Union[float, torch.Tensor]] = None,
    ) -> InverseKinematicsResult:
        r"""Inverse kinematics of several links at once (e.g. the fingertips of a hand, or of a hand on an arm): up to
        ``max_iters`` Levenberg-Marquardt iterations per row over the stacked errors of every link, all in ONE launch
        (``csrc/inverse_kinematics_multi.cu``; the algorithm is stated in ``include/drm_b200.h``).  Joints shared by several
        links move for all of them together, which separate :meth:`compute_inverse_kinematics` calls cannot do.

        Args:
            q0: start joint angles [batch_size x n_dofs] (clamped to the joint limits first)
            link_names: the links (at most 8, distinct) whose frames should reach their targets
            target_pos: target positions [n_links x batch_size x 3] (``[n_links x 3]`` for 1-D ``q0``), the layout of
                :meth:`compute_fk_and_jacobian_multi`'s outputs stacked
            target_quat: target orientations [n_links x batch_size x 4] xyzw (normalised here); None solves for the
                positions only
            pos_tol, rot_tol: a row stops once every link's position error (m) and orientation error (rad) are within these
            respect_joint_limits: clamp every iterate to :meth:`get_joint_limits`
            damping: initial damping, a float or one value per row [batch_size]; None: 1e-2
        Returns: :class:`InverseKinematicsResult` ``(q, pos_error, rot_error, converged, damping)`` with ``pos_error`` and
        ``rot_error`` [n_links x batch_size]; squeezed for 1-D ``q0``.  Joints on none of the root -> link paths are returned
        unchanged.  The outputs carry no autograd graph: they use the current values of the link parameters (learnable and
        fused ones included) but are not differentiable."""
        links = [self._name_to_idx_map[name] for name in link_names]      # KeyError for unknown links
        E = len(links)
        squeeze = q0.ndim == 1
        damping_init = engine.IK_DAMPING_INIT
        per_row = None
        if isinstance(damping, torch.Tensor):
            per_row = damping.detach()
        elif damping is not None:
            damping_init = float(damping)
        for t in (q0, target_pos, target_quat, per_row):
            assert t is None or t.device.type == self._device.type, f"Input argument of different device as module: {t}"
        if squeeze:
            q0, target_pos = q0.unsqueeze(0), target_pos.unsqueeze(1)
            target_quat = None if target_quat is None else target_quat.unsqueeze(1)
            per_row = None if per_row is None else per_row.reshape(1)
        self._check_q(q0)
        B = q0.shape[0]
        assert target_pos.shape == (E, B, 3), "target_pos must be [n_links x batch_size x 3]"
        assert target_quat is None or target_quat.shape == (E, B, 4), "target_quat must be [n_links x batch_size x 4]"
        assert per_row is None or per_row.shape == (B,), "damping must be a float or [batch_size]"
        lower, upper = self._joint_limit_tensors() if respect_joint_limits else (None, None)
        out = engine.inverse_kinematics_multi_raw(
            self._topology, links, self._link_table().detach(), q0.detach(), target_pos.detach(),
            None if target_quat is None else target_quat.detach(), lower, upper, per_row, int(max_iters), damping_init,
            float(pos_tol), float(rot_tol))
        if squeeze:
            q, pos_err, rot_err, converged, damp = out
            out = (q[0], pos_err[:, 0], rot_err[:, 0], converged[0], damp[0])
        return InverseKinematicsResult(*out)

    def _joint_limit_tensors(self):
        """(lower, upper) [n_dofs] fp32 on the model's device, from get_joint_limits(), built once."""
        if getattr(self, "_limit_cache", None) is None:
            limits = self.get_joint_limits()
            lower = torch.tensor([float(l["lower"]) for l in limits], dtype=torch.float32, device=self._device)
            upper = torch.tensor([float(l["upper"]) for l in limits], dtype=torch.float32, device=self._device)
            self._limit_cache = (lower, upper)
        return self._limit_cache

    def _check_rollout_inputs(self, required, optional, steps):
        """The argument checks every rollout starts with: each ``(name, tensor)`` of ``required``, and of ``optional``
        unless None, is a float32 tensor on the module's device; ``q0`` / ``qd0`` (the first two) are one [batch_size x
        n_dofs] or [n_dofs] shape; the input named ``steps`` is [T x batch_size x n_dofs] (or [T x n_dofs]).  Returns
        whether the inputs are 1-D (one row without a batch dimension)."""
        for name, t in tuple(required) + tuple((name, t) for name, t in optional if t is not None):
            assert type(t) is torch.Tensor, f"{name} must be a torch.Tensor"
            assert t.device.type == self._device.type, f"Input argument of different device as module: {name}"
            assert t.dtype == torch.float32, f"{name} must be float32 (got {t.dtype})"
        q0, qd0, seq = required[0][1], required[1][1], dict(required)[steps]
        assert q0.ndim in (1, 2), "q0 must have ndim of 1 or 2."
        assert qd0.shape == q0.shape, "q0 and qd0 must have the same shape."
        assert q0.shape[-1] == self._n_dofs, f"expected {self._n_dofs} joints, got {q0.shape[-1]}"
        assert seq.ndim == q0.ndim + 1 and seq.shape[1:] == q0.shape, \
            f"{steps} must be [T x batch_size x n_dofs] (or [T x n_dofs])."
        return q0.ndim == 1

    @staticmethod
    def _implicit_damping_step(implicit, use_damping, dt):
        """The checks of ``implicit_damping`` / ``implicit_damping_dt``: ``use_damping`` is set and the step ``dt`` is finite
        and > 0.  Returns ``float(dt)``."""
        dt = float(dt)
        if implicit:
            assert use_damping, "implicit damping needs use_damping=True"
            assert 0.0 < dt < float("inf"), f"implicit damping needs a finite step dt > 0 (got {dt})"
        return dt

    @staticmethod
    def _rollout_batch_dim(q0, qd0, *per_step):
        """1-D rollout inputs with the batch dimension of one row added: ``q0`` / ``qd0`` in front, every per-step (or
        per-link) tensor after its leading dimension; None stays None."""
        return (q0.unsqueeze(0), qd0.unsqueeze(0)) + tuple(None if t is None else t.unsqueeze(1) for t in per_step)

    def compute_forward_dynamics_rollout(
        self,
        q0: torch.Tensor,
        qd0: torch.Tensor,
        f: torch.Tensor,
        dt: float,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
        implicit_damping: bool = False,
    ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        r"""Integrate :meth:`compute_forward_dynamics` over ``T`` steps of semi-implicit (symplectic) Euler in ONE launch
        (``csrc/rollout.cu``).  From ``(q_0, qd_0) = (q0, qd0)``, step ``t`` computes in fp32, in this order::

            qdd_t = compute_forward_dynamics(q_t, qd_t, f[t], include_gravity, use_damping)
            qd_{t+1} = qd_t + dt * qdd_t
            q_{t+1} = q_t + dt * qd_{t+1}

        and the result is bit-identical to that Python loop on the same model.  With ``implicit_damping`` (which needs
        ``use_damping``) step t calls ``compute_forward_dynamics(..., implicit_damping_dt=dt)`` instead: the damping torque
        is taken at the end-of-step velocity, so strongly damped light links (the Allegro fingers) stay stable at any ``dt``,
        where the explicit damping diverges above about ``dt = 2 I / d``.

        Args:
            q0, qd0: initial joint angles / velocities [batch_size x n_dofs] (or [n_dofs])
            f: applied joint forces of every step [T x batch_size x n_dofs] (or [T x n_dofs]); never modified
            dt: step length in seconds (not differentiable)
        Returns: time-major ``(q, qd, qdd)``, each [T x batch_size x n_dofs] (or [T x n_dofs]), with ``q[t] = q_{t+1}``,
        ``qd[t] = qd_{t+1}`` and ``qdd[t] = qdd_t``.  Differentiable w.r.t. q0, qd0, f and every learnable link parameter
        (the articulated-body adjoint stepped backwards in time).  Argument errors raise ``AssertionError``."""
        squeeze = self._check_rollout_inputs((("q0", q0), ("qd0", qd0), ("f", f)), (), "f")
        if squeeze:
            q0, qd0, f = self._rollout_batch_dim(q0, qd0, f)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        flags |= engine.IMPLICIT_DAMPING if implicit_damping else 0
        table = self._link_table()
        dt = self._implicit_damping_step(implicit_damping, use_damping, dt)
        if torch.is_grad_enabled() and (table.requires_grad or q0.requires_grad or qd0.requires_grad or f.requires_grad):
            out = engine.ForwardDynamicsRolloutFunction.apply(table, q0, qd0, f, self._topology, flags, dt)
        else:
            out = engine.forward_dynamics_rollout_raw(self._topology, table, q0, qd0, f, dt, flags)
        return tuple(o[:, 0] for o in out) if squeeze else tuple(out)

    def compute_contact_rollout(
        self,
        q0: torch.Tensor,
        qd0: torch.Tensor,
        f: torch.Tensor,
        link_names: List[str],
        dt: float,
        target_pos: Optional[torch.Tensor] = None,
        target_quat: Optional[torch.Tensor] = None,
        stabilization: float = 0.0,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
        position_only: bool = False,
        regularization: float = 0.0,
        implicit_damping: bool = False,
    ) -> ContactRollout:
        r"""Simulate the links held by bilateral rigid contacts: :meth:`compute_contact_dynamics` integrated over ``T`` steps
        of semi-implicit Euler, with Baumgarte stabilisation towards fixed targets, all in ONE launch
        (``csrc/contact_rollout.cu``; stated in ``include/drm_b200.h``).  From ``(q, qd) = (q0, qd0)``, step ``t`` computes in
        fp32, in this order, with ``p, R`` the links' poses and ``J`` their stacked Jacobians at ``q``, ``w = stabilization``::

            e = p - target_pos  (and, in pose mode, the world-frame rotation vector of R R_target^T)
            a_ref = -(2 * w) * (J qd) - (w * w) * e                        # w = 0: a_ref = 0, no term formed
            qdd, force, ok = compute_contact_dynamics(q, qd, f[t], link_names, a_ref, ...)
            qd = qd + dt * qdd
            q = q + dt * qd

        With ``stabilization = 0`` the result is bit-identical to that Python loop with ``accel_ref = None``.  Without
        stabilisation the integrator's drift off the constraint accumulates; ``w * dt`` of about 0.2 is a good working choice
        (``examples/pinned_end_effector_iiwa.py`` holds the Kuka end effector within a fraction of a millimetre with it).
        With ``use_damping`` the joints' damping torque ``-d qd`` enters each step at the current ``qd``, so the integrate is
        explicit in it and stable only for ``dt`` below about ``2 I / d`` (``I`` a joint's effective inertia): the Allegro
        hand's fingers (damping 3-8 N m s/rad on links of a few grams) diverge within ten steps at ``dt = 1e-3`` and at
        ``1e-4``.  Simulate them with ``implicit_damping=True``: every step's forward dynamics and force response then
        take the damping implicitly (``compute_forward_dynamics(..., implicit_damping_dt=dt)``), which is stable at any
        ``dt``.

        Args:
            q0, qd0: initial joint angles / velocities [batch_size x n_dofs] (or [n_dofs])
            f: applied joint forces of every step [T x batch_size x n_dofs] (or [T x n_dofs])
            link_names: the held links (at most 8, distinct), stacked in this order; each needs a movable joint on its
                root path
            dt: step length in seconds
            target_pos: where each link's origin is held [n_links x batch_size x 3] (``[n_links x 3]`` for 1-D ``q0``);
                None: the links' poses at ``q0``
            target_quat: in pose mode, each link's held orientation [n_links x batch_size x 4] xyzw (normalised here),
                given together with ``target_pos``; must be None with ``position_only``
            stabilization: the Baumgarte rate ``w >= 0`` [1/s]
            include_gravity, use_damping, position_only, regularization: as for :meth:`compute_contact_dynamics`
            implicit_damping: take the damping implicitly with step ``dt`` (needs ``use_damping``)
        Returns: :class:`ContactRollout` ``(q, qd, qdd, force, solved)`` with ``q[t] = q_{t+1}``, ``qd[t] = qd_{t+1}``,
        ``qdd[t] = qdd_t`` and ``force[t]`` the contact forces of step ``t``; the batch dimension is dropped for 1-D inputs.
        ``solved`` is False for a row where some step was not solved; that step and every later one of the row are NaN.
        The outputs carry no autograd graph: they use the current values of the link parameters (learnable and fused ones
        included) but are not differentiable.  Argument errors raise ``AssertionError``."""
        links = self._contact_links(link_names)
        E = len(links)
        squeeze = self._check_rollout_inputs((("q0", q0), ("qd0", qd0), ("f", f)),
                                             (("target_pos", target_pos), ("target_quat", target_quat)), "f")
        if position_only:
            assert target_quat is None, "target_quat must be None with position_only"
        else:
            assert (target_pos is None) == (target_quat is None), "give target_pos and target_quat together in pose mode"
        stabilization = float(stabilization)
        assert stabilization >= 0 and stabilization != float("inf"), "stabilization must be finite and >= 0"
        if squeeze:
            q0, qd0, f, target_pos, target_quat = self._rollout_batch_dim(q0, qd0, f, target_pos, target_quat)
        B = q0.shape[0]
        assert target_pos is None or tuple(target_pos.shape) == (E, B, 3), "target_pos must be [n_links x batch_size x 3]"
        assert target_quat is None or tuple(target_quat.shape) == (E, B, 4), "target_quat must be [n_links x batch_size x 4]"
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        flags |= engine.IMPLICIT_DAMPING if implicit_damping else 0
        dt = self._implicit_damping_step(implicit_damping, use_damping, dt)
        q, qd, qdd, force, _, solved = engine.contact_rollout_raw(
            self._topology, links, self._link_table().detach(), q0.detach(), qd0.detach(), f.detach(), dt, flags,
            None if target_pos is None else target_pos.detach(), None if target_quat is None else target_quat.detach(),
            bool(position_only), float(regularization), stabilization)
        if squeeze:
            return ContactRollout(q[:, 0], qd[:, 0], qdd[:, 0], force[:, 0], solved[0])
        return ContactRollout(q, qd, qdd, force, solved)

    def compute_pd_controlled_rollout(
        self,
        q0: torch.Tensor,
        qd0: torch.Tensor,
        q_ref: torch.Tensor,
        kp: torch.Tensor,
        kd: torch.Tensor,
        dt: float,
        qd_ref: Optional[torch.Tensor] = None,
        f: Optional[torch.Tensor] = None,
        effort_limit: Optional[torch.Tensor] = None,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
        implicit_damping: bool = False,
        implicit_gains: bool = False,
    ) -> ControlledRollout:
        r"""Simulate a joint-space PD controller tracking reference trajectories: :meth:`compute_forward_dynamics_rollout`
        with the torque of every step computed from the current state, all ``T`` steps in ONE launch
        (``csrc/rollout.cu``).  From ``(q_0, qd_0) = (q0, qd0)``, step ``t`` computes in fp32, in this order::

            u = f[t] + kp * (q_ref[t] - q) + kd * (qd_ref[t] - qd)      # qd_ref / f None: zero tensors
            u = torch.clamp(u, -effort_limit, effort_limit)             # only when effort_limit is given
            qdd = compute_forward_dynamics(q, qd, u, include_gravity, use_damping)
            qd = qd + dt * qdd
            q = q + dt * qd

        and the result is bit-identical to that Python loop on the same model; with ``implicit_damping`` (needs
        ``use_damping``) the loop's call is ``compute_forward_dynamics(q, qd, u, ..., implicit_damping_dt=dt)``, stable in
        the joint damping at any ``dt``.

        The explicit step is stable only for gains inside its own limits: for one joint of inertia ``I``, with
        ``a = dt**2 kp / I`` and ``b = dt kd / I``, it needs ``b < 2`` and ``a + 2 b < 4`` (about ``dt * sqrt(kp / I) < 0.83``
        at critical damping).  ``implicit_gains=True`` (stable PD) takes the PD law at the end-of-step state instead::

            qp = q + dt * qd                                            # the position the step predicts
            u = f[t] + kp * (q_ref[t] - qp) + kd * (qd_ref[t] - qd)
            sat = ~(-effort_limit <= u <= effort_limit)                 # all False without a limit; NaN saturates
            u = torch.where(sat, torch.clamp(u, -effort_limit, effort_limit), u)
            c = torch.where(sat, 0, dt * (kd + dt * kp))
            qdd = forward dynamics of (q, qd, u) with every joint's articulated-body pivot + c    # (H + diag(c)) qdd = u - nle
            tau = torch.where(sat, u, u - c * qdd)

        so that on an unsaturated joint ``tau = f + kp (q_ref - q_next) + kd (qd_ref - qd_next)`` (the law at the state the
        step ends in, up to rounding), and the step is stable at every ``dt`` for ``kp, kd >= 0``; the signs are not checked.
        The effort limit is decided on the predicted command: a saturated joint gets the clamped torque, and an unsaturated
        joint's applied ``tau`` can exceed the limit by ``|c * qdd|``.  It combines with ``implicit_damping``
        (``include/drm_b200.h``: ``DRMB200_IMPLICIT_GAINS``).

        Args:
            q0, qd0: initial joint angles / velocities [batch_size x n_dofs] (or [n_dofs])
            q_ref: reference joint angles of every step [T x batch_size x n_dofs] (or [T x n_dofs])
            kp, kd: diagonal proportional / derivative gains, each [n_dofs] shared by every row or [batch_size x n_dofs]
                per row (only [n_dofs] for 1-D ``q0``); one may be shared and the other per row
            dt: step length in seconds (not differentiable)
            qd_ref: reference joint velocities, shaped like ``q_ref``; None: zero
            f: feed-forward joint forces, shaped like ``q_ref``; None: zero; never modified
            effort_limit: symmetric torque limit [n_dofs], every entry > 0 (``inf`` allowed); None: no limit.
                ``get_joint_limits()[i]["effort"]`` is a natural choice, but some shipped URDFs list 0 there.
            implicit_damping: take the joint damping implicitly with step ``dt`` (needs ``use_damping``)
            implicit_gains: take the PD law at the end-of-step state (stable PD, above; needs a finite ``dt > 0``)
        Returns: :class:`ControlledRollout` ``(q, qd, qdd, tau)``, each [T x batch_size x n_dofs] (or [T x n_dofs]), with
        ``q[t] = q_{t+1}``, ``qd[t] = qd_{t+1}``, ``qdd[t] = qdd_t`` and ``tau[t]`` the torque applied at step ``t``.
        Differentiable w.r.t. q0, qd0, q_ref, qd_ref, f, kp, kd and every learnable link parameter (the articulated-body
        adjoint stepped backwards in time, the clamp passing gradients where ``-effort_limit <= u <= effort_limit``); not
        w.r.t. dt or effort_limit.  Argument errors raise ``AssertionError``."""
        squeeze = self._check_rollout_inputs((("q0", q0), ("qd0", qd0), ("q_ref", q_ref), ("kp", kp), ("kd", kd)),
                                             (("qd_ref", qd_ref), ("f", f), ("effort_limit", effort_limit)), "q_ref")
        n = self._n_dofs
        for name, t in (("qd_ref", qd_ref), ("f", f)):
            assert t is None or t.shape == q_ref.shape, f"{name} must have the shape of q_ref."
        gain_shapes = ((n,),) if q0.ndim == 1 else ((n,), tuple(q0.shape))
        for name, t in (("kp", kp), ("kd", kd)):
            assert tuple(t.shape) in gain_shapes, f"{name} must be [n_dofs] or [batch_size x n_dofs] (got {tuple(t.shape)})"
        if effort_limit is not None:
            assert tuple(effort_limit.shape) == (n,), "effort_limit must be [n_dofs]."
            # the values need a host read (a device synchronisation): done once per limit tensor and version, so a loop that
            # passes the same limit pays it once; skipped while a CUDA graph is being captured, which forbids it
            checked = getattr(self, "_checked_effort_limit", None)
            if not (checked is not None and checked[0]() is effort_limit and checked[1] == effort_limit._version) \
                    and not torch.cuda.is_current_stream_capturing():
                assert bool((effort_limit > 0).all()), "effort_limit must be > 0 (inf allowed) and not NaN."
                self._checked_effort_limit = (weakref.ref(effort_limit), effort_limit._version)
        if squeeze:
            q0, qd0, q_ref, qd_ref, f = self._rollout_batch_dim(q0, qd0, q_ref, qd_ref, f)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        flags |= engine.IMPLICIT_DAMPING if implicit_damping else 0
        flags |= engine.IMPLICIT_GAINS if implicit_gains else 0
        table = self._link_table()
        dt = self._implicit_damping_step(implicit_damping, use_damping, dt)
        if implicit_gains:
            assert 0.0 < dt < float("inf"), f"implicit gains need a finite step dt > 0 (got {dt})"
        lim = None if effort_limit is None else effort_limit.detach()
        if kp.shape != kd.shape:
            # the kernel reads both gains in one layout: the shared one becomes a per-row view (its gradient is the sum of
            # the per-row ones, through the expand's backward)
            kp, kd = kp.expand(q0.shape), kd.expand(q0.shape)
        diff = (table, q0, qd0, q_ref, qd_ref, f, kp, kd)
        if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in diff):
            out = engine.PDRolloutFunction.apply(*diff, self._topology, flags, dt, lim)
        else:
            out = engine.pd_rollout_raw(self._topology, table, q0, qd0, q_ref, kp, kd, dt, flags, qd_ref, f, lim)
        return ControlledRollout(*(o[:, 0] for o in out)) if squeeze else ControlledRollout(*out)

    @tensor_check
    def compute_forward_dynamics_crba(
        self,
        q: torch.Tensor,
        qd: torch.Tensor,
        f: torch.Tensor,
        include_gravity: Optional[bool] = True,
        use_damping: Optional[bool] = False,
    ) -> torch.Tensor:
        r"""Forward dynamics as ``H(q)^-1 (f - nle(q, qd))``: n + 2 stacked RNEA evaluations (two launches) and a
        batched ``torch.linalg.solve``.  Equal to :meth:`compute_forward_dynamics` when every ``inertia_mat`` is
        symmetric; kept as an independent cross-check of the articulated-body kernel."""
        self._check_q(q, qd, f)
        nle = self.compute_inverse_dynamics(q, qd, torch.zeros_like(q), include_gravity, use_damping)
        H = self.compute_lagrangian_inertia_matrix(q, include_gravity=False, use_damping=False)
        return torch.linalg.solve(H, (f - nle).unsqueeze(2)).squeeze(2)

    @tensor_check
    def update_kinematic_state(self, q: torch.Tensor, qd: torch.Tensor) -> None:
        r"""World pose and body-frame spatial velocity of every link for joint state ``(q, qd)``
        (``robot_model.py:140-195``).  Afterwards ``model._bodies[i].pose`` (a ``CoordinateTransform``) and
        ``model._bodies[i].vel`` (a ``SpatialMotionVec``) are available like in the reference.  The fused FK / RNEA kernels
        write no per-link state to HBM, so this only RECORDS the joint state; the first access of a body's ``pose`` /
        ``vel`` runs ONE launch of the all-links kernel (``csrc/kinematic_state.cu``) and later accesses are views of its
        link-major output.  ``compute_inverse_dynamics`` records its ``(q, qd)`` the same way (the reference updates the
        kinematic state as a side effect there, ``robot_model.py:335``).  This state is not differentiable."""
        self._check_q(q, qd)
        self._kin_inputs = (q.detach(), qd.detach())
        self._kin_state = None
        return

    def _kinematic_state(self):
        if getattr(self, "_kin_state", None) is None:
            inputs = getattr(self, "_kin_inputs", None)
            if inputs is None:
                raise RuntimeError("no kinematic state: call update_kinematic_state(q, qd) first")
            with torch.no_grad():
                poses, _, vels = engine.kinematic_state_raw(self._topology, self._link_table().detach(), *inputs)
            self._kin_state = (poses, vels)
        return self._kin_state

    def _body_pose(self, i):
        from .spatial_vector_algebra import CoordinateTransform
        block = self._kinematic_state()[0][i]                     # [12, B]
        return CoordinateTransform(rot=block[:9].t().reshape(-1, 3, 3), trans=block[9:12].t().contiguous(),
                                   device=self._device)

    def _body_vel(self, i):
        from .spatial_vector_algebra import SpatialMotionVec
        block = self._kinematic_state()[1][i]                     # [6, B]: ang, lin
        return SpatialMotionVec(lin_motion=block[3:6].t().contiguous(), ang_motion=block[0:3].t().contiguous())

    @tensor_check
    def compute_forward_kinematics_all_links(self, q: torch.Tensor) -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
        r"""``{link_name: (pos, quat)}`` for every link (``robot_model.py:198-221``) from ONE launch of the all-links
        kernel.  Differentiable w.r.t. ``q`` and every learnable link parameter, like the reference's recursion (the
        adjoint runs the single-link FK backward kernel once per link that received a gradient).
        Like the reference, 1-D inputs give un-squeezed ``[1, .]`` values (the dict bypasses the squeeze)."""
        self._check_q(q)
        table = self._link_table()
        if torch.is_grad_enabled() and (q.requires_grad or table.requires_grad):
            pos, quat = engine.AllLinksFkFunction.apply(table, q, self._topology)
        else:
            poses, quats, _ = engine.kinematic_state_raw(self._topology, table, q, None, want_poses=True, want_quats=True)
            pos, quat = poses[:, 9:12].transpose(1, 2), quats.transpose(1, 2)
        return {name: (pos[i].contiguous(), quat[i].contiguous()) for i, name in enumerate(self.get_link_names())}

    # per-body dynamic state (reference: `_bodies[i].acc / .force` after compute_inverse_dynamics, robot_model.py:262-301)
    def _remember_dynamic_inputs(self, q, qd, qdd, flags):
        self._dyn_inputs = (q.detach(), qd.detach(), qdd.detach(), flags & (engine.GRAVITY | engine.DAMPING))
        self._dyn_state = None
        self._kin_inputs = (q.detach(), qd.detach())               # robot_model.py:335: update_kinematic_state(q, qd)
        self._kin_state = None

    def _dynamic_state(self):
        """(vels, accs, forces) blocks [N, 6, B] for the inputs of the last compute_inverse_dynamics call: ONE launch of
        the dump variant of the RNEA kernel, issued on first access (the fused kernel itself writes no per-link state)."""
        if getattr(self, "_dyn_state", None) is None:
            inputs = getattr(self, "_dyn_inputs", None)
            if inputs is None:
                raise RuntimeError("no dynamic state: call compute_inverse_dynamics(q, qd, qdd) first")
            q, qd, qdd, flags = inputs
            with torch.no_grad():
                _, vels, accs, forces = engine.dynamic_state_raw(self._topology, self._link_table().detach(), q, qd, qdd,
                                                                 flags, want_tau=False)
            self._dyn_state = (vels, accs, forces)
        return self._dyn_state

    def _body_acc(self, i):
        from .spatial_vector_algebra import SpatialMotionVec
        block = self._dynamic_state()[1][i]                      # [6, B]: ang, lin
        return SpatialMotionVec(lin_motion=block[3:6].t().contiguous(), ang_motion=block[0:3].t().contiguous())

    def _body_force(self, i):
        from .spatial_vector_algebra import SpatialForceVec
        block = self._dynamic_state()[2][i]                      # [6, B]: torque, force
        return SpatialForceVec(lin_force=block[3:6].t().contiguous(), ang_force=block[0:3].t().contiguous())

    # ------------------------------------------------------------------------------------------
    # learnable link parameters (robot_model.py:669-713)
    # ------------------------------------------------------------------------------------------
    def _get_parent_object_of_param(self, link_name: str, parameter_name: str):
        body_idx = self._name_to_idx_map[link_name]
        if parameter_name in ["trans", "rot_angles", "joint_damping"]:
            return self._bodies[body_idx]
        if parameter_name in ["mass", "inertia_mat", "com"]:
            return self._bodies[body_idx].inertia
        raise AttributeError(
            "Invalid parameter name. Accepted parameter names are: "
            "trans, rot_angles, joint_damping, mass, inertia_mat, com"
        )

    def make_link_param_learnable(self, link_name: str, parameter_name: str, parametrization: torch.nn.Module):
        owner = self._get_parent_object_of_param(link_name, parameter_name)
        owner.__delattr__(parameter_name)
        owner.add_module(parameter_name, parametrization.to(self._device))
        if getattr(self, "fused_link_params", None) is not None:
            raise RuntimeError("make_link_param_learnable after fuse_learnable_parameters(): fuse once, after the last one")
        self.invalidate_link_table()

    def _learnable_module(self, link_name: str, parameter_name: str):
        owner = self._get_parent_object_of_param(link_name, parameter_name)
        module = getattr(owner, parameter_name)
        assert isinstance(module, torch.nn.Module), f"{parameter_name} of {link_name} is not a learnable module."
        return module

    def _set_learnable_link_param_frozen(self, link_name: str, parameter_name: str, frozen: bool):
        module = self._learnable_module(link_name, parameter_name)
        if getattr(self, "fused_link_params", None) is not None:
            raise RuntimeError("freeze / unfreeze_learnable_link_param after fuse_learnable_parameters(): the flat vector "
                               "holds what was unfrozen when it was built; freeze before fusing")
        for param in module.parameters():
            param.requires_grad = not frozen

    def freeze_learnable_link_param(self, link_name: str, parameter_name: str):
        """Stop learning this link parameter: its module keeps its value and gets no gradient.  A module installed on
        several links is frozen on all of them.  Call before ``fuse_learnable_parameters`` (raises ``RuntimeError``
        after): a frozen module's value becomes a constant of the fused table."""
        self._set_learnable_link_param_frozen(link_name, parameter_name, True)

    def unfreeze_learnable_link_param(self, link_name: str, parameter_name: str):
        """Undo ``freeze_learnable_link_param`` (raises ``RuntimeError`` after ``fuse_learnable_parameters``)."""
        self._set_learnable_link_param_frozen(link_name, parameter_name, False)

    # ------------------------------------------------------------------------------------------
    # introspection (robot_model.py:715-754)
    # ------------------------------------------------------------------------------------------
    def get_joint_limits(self) -> List[Dict[str, torch.Tensor]]:
        return [self._bodies[idx].get_joint_limits() for idx in self._controlled_joints]

    def get_link_names(self) -> List[str]:
        return [body.name for body in self._bodies]

    def print_link_names(self) -> None:
        for body in self._bodies:
            print(body.name)

    def print_learnable_params(self) -> None:
        for name, param in self.named_parameters():
            print(f"{name}: {param}")


class DifferentiableKUKAiiwa(DifferentiableRobotModel):
    def __init__(self, device=None):
        self.urdf_path = os.path.join(robot_description_folder, "kuka_iiwa/urdf/iiwa7.urdf")
        self.learnable_rigid_body_config = None
        super().__init__(self.urdf_path, "differentiable_kuka_iiwa", device=device)


class DifferentiableFrankaPanda(DifferentiableRobotModel):
    def __init__(self, device=None):
        self.urdf_path = os.path.join(robot_description_folder, "panda_description/urdf/panda_no_gripper.urdf")
        self.learnable_rigid_body_config = None
        super().__init__(self.urdf_path, "differentiable_franka_panda", device=device)


class DifferentiableTwoLinkRobot(DifferentiableRobotModel):
    def __init__(self, device=None):
        self.urdf_path = os.path.join(robot_description_folder, "2link_robot.urdf")
        self.learnable_rigid_body_config = None
        super().__init__(self.urdf_path, "diff_2d_robot", device=device)


class DifferentiableTrifingerEdu(DifferentiableRobotModel):
    def __init__(self, device=None):
        self.urdf_path = os.path.join(robot_description_folder, "trifinger_edu_description/trifinger_edu.urdf")
        self.learnable_rigid_body_config = None
        super().__init__(self.urdf_path, "trifinger_edu", device=device)
