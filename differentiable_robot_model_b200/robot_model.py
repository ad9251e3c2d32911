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
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

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
        after the last ``make_link_param_learnable``; values and gradients are the same as on the per-module path (the
        modules' own Parameters become views of the flat storage and stop requiring grad).  Raises ``ValueError`` for
        parametrisations other than UnconstrainedScalar / UnconstrainedTensor / PositiveScalar."""
        if self._device.type != "cuda":
            raise RuntimeError("fuse_learnable_parameters needs a CUDA model")
        self.fused_link_params = None
        self.fused_link_params = FusedLinkParameters(self._bodies, self._device)
        return self.fused_link_params.flat

    def _kinematic_params_learnable(self) -> bool:
        """True if any joint origin (``trans`` / ``rot_angles`` of a movable link) is a learnable module with a
        parameter that requires grad -- then the backward kernels must produce the F / r columns of the table
        gradient; otherwise the RNEA backward can take the single-sweep inertial path."""
        for body in self._bodies:
            if body.joint_idx is None:
                continue
            for name in ("trans", "rot_angles"):
                attr = getattr(body, name)
                if isinstance(attr, torch.nn.Module):
                    params = list(attr.parameters())
                    fused = getattr(self, "fused_link_params", None)
                    if fused is not None and params:                            # views of the flat vector
                        if fused.flat.requires_grad:
                            return True
                        continue
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
    ) -> torch.Tensor:
        r"""Joint accelerations under applied joint forces ``f``: the articulated-body algorithm of
        ``robot_model.py:488-624`` in ONE launch (``csrc/aba.cu``), with the reference's arithmetic (general 6x6
        articulated inertias -- ``inertia_mat`` is never symmetrised --, ``+1e-37`` regularisers).  Differentiable
        w.r.t. q, qd, f and every learnable link parameter through the analytic adjoint kernel.  Unlike the reference
        this does not overwrite the caller's ``f`` when ``use_damping`` is set (``robot_model.py:521``)."""
        self._check_q(q, qd, f)
        flags = (engine.GRAVITY if include_gravity else 0) | (engine.DAMPING if use_damping else 0)
        return engine.ForwardDynamicsFunction.apply(self._link_table(), q, qd, f, self._topology, flags, self._folded_table())

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

    def freeze_learnable_link_param(self, link_name: str, parameter_name: str):
        for param in self._learnable_module(link_name, parameter_name).parameters():
            param.requires_grad = False

    def unfreeze_learnable_link_param(self, link_name: str, parameter_name: str):
        for param in self._learnable_module(link_name, parameter_name).parameters():
            param.requires_grad = True

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
