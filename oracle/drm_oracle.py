"""TEST INFRASTRUCTURE -- CPU oracle for the FK / Jacobian / inverse-dynamics hot path.

This is a restatement, in plain batched torch (CPU, fp32 or fp64), of the algorithm the reference
implements with per-link ``nn.Module`` state.  It exists to CHECK the CUDA engine; only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import
it, and never as the thing measured or shipped.  It does not import the product package.

Parity pinning: the reference ships no golden vectors (its tests compare against live pybullet,
which is not installable here), so the oracle is pinned against outputs of the reference itself:
``tests/golden/make_golden.py`` imports ``/root/reference`` unmodified (via ``oracle/refshim``) in the
build container and stores seeded inputs / outputs / autograd gradients under ``tests/golden/``;
``tests/test_oracle.py`` checks this file against them (and against the known answers in
SURVEY.md section 8c).

Reference lines followed (relative to /root/reference/differentiable_robot_model/):
  load_robot              urdf_utils.py:28-126, robot_model.py:114-137
  joint_transform         rigid_body.py:130-157, spatial_vector_algebra.py:14-53
  kinematic_state         robot_model.py:140-195, spatial_vector_algebra.py:92-106, 226-236
  quaternion              spatial_vector_algebra.py:108-136
  forward_kinematics      robot_model.py:224-248
  jacobian                robot_model.py:627-667
  inverse_dynamics        robot_model.py:251-375, spatial_vector_algebra.py:204-224, 281-291, 321-338
  dynamic_state           robot_model.py:183-193, 262-301 (the per-link state inverse_dynamics computes)
"""
import os
import sys
from dataclasses import dataclass, field
from typing import List, Optional

import torch

_SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "refshim")


def _urdf_class():
    if _SHIM not in sys.path:
        sys.path.insert(0, _SHIM)
    from urdf_parser_py.urdf import URDF
    return URDF


@dataclass
class Robot:
    """Per-link parameters in URDF document order (= reference body index order)."""
    names: List[str]
    parent: List[int]                 # -1 for the root
    dof: List[int]                    # joint index or -1 for fixed joints
    joint_type: List[str]
    limits: List[Optional[dict]]
    axis: torch.Tensor                # [N,3]
    trans: torch.Tensor               # [N,3]
    rpy: torch.Tensor                 # [N,3]
    mass: torch.Tensor                # [N]
    com: torch.Tensor                 # [N,3]
    inertia: torch.Tensor             # [N,3,3]
    damping: torch.Tensor             # [N]
    n_dofs: int = 0
    controlled: List[int] = field(default_factory=list)

    def index(self, name):
        return self.names.index(name)

    def to(self, dtype):
        kw = {k: getattr(self, k).to(dtype) for k in ("axis", "trans", "rpy", "mass", "com", "inertia", "damping")}
        return Robot(self.names, self.parent, self.dof, self.joint_type, self.limits, n_dofs=self.n_dofs,
                     controlled=self.controlled, **kw)


def load_robot(urdf_path, dtype=torch.float32):
    """URDF -> Robot.  Values are read as float32 first (the reference stores fp32 constants,
    urdf_utils.py:48-53,86-97) and then widened, so an fp64 oracle sees the same numbers."""
    urdf = _urdf_class().from_xml_file(urdf_path)
    child_joint = {}
    for j in urdf.joints:
        child_joint.setdefault(j.child, j)
    names = [l.name for l in urdf.links]
    N = len(names)
    parent, dof, jtype, limits = [-1] * N, [-1] * N, ["fixed"] * N, [None] * N
    axis, trans, rpy = torch.zeros(N, 3), torch.zeros(N, 3), torch.zeros(N, 3)
    mass, com, inertia, damping = torch.ones(N), torch.zeros(N, 3), torch.eye(3).repeat(N, 1, 1), torch.zeros(N)
    n_dofs, controlled = 0, []
    for i, link in enumerate(urdf.links):
        if i > 0:                                              # link 0 is the root (urdf_utils.py:33-40)
            j = child_joint[link.name]
            parent[i] = names.index(j.parent)
            trans[i] = torch.tensor(j.origin.position, dtype=torch.float32)
            rpy[i] = torch.tensor(j.origin.rotation, dtype=torch.float32)
            jtype[i] = j.type
            if j.type != "fixed":                              # prismatic / continuous == revolute (robot_model.py:123)
                dof[i] = n_dofs
                n_dofs += 1
                controlled.append(i)
                axis[i] = torch.tensor(j.axis, dtype=torch.float32)
                limits[i] = dict(effort=j.limit.effort, lower=j.limit.lower, upper=j.limit.upper,
                                 velocity=j.limit.velocity)
                damping[i] = j.dynamics.damping if j.dynamics is not None else 0.0
        if link.inertial is not None:
            mass[i] = link.inertial.mass
            com[i] = torch.tensor(link.inertial.origin.position, dtype=torch.float32)
            I = link.inertial.inertia
            inertia[i] = torch.tensor([[I.ixx, I.ixy, I.ixz], [I.ixy, I.iyy, I.iyz], [I.ixz, I.iyz, I.izz]],
                                      dtype=torch.float32)
    robot = Robot(names, parent, dof, jtype, limits, axis, trans, rpy, mass, com, inertia, damping,
                  n_dofs=n_dofs, controlled=controlled)
    return robot.to(dtype)


# ------------------------------------------------------------------------------------------------
def _elem_rot(k, angle):
    """x_rot / y_rot / z_rot (spatial_vector_algebra.py:14-53) for angle [B] -> [B,3,3]."""
    c, s = torch.cos(angle), torch.sin(angle)
    one, zero = torch.ones_like(c), torch.zeros_like(c)
    if k == 0:
        rows = [one, zero, zero, zero, c, -s, zero, s, c]
    elif k == 1:
        rows = [c, zero, s, zero, one, zero, -s, zero, c]
    else:
        rows = [c, -s, zero, s, c, zero, zero, zero, one]
    return torch.stack(rows, dim=-1).reshape(-1, 3, 3)


def _skew(v):
    """vector3_to_skew_symm_matrix (utils.py:40-50), v [B,3] -> [B,3,3]."""
    z = torch.zeros_like(v[:, 0])
    return torch.stack([z, -v[:, 2], v[:, 1], v[:, 2], z, -v[:, 0], -v[:, 1], v[:, 0], z], dim=-1).reshape(-1, 3, 3)


def _cross(a, b):
    """cross_product via skew matmul (utils.py:21-25)."""
    return (_skew(a) @ b.unsqueeze(2)).squeeze(2)


def joint_transform(robot, i, q):
    """Joint pose of link i: (R [B,3,3], t [1,3]) -- rigid_body.py:138-156."""
    roll, pitch, yaw = robot.rpy[i, 0:1], robot.rpy[i, 1:2], robot.rpy[i, 2:3]
    fixed = (_elem_rot(2, yaw) @ _elem_rot(1, pitch)) @ _elem_rot(0, roll)         # [1,3,3]
    if robot.dof[i] < 0:
        angle = torch.zeros(q.shape[0], dtype=q.dtype)           # ctor state of fixed joints (rigid_body.py:64-67)
        k, sign = 2, 0.0
    else:
        ax = robot.axis[i]
        if abs(float(ax[0])) == 1:
            k = 0
        elif abs(float(ax[1])) == 1:
            k = 1
        else:
            k = 2
        sign = torch.sign(ax[k])
        angle = sign * q[:, robot.dof[i]]
    return fixed @ _elem_rot(k, angle), robot.trans[i:i + 1]


def kinematic_state(robot, q, qd=None):
    """World poses (R, p) and body-frame spatial velocities (ang, lin) of every link
    (update_kinematic_state, robot_model.py:140-195)."""
    B = q.shape[0]
    if qd is None:
        qd = torch.zeros_like(q)
    eye = torch.eye(3, dtype=q.dtype).expand(B, 3, 3)
    zeros = torch.zeros(B, 3, dtype=q.dtype)
    R, p, w, v, joints = [eye], [zeros], [zeros], [zeros], [None]
    for i in range(1, len(robot.names)):
        par = robot.parent[i]
        Rj, tj = joint_transform(robot, i, q)
        joints.append((Rj, tj))
        # pose = parent.pose o joint_pose (spatial_vector_algebra.py:98-103)
        R.append(R[par] @ Rj)
        p.append((R[par] @ tj.expand(B, 3).unsqueeze(2)).squeeze(2) + p[par])
        # velocity: parent velocity transformed by the inverse joint pose (sva:92-96, 226-236) + joint velocity
        Rt = Rj.transpose(-2, -1)
        tinv = -(Rt @ tj.expand(B, 3).unsqueeze(2)).squeeze(2)
        new_ang = (Rt @ w[par].unsqueeze(2)).squeeze(2)
        new_lin = ((_skew(tinv) @ Rt) @ w[par].unsqueeze(2)).squeeze(2) + (Rt @ v[par].unsqueeze(2)).squeeze(2)
        jw = qd[:, robot.dof[i]:robot.dof[i] + 1] @ robot.axis[i:i + 1] if robot.dof[i] >= 0 else zeros
        w.append(jw + new_ang)
        v.append(new_lin)
    return R, p, w, v, joints


def quaternion(R):
    """xyzw quaternion with the branch structure of get_quaternion (spatial_vector_algebra.py:108-136),
    vectorised over the batch (the reference loops over batch elements in Python)."""
    d0, d1, d2 = R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]
    tr = d0 + d1 + d2
    one = torch.ones_like(tr)
    case_a = tr + one > one                                      # "tn > M[3,3]" with tn = trace(M), M[3,3] = 1
    i2 = (~case_a) & (d2 > torch.maximum(d0, d1))
    i1 = (~case_a) & (~i2) & (d1 > d0)
    i0 = (~case_a) & (~i2) & (~i1)
    qa = torch.stack([R[:, 2, 1] - R[:, 1, 2], R[:, 0, 2] - R[:, 2, 0], R[:, 1, 0] - R[:, 0, 1], tr + 1], dim=1)
    t0 = d0 - (d1 + d2) + 1
    q0 = torch.stack([t0, R[:, 0, 1] + R[:, 1, 0], R[:, 2, 0] + R[:, 0, 2], R[:, 2, 1] - R[:, 1, 2]], dim=1)
    t1 = d1 - (d2 + d0) + 1
    q1 = torch.stack([R[:, 0, 1] + R[:, 1, 0], t1, R[:, 1, 2] + R[:, 2, 1], R[:, 0, 2] - R[:, 2, 0]], dim=1)
    t2 = d2 - (d0 + d1) + 1
    q2 = torch.stack([R[:, 2, 0] + R[:, 0, 2], R[:, 1, 2] + R[:, 2, 1], t2, R[:, 1, 0] - R[:, 0, 1]], dim=1)
    t = torch.where(case_a, tr + 1, torch.where(i2, t2, torch.where(i1, t1, t0)))
    qq = torch.where(case_a[:, None], qa, torch.where(i2[:, None], q2, torch.where(i1[:, None], q1, q0)))
    assert bool((case_a | i0 | i1 | i2).all())
    return qq * (0.5 / torch.sqrt(t))[:, None]


def quaternion_per_element(R):
    """The reference's get_quaternion AS SHIPPED: a Python loop over batch elements with data-dependent branches
    (spatial_vector_algebra.py:116-135).  Only for small samples -- it is what makes the shipped
    compute_forward_kinematics / compute_endeffector_jacobian run at ~10 k configurations/s on a CPU."""
    import math
    B = R.shape[0]
    out = torch.empty(B, 4, dtype=R.dtype)
    for b in range(B):
        m = R[b]
        tr = m[0, 0] + m[1, 1] + m[2, 2] + 1
        if tr > 1:
            t = tr
            vals = {3: t, 2: m[1, 0] - m[0, 1], 1: m[0, 2] - m[2, 0], 0: m[2, 1] - m[1, 2]}
        else:
            i, j, k = 0, 1, 2
            if m[1, 1] > m[0, 0]:
                i, j, k = 1, 2, 0
            if m[2, 2] > m[i, i]:
                i, j, k = 2, 0, 1
            t = m[i, i] - (m[j, j] + m[k, k]) + 1
            vals = {i: t, j: m[i, j] + m[j, i], k: m[k, i] + m[i, k], 3: m[k, j] - m[j, k]}
        scale = 0.5 / math.sqrt(float(t))
        for c in range(4):
            out[b, c] = vals[c] * scale
    return out


def forward_kinematics(robot, q, link_name):
    R, p, _, _, _ = kinematic_state(robot, q)
    i = robot.index(link_name)
    return p[i], quaternion(R[i])


def jacobian(robot, q, link_name):
    """Geometric Jacobian in the world frame (robot_model.py:627-667): columns of joints on the
    ee->root path are z x (p_e - p_i) / z, the rest zero."""
    R, p, _, _, _ = kinematic_state(robot, q)
    B = q.shape[0]
    e = robot.index(link_name)
    lin = torch.zeros(B, 3, robot.n_dofs, dtype=q.dtype)
    ang = torch.zeros(B, 3, robot.n_dofs, dtype=q.dtype)
    lin_cols, ang_cols = {}, {}
    i = e
    while i > 0:
        if robot.dof[i] >= 0:
            z = R[i] @ robot.axis[i]
            lin_cols[robot.dof[i]] = torch.cross(z, p[e] - p[i], dim=-1)
            ang_cols[robot.dof[i]] = z
        i = robot.parent[i]
    zero = torch.zeros(B, 3, dtype=q.dtype)
    lin = torch.stack([lin_cols.get(k, zero) for k in range(robot.n_dofs)], dim=2)
    ang = torch.stack([ang_cols.get(k, zero) for k in range(robot.n_dofs)], dim=2)
    return lin, ang


def _inertia_times(robot, i, ang, lin):
    """multiply_motion_vec (spatial_vector_algebra.py:321-338) -> (lin_force, ang_force)."""
    m, c, Ic = robot.mass[i], robot.com[i:i + 1], robot.inertia[i:i + 1]
    mcom = c * m
    S = _skew(c)
    Io = Ic + m * (S @ S.transpose(-2, -1))
    B = ang.shape[0]
    f_lin = m * lin - _cross(mcom.expand(B, 3), ang)
    f_ang = (Io.expand(B, 3, 3) @ ang.unsqueeze(2)).squeeze(2) + _cross(mcom.expand(B, 3), lin)
    return f_lin, f_ang


def inverse_dynamics(robot, q, qd, qdd, include_gravity=True, use_damping=True):
    """RNEA (robot_model.py:251-375)."""
    return _rnea(robot, q, qd, qdd, include_gravity, use_damping)["tau"]


def dynamic_state(robot, q, qd, qdd, include_gravity=True, use_damping=True):
    """The per-link state the reference leaves in its bodies after compute_inverse_dynamics (robot_model.py:183-193,
    262-301), from the same evaluation as inverse_dynamics: dict of [N, B, 3] tensors "vel_ang", "vel_lin" (body-frame
    spatial velocity), "acc_ang", "acc_lin" (al, a: spatial acceleration, gravity as a base acceleration),
    "force_ang", "force_lin" (body wrench with the wrenches of all descendants accumulated), plus "tau" [B, n]."""
    s = _rnea(robot, q, qd, qdd, include_gravity, use_damping)
    return {k: (v if k == "tau" else torch.stack(v)) for k, v in s.items()}


def _rnea(robot, q, qd, qdd, include_gravity, use_damping):
    B = q.shape[0]
    N = len(robot.names)
    R, p, w, v, joints = kinematic_state(robot, q, qd)
    zeros = torch.zeros(B, 3, dtype=q.dtype)
    g = torch.zeros(B, 3, dtype=q.dtype)
    if include_gravity:
        g = torch.stack([zeros[:, 0], zeros[:, 0], 9.81 * torch.ones(B, dtype=q.dtype)], dim=1)
    al, a = [zeros], [g]
    for i in range(1, N):
        par = robot.parent[i]
        Rj, tj = joints[i]
        Rt = Rj.transpose(-2, -1)
        tinv = -(Rt @ tj.expand(B, 3).unsqueeze(2)).squeeze(2)
        acc_ang = (Rt @ al[par].unsqueeze(2)).squeeze(2)
        acc_lin = ((_skew(tinv) @ Rt) @ al[par].unsqueeze(2)).squeeze(2) + (Rt @ a[par].unsqueeze(2)).squeeze(2)
        if robot.dof[i] >= 0:
            jw = qd[:, robot.dof[i]:robot.dof[i] + 1] @ robot.axis[i:i + 1]
            ja = qdd[:, robot.dof[i]:robot.dof[i] + 1] @ robot.axis[i:i + 1]
        else:
            jw, ja = zeros, zeros
        # body.vel x joint_vel (cross_motion_vec, sva:204-213); joint_vel.lin == 0
        al.append(acc_ang + ja + _cross(w[i], jw))
        a.append(acc_lin + _cross(v[i], jw))
    f_lin = [zeros for _ in range(N)]
    f_ang = [zeros for _ in range(N)]
    for i in range(N - 1, 0, -1):
        Rj, tj = joints[i]
        ia_lin, ia_ang = _inertia_times(robot, i, al[i], a[i])
        iv_lin, iv_ang = _inertia_times(robot, i, w[i], v[i])
        # cross_force_vec (sva:215-224)
        f_lin[i] = f_lin[i] + ia_lin + _cross(w[i], iv_lin)
        f_ang[i] = f_ang[i] + ia_ang + _cross(w[i], iv_ang) + _cross(v[i], iv_lin)
        par = robot.parent[i]
        # SpatialForceVec.transform by the joint pose (sva:281-291)
        new_lin = (Rj @ f_lin[i].unsqueeze(2)).squeeze(2)
        new_ang = ((_skew(tj.expand(B, 3)) @ Rj) @ f_lin[i].unsqueeze(2)).squeeze(2) + (Rj @ f_ang[i].unsqueeze(2)).squeeze(2)
        f_lin[par] = f_lin[par] + new_lin
        f_ang[par] = f_ang[par] + new_ang
    cols = []
    for i in robot.controlled:
        ax = robot.axis[i]
        k = int(torch.where(ax != 0)[0])                          # robot_model.py:357
        cols.append(torch.sign(ax[k]) * f_ang[i][:, k])
    tau = torch.stack(cols, dim=1) if cols else q.new_zeros(B, 0)
    if use_damping and cols:
        tau = tau + torch.stack([robot.damping[i] for i in robot.controlled]).unsqueeze(0) * qd
    return {"tau": tau, "vel_ang": w, "vel_lin": v, "acc_ang": al, "acc_lin": a, "force_ang": f_ang, "force_lin": f_lin}


def _spatial_inertia(robot, i):
    """get_spatial_mat (spatial_vector_algebra.py:340-372): 6x6 in [ang; lin] order, NOT symmetrised."""
    m, c, Ic = robot.mass[i], robot.com[i], robot.inertia[i]
    S = _skew(c.unsqueeze(0))[0]
    Io = Ic + m * (S @ S.t())
    Smc = _skew((m * c).unsqueeze(0))[0]
    top = torch.cat([Io, Smc], dim=1)
    bot = torch.cat([Smc.t(), m * torch.eye(3, dtype=Ic.dtype)], dim=1)
    return torch.cat([top, bot], dim=0)


def _motion_matrix(Rj, tj):
    """CoordinateTransform.to_matrix (spatial_vector_algebra.py:138-154): [[R^T, 0], [-R^T t^, R^T]]."""
    B = Rj.shape[0]
    Rt = Rj.transpose(-2, -1)
    top = torch.cat([Rt, torch.zeros(B, 3, 3, dtype=Rj.dtype)], dim=2)
    bot = torch.cat([-(Rt @ _skew(tj.expand(B, 3))), Rt], dim=2)
    return torch.cat([top, bot], dim=1)


def forward_dynamics(robot, q, qd, f, include_gravity=True, use_damping=False):
    """Articulated-body algorithm exactly as the reference evaluates it (robot_model.py:488-624), including its
    use of the COLUMN U = IA S in both the rank-1 update and the joint-acceleration formula (so for a
    non-symmetric inertia_mat the result is the reference's, not H^-1 (f - nle)), the +1e-37 regularisers
    (:570, :582) and zero-axis "joints" for fixed links.  The reference additionally overwrites the caller's f
    in place when use_damping is set (:521); this restatement leaves f untouched.
    Spatial vectors are [ang; lin] (get_vector, sva:238-239)."""
    B = q.shape[0]
    N = len(robot.names)
    dt = q.dtype
    if use_damping:
        f = f - torch.stack([robot.damping[i] for i in robot.controlled]).unsqueeze(0) * qd
    R, p, w, v, joints = kinematic_state(robot, q, qd)
    zeros = torch.zeros(B, 3, dtype=dt)
    g = torch.stack([zeros[:, 0], zeros[:, 0], (9.81 if include_gravity else 0.0) * torch.ones(B, dtype=dt)], dim=1)
    c, pA, IA = [None] * N, [None] * N, [None] * N
    for i in range(1, N):
        jw = qd[:, robot.dof[i]:robot.dof[i] + 1] @ robot.axis[i:i + 1] if robot.dof[i] >= 0 else zeros
        c[i] = torch.cat([_cross(w[i], jw), _cross(v[i], jw)], dim=1)            # cross_motion_vec, joint_vel.lin = 0
        h_lin, h_ang = _inertia_times(robot, i, w[i], v[i])
        pA[i] = torch.cat([_cross(w[i], h_ang) + _cross(v[i], h_lin), _cross(w[i], h_lin)], dim=1)   # cross_force_vec
        IA[i] = _spatial_inertia(robot, i).unsqueeze(0).repeat(B, 1, 1)
    U, d, u = [None] * N, [None] * N, [None] * N
    for i in range(N - 1, 0, -1):
        S = torch.cat([robot.axis[i:i + 1].expand(B, 3), zeros], dim=1)          # joint axis, zero for fixed links
        U[i] = (IA[i] @ S.unsqueeze(2)).squeeze(2)
        d[i] = (S * U[i]).sum(-1)
        u[i] = -(pA[i] * S).sum(-1)
        if robot.dof[i] >= 0:
            u[i] = f[:, robot.dof[i]] + u[i]
        par = robot.parent[i]
        if par > 0:
            Ud = U[i] / (d[i].unsqueeze(1) + 1e-37)
            IAi = IA[i] - U[i].unsqueeze(2) @ Ud.unsqueeze(1)
            pa = pA[i] + (IAi @ c[i].unsqueeze(2)).squeeze(2) + U[i] * (u[i] / (d[i] + 1e-37)).unsqueeze(1)
            Rj, tj = joints[i]
            X = _motion_matrix(Rj, tj)
            IA[par] = IA[par] + X.transpose(-2, -1) @ IAi @ X
            # SpatialForceVec.transform by the joint pose (sva:281-291)
            pl = (Rj @ pa[:, 3:].unsqueeze(2)).squeeze(2)
            pg = ((_skew(tj.expand(B, 3)) @ Rj) @ pa[:, 3:].unsqueeze(2)).squeeze(2) + (Rj @ pa[:, :3].unsqueeze(2)).squeeze(2)
            pA[par] = pA[par] + torch.cat([pg, pl], dim=1)
    acc = [torch.cat([zeros, g], dim=1)] + [None] * (N - 1)
    cols = [None] * robot.n_dofs
    for i in range(1, N):
        Rj, tj = joints[i]
        X = _motion_matrix(Rj, tj)                                               # transform by the inverse joint pose
        a = (X @ acc[robot.parent[i]].unsqueeze(2)).squeeze(2) + c[i]
        if robot.dof[i] >= 0:
            qdd_i = (1.0 / d[i]) * (u[i] - (U[i] * a).sum(-1))
            cols[robot.dof[i]] = qdd_i
            a = a + torch.cat([robot.axis[i:i + 1].expand(B, 3), zeros], dim=1) * qdd_i.unsqueeze(1)
        acc[i] = a
    return torch.stack(cols, dim=1)


def sample_inputs(robot, batch, seed=0, dtype=torch.float32, vel_scale=0.2, acc_scale=0.4):
    """Seeded synthetic inputs: q ~ U(joint limits), qd ~ U(+-0.2 vel_limit), qdd ~ U(+-0.4 vel_limit)
    (BASELINE.md section 3; ranges of data_utils.py:76-98)."""
    gen = torch.Generator().manual_seed(seed)
    lo = torch.tensor([robot.limits[i]["lower"] for i in robot.controlled], dtype=torch.float64)
    hi = torch.tensor([robot.limits[i]["upper"] for i in robot.controlled], dtype=torch.float64)
    vel = torch.tensor([robot.limits[i]["velocity"] for i in robot.controlled], dtype=torch.float64)
    u = torch.rand(3, batch, robot.n_dofs, generator=gen, dtype=torch.float64)
    q = lo + (hi - lo) * u[0]
    qd = (2 * u[1] - 1) * vel_scale * vel
    qdd = (2 * u[2] - 1) * acc_scale * vel
    return q.to(dtype), qd.to(dtype), qdd.to(dtype)


# ------------------------------------------------------------------------------------------------
# flat-table view (layout of include/drm_b200.h) -- used to check the kernels' table gradients
# ------------------------------------------------------------------------------------------------
def axis_codes(robot):
    """0 fixed, +-1/+-2/+-3 = +-x/+-y/+-z per link."""
    codes = []
    for i in range(len(robot.names)):
        if robot.dof[i] < 0:
            codes.append(0)
            continue
        ax = robot.axis[i]
        k = int(torch.where(ax != 0)[0])
        codes.append((k + 1) if float(ax[k]) > 0 else -(k + 1))
    return codes


def link_table(robot):
    """Differentiable [N,28] table [F(9) r(3) Io(9) mc(3) m d 0 0] from the Robot parameters."""
    rows = []
    for i in range(len(robot.names)):
        roll, pitch, yaw = robot.rpy[i, 0:1], robot.rpy[i, 1:2], robot.rpy[i, 2:3]
        F = ((_elem_rot(2, yaw) @ _elem_rot(1, pitch)) @ _elem_rot(0, roll))[0]
        c = robot.com[i:i + 1]
        S = _skew(c)[0]
        Io = robot.inertia[i] + robot.mass[i] * (S @ S.T)
        rows.append(torch.cat([F.reshape(9), robot.trans[i], Io.reshape(9), robot.mass[i] * robot.com[i],
                               robot.mass[i].reshape(1), robot.damping[i].reshape(1),
                               torch.zeros(2, dtype=robot.trans.dtype)]))
    return torch.stack(rows)
