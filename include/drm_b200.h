/*
 * drm_b200.h -- C ABI of the batched rigid-body kinematics/dynamics engine (CUDA, sm_90a).
 *
 * This is the drop-in boundary for the hot path of facebookresearch/differentiable-robot-model
 * (reference paths below are relative to /root/reference):
 *
 *   drmb200_fk_jacobian        replaces  DifferentiableRobotModel.compute_forward_kinematics
 *                                        (differentiable_robot_model/robot_model.py:224-248) and
 *                                        compute_endeffector_jacobian (robot_model.py:627-667),
 *                                        i.e. update_kinematic_state (robot_model.py:140-195) +
 *                                        CoordinateTransform.get_quaternion
 *                                        (spatial_vector_algebra.py:108-136) in one launch.
 *   drmb200_fk_jacobian_backward         the analytic adjoint of the above (the reference relies on
 *                                        autograd over its per-link op graph; no single line).
 *   drmb200_inverse_dynamics   replaces  compute_inverse_dynamics (robot_model.py:306-375) =
 *                                        update_kinematic_state + iterative_newton_euler
 *                                        (robot_model.py:251-303) + axis projection + damping.
 *   drmb200_inverse_dynamics_backward    analytic adjoint of RNEA (SURVEY.md Appendix B.2).
 *   drmb200_forward_dynamics   replaces  compute_forward_dynamics (robot_model.py:488-624), the articulated-body
 *                                        algorithm, in one launch.
 *   drmb200_forward_dynamics_rollout     many semi-implicit Euler steps of the above in one launch (the reference
 *                                        integrates with a Python loop around compute_forward_dynamics), and its adjoint.
 *   drmb200_pd_rollout                   the same rollout driven by a diagonal joint-space PD loop around reference
 *                                        trajectories, in one launch, and its adjoint (the reference: a Python loop).
 *   drmb200_inverse_dynamics_derivatives / drmb200_forward_dynamics_derivatives   the Jacobians of the two above w.r.t.
 *                                        q, qd (and f), [B, n, n] each, one launch (the reference: autograd, row by row).
 *   drmb200_inverse_kinematics           Levenberg-Marquardt inverse kinematics of one link for a batch of pose targets,
 *                                        all iterations in one launch (the reference has no IK).
 *   drmb200_inverse_kinematics_multi     the same for several links at once (one solve over their stacked errors).
 *   drmb200_operational_space_dynamics   inverse operational-space inertia J G J^T and the velocities, bias and true
 *                                        accelerations of several links, one launch (the reference has none of these).
 *   drmb200_contact_dynamics / drmb200_contact_impulse   joint accelerations and contact forces under rigid contacts at
 *                                        several links, and the joint velocities and impulses of an impact there, one launch
 *                                        each (the reference has none of these); drmb200_contact_dynamics_backward /
 *                                        drmb200_contact_impulse_backward are their analytic adjoints.
 *   drmb200_contact_rollout              T semi-implicit Euler steps of the contact dynamics with Baumgarte stabilisation
 *                                        towards fixed link targets, one launch (the reference has none of these).
 *   drmb200_dynamics_regressor           the joint-torque regressor Y, tau = Y . (I_o, mc, m, damping of every link), one
 *                                        launch (the reference: autograd of compute_inverse_dynamics, row by row).
 *   drmb200_energy_momentum              kinetic and potential energy, generalized momentum H(q) qd, centre of mass, its
 *                                        velocity and its Jacobian, one launch (the reference has none of these).
 *   drmb200_fk_jacobian_host   the same FK+Jacobian op on HOST buffers (pinned or pageable):
 *                              chunked H2D -> kernel -> D2H pipeline on internal streams.
 *
 * The reference has no FFI of its own (it is pure Python); the reference-side binding is the
 * ctypes stub shown in INTEGRATION.md.  All entry points are `extern "C"`, take plain pointers
 * and sizes, never throw, never synchronise the device (except the *_host variants, which return
 * after their last D2H copy completed) and return 0 on success or a negative DRMB200_E* code.
 *
 * Data layout (all fp32, contiguous, row-major; the reference is fp32-only):
 *   q, qd, qdd, tau      [B, n_dofs]
 *   pos                  [B, 3]
 *   quat                 [B, 4]    xyzw, branch structure of spatial_vector_algebra.py:116-135
 *   jac_lin, jac_ang     [B, 3, n_dofs]
 *   table                [n_links, DRMB200_TABLE_STRIDE]  the differentiable link table, device
 *                        memory, one row per link in URDF document order:
 *        [0:9)   F      fixed joint rotation Rz(yaw)Ry(pitch)Rx(roll), row-major (rigid_body.py:138-143)
 *        [9:12)  r      joint origin translation                       (rigid_body.py:146)
 *        [12:21) I_o    rotational inertia about the link origin, row-major, NOT symmetrised
 *                       I_c + m S(c)S(c)^T                             (spatial_vector_algebra.py:324-327)
 *        [21:24) mc     mass * centre of mass                          (spatial_vector_algebra.py:323)
 *        [24]    m      mass
 *        [25]    d      joint damping                                  (robot_model.py:368-373)
 *        [26:28) pad
 *   table_grad           same shape; batch-summed adjoint of every table entry.
 */
#ifndef DRM_B200_H
#define DRM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DRMB200_MAX_LINKS 64
#define DRMB200_TABLE_STRIDE 28

/* status codes */
#define DRMB200_OK 0
#define DRMB200_EINVAL (-1)   /* null pointer, negative batch, bad link index, bad topology */
#define DRMB200_ECUDA (-2)    /* CUDA runtime error; see drmb200_last_error() */
#define DRMB200_ELIMIT (-3)   /* model exceeds DRMB200_MAX_LINKS */

/* flags for the dynamics entry points (robot_model.py:311-312) */
#define DRMB200_GRAVITY 1u    /* include_gravity: base linear acceleration (0, 0, +9.81) */
#define DRMB200_DAMPING 2u    /* use_damping: tau += damping * qd */
/* drmb200_inverse_dynamics_backward only: the caller needs just the inertial columns of table_grad (I_o, mc, m)
 * and the damping column -- nothing kinematic (F, r) is learnable and q_grad / qd_grad / qdd_grad are NULL.
 * Selects a single-sweep kernel (~6x fewer instructions); the F / r columns of table_grad are left untouched. */
#define DRMB200_INERTIAL_GRADS_ONLY 4u
/* the rollouts (drmb200_forward_dynamics_rollout(_backward), drmb200_pd_rollout(_backward), drmb200_contact_rollout) only:
 * implicit joint damping with step h = dt, as defined at drmb200_forward_dynamics_implicit_damping.  Needs
 * DRMB200_DAMPING and a finite dt > 0, else DRMB200_EINVAL. */
#define DRMB200_IMPLICIT_DAMPING 8u
/* drmb200_pd_rollout(_backward) only: implicit PD gains (stable PD) with step h = dt, as defined at drmb200_pd_rollout.
 * Needs a finite dt > 0, else DRMB200_EINVAL; combines freely with DRMB200_IMPLICIT_DAMPING.  The other rollouts return
 * DRMB200_EINVAL for it. */
#define DRMB200_IMPLICIT_GAINS 16u

/*
 * Immutable kinematic-tree topology, host memory, links in URDF document order
 * (= reference body index order, robot_model.py:114).  parent[i] < i for every i > 0 is required
 * (all shipped URDFs satisfy it; the host loader checks).
 */
typedef struct drmb200_topology {
    int32_t n_links;
    int32_t n_dofs;
    int8_t parent[DRMB200_MAX_LINKS]; /* -1 for the root (link 0)                              */
    int8_t axis[DRMB200_MAX_LINKS];   /* 0 fixed; +-1 / +-2 / +-3 = revolute about +-x / +-y / +-z */
    int8_t dof[DRMB200_MAX_LINKS];    /* column in q / tau / Jacobian, -1 for fixed joints      */
} drmb200_topology_t;

/* Library / build introspection. */
int drmb200_version(void);                 /* 10000*major + 100*minor + patch */
const char* drmb200_last_error(void);      /* thread-local text of the last failure */
int64_t drmb200_launch_count(void);        /* kernels launched by this library since load */
/* Tuning knobs (not part of the reference-facing surface; environment DRMB200_<NAME> sets the initial value):
 *   "fk_variant": 1 = TMA bulk-copy staging (default), 0 = cooperative float4 staging;
 *   "fk_tile":    configurations per CTA of the FK kernel, 64 / 128 / 256, 0 = chosen from the batch size (default);
 *   "fk_unroll":  0 = rolled chain walk, 1 = unrolled register-Jacobian kernel (paths <= 8 links), 2 = auto (default);
 *   "fk_packed":  1 = f32x2 pair arithmetic in the rolled chain walk (default), 0 = scalar FMA,
 *                 2 = two configurations per thread in the two f32x2 lanes (kept for A/B);
 *   "rnea_packed": 1 = f32x2 pair arithmetic in the inverse-dynamics kernel (default), 0 = scalar FMA;
 *   "rnea_fold":  1 = the inverse-dynamics kernel walks only the movable links, links behind fixed joints are folded into
 *                 their nearest movable ancestor while the table is staged (default), 0 = one step per link like the reference;
 *   "rnea_bwd_chain": drmb200_inverse_dynamics_backward on robots whose links form one serial chain (every link's parent is
 *                 the link before it): 1 = the two-sweep adjoint kernel (default), 0 = the general tree kernel;
 *   "host_fused": drmb200_fk_jacobian_host on page-locked buffers: 1 = one launch whose TMA copies cross PCIe (default),
 *                 0 = staged H2D -> kernel -> D2H pipeline;
 *   "fk_pdl":     programmatic dependent launch of drmb200_fk_jacobian.  0 (default): ordinary stream-ordered launches.
 *                 2: for a stream of independent batches -- a launch may begin (load q, walk the chains) while the FK
 *                 launches before it on the same stream are still running, and waits for them before its first global
 *                 WRITE.  Results are identical to mode 0 for every legal call sequence: the library tracks the output
 *                 ranges of the FK launches that can still be in flight on the stream and issues an ordinary launch
 *                 whenever q or the table of the new launch overlaps one of them (and for batches too small to bound
 *                 how many launches can be in flight).  Measured on an H100 SXM (400 W power limit): 5.96 us instead of
 *                 9.11 us per stream-ordered launch of 65 536 Kuka configurations.  1: wait before the first global read (A/B only, slower than 0). */
int drmb200_set_option(const char* name, int value);
int drmb200_get_option(const char* name, int* value);   /* the value in effect (environment / default / last set) */

/*
 * FK (+ geometric Jacobian) of link `ee_link` for a batch of joint configurations.
 * Any of pos / quat / (jac_lin, jac_ang) may be NULL to skip that output (jac_lin and jac_ang
 * must be both NULL or both non-NULL).  Columns of joints that are not on the ee->root path are
 * written as zeros (robot_model.py:646-649).  Device pointers; asynchronous on `cuda_stream`.
 */
int drmb200_fk_jacobian(const drmb200_topology_t* topo, int32_t ee_link,
                        const float* table, const float* q, int64_t batch,
                        float* pos, float* quat, float* jac_lin, float* jac_ang,
                        void* cuda_stream);

/*
 * FK (+ geometric Jacobians) of SEVERAL links in one walk of the kinematic tree: the union of the root -> link paths is
 * walked once per configuration and every requested link emits its outputs as the walk passes it (hands and multi-limb
 * robots: BASELINE config 4 evaluates the four Allegro fingertips; the reference needs one compute_endeffector_jacobian
 * call -- and one full update_kinematic_state pass, robot_model.py:140-195 -- per fingertip).
 *   ee_links [n_ee]  host array of distinct link indices, 1 <= n_ee <= 8 (the root is allowed);
 *   outputs          pos [n_ee, B, 3], quat [n_ee, B, 4], jac_lin / jac_ang [n_ee, B, 3, n_dofs]; block e equals what
 *                    drmb200_fk_jacobian returns for ee_links[e] (bit for bit); NULL skips an output as above.
 */
int drmb200_fk_jacobian_multi(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links,
                              const float* table, const float* q, int64_t batch,
                              float* pos, float* quat, float* jac_lin, float* jac_ang, void* cuda_stream);

/*
 * Adjoint of drmb200_fk_jacobian.  g_* are the upstream gradients of the corresponding outputs
 * (NULL = zero).  Writes q_grad [B, n_dofs] (may be NULL) and accumulates the batch-summed
 * gradient of the table into table_grad [n_links, 28] (may be NULL; must be zero-initialised or
 * hold a running sum).  `workspace` must hold drmb200_table_grad_workspace_bytes(topo, batch) bytes.
 */
int64_t drmb200_table_grad_workspace_bytes(const drmb200_topology_t* topo, int64_t batch);
int drmb200_fk_jacobian_backward(const drmb200_topology_t* topo, int32_t ee_link,
                                 const float* table, const float* q, int64_t batch,
                                 const float* g_pos, const float* g_quat,
                                 const float* g_jac_lin, const float* g_jac_ang,
                                 float* q_grad, float* table_grad,
                                 void* workspace, void* cuda_stream);

/*
 * Recursive Newton-Euler inverse dynamics, tau [B, n_dofs].  flags = DRMB200_GRAVITY | DRMB200_DAMPING.
 */
int drmb200_inverse_dynamics(const drmb200_topology_t* topo,
                             const float* table, const float* q, const float* qd, const float* qdd,
                             int64_t batch, uint32_t flags, float* tau, void* cuda_stream);

/*
 * Folding once, for tables that do not change between launches (constant models).  drmb200_inverse_dynamics folds the links
 * behind fixed joints into their movable ancestors while it stages the table ("rnea_fold"), once per CTA: 13-15 % of the
 * kernel.  A caller whose table is constant can fold it ONCE:
 *   drmb200_folded_table_rows   rows of the folded table (root + movable links), 0 if the topology has nothing to fold
 *                               (or "rnea_fold" is off), < 0 on a bad topology;
 *   drmb200_fold_link_table     table [n_links, 28] -> folded [rows, 28] (canonical joint frames; one tiny launch);
 *   drmb200_inverse_dynamics_prefolded   the same kernel reading the folded rows with a plain copy; tau is bit-identical to
 *                               drmb200_inverse_dynamics on the table the rows were folded from.
 */
int64_t drmb200_folded_table_rows(const drmb200_topology_t* topo);
int drmb200_fold_link_table(const drmb200_topology_t* topo, const float* table, float* folded, void* cuda_stream);
int drmb200_inverse_dynamics_prefolded(const drmb200_topology_t* topo,
                                       const float* folded, const float* q, const float* qd, const float* qdd,
                                       int64_t batch, uint32_t flags, float* tau, void* cuda_stream);
/* the mass-matrix and articulated-body kernels fold the same way; the same rows serve them */
int drmb200_mass_matrix_prefolded(const drmb200_topology_t* topo, const float* folded, const float* q, int64_t batch,
                                  float* H, void* cuda_stream);
int drmb200_forward_dynamics_prefolded(const drmb200_topology_t* topo,
                                       const float* folded, const float* q, const float* qd, const float* f,
                                       int64_t batch, uint32_t flags, float* qdd, void* cuda_stream);

/*
 * Inverse dynamics PLUS the per-link state the reference leaves behind in its body objects after
 * compute_inverse_dynamics (robot_model.py:183-193 `vel`, :262-277 `acc`, :284-301 `force`), in one launch.  Link-major,
 * component-major blocks (coalesced stores), natural link frames, row order (angular 3, linear 3):
 *   vels   [n_links, 6, B]  body-frame spatial velocity            (SpatialMotionVec .ang, .lin)
 *   accs   [n_links, 6, B]  body-frame spatial acceleration, base acceleration (0, 0, 9.81) folded in when GRAVITY is set
 *   forces [n_links, 6, B]  wrench of the link plus everything it carries (SpatialForceVec .ang = torque, .lin = force);
 *                           row 0 is the wrench transmitted to the root
 * Any of tau / vels / accs / forces may be NULL.
 */
int drmb200_dynamic_state(const drmb200_topology_t* topo,
                          const float* table, const float* q, const float* qd, const float* qdd,
                          int64_t batch, uint32_t flags, float* tau, float* vels, float* accs, float* forces,
                          void* cuda_stream);

/*
 * Adjoint of drmb200_inverse_dynamics given g_tau [B, n_dofs].  Any of q_grad / qd_grad / qdd_grad
 * [B, n_dofs] and table_grad [n_links, 28] may be NULL.
 */
int drmb200_inverse_dynamics_backward(const drmb200_topology_t* topo,
                                      const float* table, const float* q, const float* qd,
                                      const float* qdd, int64_t batch, uint32_t flags,
                                      const float* g_tau,
                                      float* q_grad, float* qd_grad, float* qdd_grad,
                                      float* table_grad, void* workspace, void* cuda_stream);

/*
 * Joint-space inertia matrix H [B, n_dofs, n_dofs] (row-major per configuration): replaces
 * compute_lagrangian_inertia_matrix (robot_model.py:403-450; there n_dofs + 1 inverse-dynamics evaluations whose
 * difference cancels gravity and damping) with ONE launch that evaluates the n_dofs unit-acceleration columns
 * H[:, :, j] = ID(q, 0, e_j) - ID(q, 0, 0) for zero velocity and zero gravity.
 */
int drmb200_mass_matrix(const drmb200_topology_t* topo, const float* table, const float* q, int64_t batch,
                        float* H, void* cuda_stream);

/*
 * Articulated-body forward dynamics, qdd [B, n_dofs] from applied joint forces f [B, n_dofs]: replaces
 * compute_forward_dynamics (robot_model.py:488-624) in one launch, with the reference's arithmetic (general 6x6
 * articulated inertias, U = IA S used as a column, +1e-37 regularisers).  flags = DRMB200_GRAVITY | DRMB200_DAMPING
 * (damping: f - damping * qd is applied internally; the caller's f is NOT modified, unlike robot_model.py:521).
 */
int drmb200_forward_dynamics(const drmb200_topology_t* topo,
                             const float* table, const float* q, const float* qd, const float* f,
                             int64_t batch, uint32_t flags, float* qdd, void* cuda_stream);

/*
 * Adjoint of drmb200_forward_dynamics given g_qdd [B, n_dofs] (the reference differentiates its op graph with
 * autograd; this is the analytic reverse-mode recursion, exact also for non-symmetric inertia matrices).  Any of
 * q_grad / qd_grad / f_grad [B, n_dofs] and table_grad [n_links, 28] may be NULL; table_grad is accumulated into.
 * `workspace` (always required) must hold drmb200_forward_dynamics_backward_workspace_bytes() bytes: the per-CTA partial
 * tables plus an L2-resident scratch for the 6x6 articulated inertias of the persistent CTAs.
 */
int64_t drmb200_forward_dynamics_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch);
int drmb200_forward_dynamics_backward(const drmb200_topology_t* topo,
                                      const float* table, const float* q, const float* qd, const float* f,
                                      int64_t batch, uint32_t flags, const float* g_qdd,
                                      float* q_grad, float* qd_grad, float* f_grad,
                                      float* table_grad, void* workspace, void* cuda_stream);

/*
 * Forward dynamics with implicit joint damping of step h = dt > 0 (finite): the articulated-body arithmetic of
 * drmb200_forward_dynamics with one change -- every movable joint's pivot d_i = S^T IA_i S becomes d_i + h damping_i
 * wherever it is used (the 1/(d + 1e-37) of the articulated-inertia pass, the 1/d of the acceleration pass).  The damping
 * torque -damping * qd is still applied, so flags must hold DRMB200_DAMPING (DRMB200_GRAVITY as for
 * drmb200_forward_dynamics; DRMB200_IMPLICIT_DAMPING is implied).  For a symmetric inertia this is
 *     qdd = (H(q) + h diag(damping))^-1 (f - nle(q, qd)),   nle including the damping torque,
 * the acceleration of a semi-implicit Euler step of length h whose damping torque is taken at the end-of-step velocity
 * qd + h qdd: the step is unconditionally stable in the damping, where the explicit one needs h below about 2 I / d.  For a
 * non-symmetric inertia_mat the arithmetic is the definition, as for drmb200_forward_dynamics.  The rollouts take exactly
 * this qdd_t (h = dt) with DRMB200_IMPLICIT_DAMPING.  The backward is the analytic adjoint of that arithmetic: the pivot's
 * adjoint also reaches the damping column of table_grad; dt is not differentiated.  Its workspace is
 * drmb200_forward_dynamics_backward_workspace_bytes().  DRMB200_EINVAL without DRMB200_DAMPING or for a dt that is not
 * finite and > 0; otherwise the errors of drmb200_forward_dynamics / drmb200_forward_dynamics_backward.
 */
int drmb200_forward_dynamics_implicit_damping(const drmb200_topology_t* topo,
                                              const float* table, const float* q, const float* qd, const float* f,
                                              int64_t batch, uint32_t flags, float dt, float* qdd, void* cuda_stream);
int drmb200_forward_dynamics_implicit_damping_backward(const drmb200_topology_t* topo,
                                                       const float* table, const float* q, const float* qd, const float* f,
                                                       int64_t batch, uint32_t flags, float dt, const float* g_qdd,
                                                       float* q_grad, float* qd_grad, float* f_grad,
                                                       float* table_grad, void* workspace, void* cuda_stream);

/*
 * Forward-dynamics rollout: n_steps steps of semi-implicit (symplectic) Euler over drmb200_forward_dynamics in ONE launch.
 * Starting from (q_0, qd_0) = (q0, qd0), step t = 0 .. n_steps-1 computes, in fp32 and in exactly this order,
 *     qdd_t = FD(q_t, qd_t, f_t);   qd_{t+1} = qd_t + dt * qdd_t;   q_{t+1} = q_t + dt * qd_{t+1}
 * (each "+ dt *" a rounded multiply, then a rounded add -- no FMA), so the trajectory is bit-identical to a loop of
 * drmb200_forward_dynamics launches followed by those two updates.  flags mean what they mean for drmb200_forward_dynamics;
 * with DRMB200_IMPLICIT_DAMPING (and DRMB200_DAMPING) FD is drmb200_forward_dynamics_implicit_damping with h = dt, and the
 * trajectory is bit-identical to a loop of those launches.
 * Layout is time-major:
 *   q0, qd0              [B, n_dofs]
 *   f                    [n_steps, B, n_dofs]   applied joint forces of every step (never modified)
 *   q, qd                [n_steps, B, n_dofs]   q[t] = q_{t+1}, qd[t] = qd_{t+1}
 *   qdd                  [n_steps, B, n_dofs]   qdd[t] = qdd_t; may be NULL
 * The table is staged (and folded) once per CTA and the state stays in shared memory for all steps.  Outputs must not alias
 * inputs.  batch == 0 or n_steps == 0 is a no-op.
 */
int drmb200_forward_dynamics_rollout(const drmb200_topology_t* topo, const float* table,
                                     const float* q0, const float* qd0, const float* f, int64_t batch, int32_t n_steps,
                                     float dt, uint32_t flags, float* q, float* qd, float* qdd, void* cuda_stream);

/*
 * Adjoint of drmb200_forward_dynamics_rollout.  q / qd are the forward's outputs (the step inputs of steps 1 .. n_steps-1);
 * g_q / g_qd / g_qdd [n_steps, B, n_dofs] are the upstream gradients of q / qd / qdd (NULL = zero).  Writes q0_grad /
 * qd0_grad [B, n_dofs] and f_grad [n_steps, B, n_dofs] (each may be NULL) and accumulates the table gradient of all steps
 * into table_grad (may be NULL).  Runs the analytic adjoint of drmb200_forward_dynamics_backward once per step, t = n_steps-1
 * .. 0, with one element-wise launch per step between them (2 n_steps + 2 launches).  `workspace` must hold
 * drmb200_forward_dynamics_rollout_backward_workspace_bytes(topo, batch) bytes; it does not depend on n_steps.  Outputs
 * must not alias inputs.  With DRMB200_IMPLICIT_DAMPING each step runs the adjoint of
 * drmb200_forward_dynamics_implicit_damping_backward (h = dt).
 */
int64_t drmb200_forward_dynamics_rollout_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch);
int drmb200_forward_dynamics_rollout_backward(const drmb200_topology_t* topo, const float* table,
                                              const float* q0, const float* qd0, const float* f, int64_t batch,
                                              int32_t n_steps, float dt, uint32_t flags,
                                              const float* q, const float* qd,
                                              const float* g_q, const float* g_qd, const float* g_qdd,
                                              float* q0_grad, float* qd0_grad, float* f_grad,
                                              float* table_grad, void* workspace, void* cuda_stream);

/*
 * PD-controlled rollout: drmb200_forward_dynamics_rollout with a diagonal joint-space PD law closing the loop inside the
 * same launch.  Starting from (q_0, qd_0) = (q0, qd0), step t = 0 .. n_steps-1 computes, in fp32 and in exactly this
 * order, every operation rounded separately (no FMA):
 *     e_t   = q_ref[t] - q_t
 *     ed_t  = qd_ref[t] - qd_t                          qd_ref NULL: a zero tensor (0.f - qd_t)
 *     u_t   = (f[t] + kp * e_t) + kd * ed_t             f NULL: a zero tensor (0.f + kp * e_t); each "kp *" one rounded
 *                                                       multiply, then a rounded add
 *     tau_t = clamp(u_t, -effort_limit, effort_limit)   only when effort_limit is given; NaN propagates (torch.clamp)
 *     qdd_t = FD(q_t, qd_t, tau_t)                      exactly drmb200_forward_dynamics with the same flags
 *                                                       (drmb200_forward_dynamics_implicit_damping with h = dt under
 *                                                       DRMB200_IMPLICIT_DAMPING)
 *     qd_{t+1} = qd_t + dt * qdd_t;   q_{t+1} = q_t + dt * qd_{t+1}   as drmb200_forward_dynamics_rollout
 * so the trajectory is bit-identical to the torch loop
 *     u = f[t] + kp * (q_ref[t] - q) + kd * (qd_ref[t] - qd); u = clamp(u, -lim, lim);
 *     qdd = forward_dynamics(q, qd, u); qd = qd + dt * qdd; q = q + dt * qd
 * Layout is time-major:
 *   q0, qd0                        [B, n_dofs]
 *   q_ref, qd_ref, f               [n_steps, B, n_dofs]   qd_ref and f may be NULL (never modified)
 *   kp, kd                         both [n_dofs], shared by every row (gains_per_row = 0), or both [B, n_dofs]
 *                                  (gains_per_row = 1)
 *   effort_limit                   [n_dofs], every entry > 0 (inf allowed), or NULL for no limit
 *   q, qd, qdd, tau                [n_steps, B, n_dofs]   q[t] = q_{t+1}, qd[t] = qd_{t+1}, qdd[t] = qdd_t, tau[t] = tau_t;
 *                                  qdd may be NULL
 * No allocation, no synchronisation, graph-capturable.  Outputs must not alias inputs.  batch == 0 or n_steps == 0 is a
 * no-op.  DRMB200_EINVAL for a NULL required pointer or a negative size.  A CTA holds 64 or 32 configurations, or 16 when
 * 32 need more than 227 KB of shared memory (per-row gains and all three input streams take a 63-DoF chain there);
 * DRMB200_ELIMIT only when a 16-configuration CTA still needs more (the message names the bytes).
 *
 * DRMB200_IMPLICIT_GAINS (stable PD; needs a finite dt > 0, combines with DRMB200_IMPLICIT_DAMPING): the PD law is taken
 * at the end-of-step state.  With h = dt, step t computes, every operation rounded separately (no FMA but the pivot's):
 *     qp     = q_t + h * qd_t                            the position the step predicts at the current velocity
 *     e      = q_ref[t] - qp;   ed = qd_ref[t] - qd_t     (qd_ref NULL: 0.f - qd_t)
 *     u^     = (f[t] + kp * e) + kd * ed                 (f NULL: 0.f + kp * e)
 *     sat    = effort_limit given and !(-lim <= u^ <= lim)   torch.clamp's rule; NaN counts as saturated
 *     u      = sat ? clamp(u^, -lim, lim) : u^
 *     c      = sat ? 0 : h * (kd + h * kp)               per row and joint, per step
 *     qdd_t  = FD'(q_t, qd_t, u)    the ABA of drmb200_forward_dynamics (of drmb200_forward_dynamics_implicit_damping
 *                                   under DRMB200_IMPLICIT_DAMPING) with every movable joint k's pivot d_k (+ h damping_k)
 *                                   then + c_k, one rounded add
 *     tau_t  = sat ? u : u - c * qdd_t
 * and the integrate as above.  For a symmetric inertia (H + h D_impl + diag(h kd + h^2 kp)) qdd_t = u^ - nle, so on an
 * unsaturated joint tau_t = f + kp (q_ref - q_{t+1}) + kd (qd_ref - qd_{t+1}) up to rounding: the PD law at the
 * end-of-step state.  For one joint of inertia I with kp, kd >= 0 the step is stable at every h, where the explicit one
 * needs h kd / I < 2 and h^2 kp / I + 2 h kd / I < 4.  The gains' signs are not checked (that would need a host
 * synchronisation): negative gains may leave a pivot <= 0.  The effort limit is decided on the predicted command u^: a
 * saturated joint gets the clamped constant torque and no pivot term, and an unsaturated joint's applied tau_t may exceed
 * the limit by |c qdd_t| (an exact saturating solve would need an active-set iteration).  For a non-symmetric inertia_mat
 * the arithmetic above is the definition.
 */
int drmb200_pd_rollout(const drmb200_topology_t* topo, const float* table,
                       const float* q0, const float* qd0, const float* q_ref, const float* qd_ref, const float* f,
                       const float* kp, const float* kd, int32_t gains_per_row, const float* effort_limit,
                       int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                       float* q, float* qd, float* qdd, float* tau, void* cuda_stream);

/*
 * Adjoint of drmb200_pd_rollout.  The inputs are the forward's, plus its outputs q / qd (the step inputs of steps
 * 1 .. n_steps-1) and tau (every step's applied torque); g_q / g_qd / g_qdd / g_tau [n_steps, B, n_dofs] are the upstream
 * gradients of q / qd / qdd / tau (NULL = zero).  Writes q0_grad / qd0_grad [B, n_dofs], q_ref_grad / qd_ref_grad /
 * f_grad [n_steps, B, n_dofs] and kp_grad / kd_grad PER ROW, [B, n_dofs], whichever the gains' shape (a shared gain's
 * gradient is their sum over rows); each may be NULL.  Accumulates the table gradient of all steps into table_grad (may be
 * NULL).  The clamp passes the gradient where -effort_limit <= u_t <= effort_limit (torch.clamp's rule), u_t recomputed
 * bit-exactly.  Runs the analytic adjoint of drmb200_forward_dynamics_backward once per step, t = n_steps-1 .. 0, at
 * (q_t, qd_t, tau_t) (the implicit-damping adjoint under DRMB200_IMPLICIT_DAMPING), with one element-wise launch per
 * step between them (2 n_steps + 2 launches, no atomics: bitwise reproducible).  `workspace` must hold drmb200_pd_rollout_backward_workspace_bytes(topo, batch) bytes; it does not depend
 * on n_steps.  Outputs must not alias inputs.
 * DRMB200_IMPLICIT_GAINS: the adjoint of that step, still 2 n_steps + 2 launches without atomics.  Each element-wise
 * launch recomputes u^_t, sat_t, u_t and c_t bit-exactly from (q_t, qd_t) and the ABA adjoint runs at (q_t, qd_t, u_t)
 * with the pivot addends c_t, returning their adjoint c-bar and its recomputed qdd_t as well; with mask = !sat,
 * gu = mask (f-bar + g_tau) and gc = mask (c-bar - qdd_t g_tau), the feedback terms become a_q -= kp gu,
 * a_qd -= (kd + h kp) gu, kp_grad += gu e + h^2 gc, kd_grad += gu ed + h gc (q_ref_grad = kp gu, qd_ref_grad = kd gu,
 * f_grad = gu), and g_qdd_t gets -c_t g_tau[t].  The workspace bound covers this case too: it is larger than before the
 * flag existed, by four [B, n_dofs] fp32 slices.
 */
int64_t drmb200_pd_rollout_backward_workspace_bytes(const drmb200_topology_t* topo, int64_t batch);
int drmb200_pd_rollout_backward(const drmb200_topology_t* topo, const float* table,
                                const float* q0, const float* qd0, const float* q_ref, const float* qd_ref, const float* f,
                                const float* kp, const float* kd, int32_t gains_per_row, const float* effort_limit,
                                int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                                const float* q, const float* qd, const float* tau,
                                const float* g_q, const float* g_qd, const float* g_qdd, const float* g_tau,
                                float* q0_grad, float* qd0_grad, float* q_ref_grad, float* qd_ref_grad, float* f_grad,
                                float* kp_grad, float* kd_grad, float* table_grad, void* workspace, void* cuda_stream);

/*
 * Jacobians of the dynamics, one launch each (forward-mode recursions, csrc/dynamics_derivatives.cu).  Every matrix is
 * [B, n_dofs, n_dofs], row-major per configuration, out[b, i, j] = d y_i / d x_j of exactly what drmb200_inverse_dynamics /
 * drmb200_forward_dynamics compute with the same flags and table (any inertia matrix, non-symmetric ones included: the
 * forward-dynamics derivatives differentiate the articulated-body arithmetic itself, not -H^-1 dtau).
 *   drmb200_inverse_dynamics_derivatives   dtau_dq, dtau_dqd
 *   drmb200_forward_dynamics_derivatives   dqdd_dq, dqdd_dqd, dqdd_df   (dqdd_df[:, :, j] = forward dynamics at (q, 0, e_j)
 *                                          without gravity or damping: the articulated-body algorithm is affine in f)
 * Caller-allocated outputs; NULL skips a matrix (all NULL: nothing is launched).  No allocation, no synchronisation: a call
 * can be captured in a CUDA graph.  The *_prefolded variants read the rows of drmb200_fold_link_table.  A model whose
 * per-CTA footprint exceeds 227 KB of shared memory even at one configuration per CTA returns DRMB200_ELIMIT (about 50 DoF
 * for inverse dynamics and 38 for forward dynamics on a serial chain).
 */
int drmb200_inverse_dynamics_derivatives(const drmb200_topology_t* topo,
                                         const float* table, const float* q, const float* qd, const float* qdd,
                                         int64_t batch, uint32_t flags, float* dtau_dq, float* dtau_dqd, void* cuda_stream);
int drmb200_inverse_dynamics_derivatives_prefolded(const drmb200_topology_t* topo,
                                                   const float* folded, const float* q, const float* qd, const float* qdd,
                                                   int64_t batch, uint32_t flags, float* dtau_dq, float* dtau_dqd,
                                                   void* cuda_stream);
int drmb200_forward_dynamics_derivatives(const drmb200_topology_t* topo,
                                         const float* table, const float* q, const float* qd, const float* f,
                                         int64_t batch, uint32_t flags, float* dqdd_dq, float* dqdd_dqd, float* dqdd_df,
                                         void* cuda_stream);
int drmb200_forward_dynamics_derivatives_prefolded(const drmb200_topology_t* topo,
                                                   const float* folded, const float* q, const float* qd, const float* f,
                                                   int64_t batch, uint32_t flags, float* dqdd_dq, float* dqdd_dqd,
                                                   float* dqdd_df, void* cuda_stream);

/*
 * Inverse kinematics of link `ee_link`: damped least-squares (Levenberg-Marquardt) iterations for a batch of targets in ONE
 * launch, one thread per row, all iterations on chip (csrc/inverse_kinematics.cu).  Per row b, in fp32:
 *   q <- clamp(q0[b], lower, upper) (fminf(fmaxf(x, lower), upper) per joint; skipped when both are NULL),
 *   lambda <- damping_in[b] (damping_init when damping_in is NULL), then evaluate at q: the pose (p, R) and the geometric
 *   Jacobian J [6, n] (as drmb200_fk_jacobian, J_lin over J_ang) and the error
 *     e_pos = target_pos[b] - p;  q_err = quat* (x) conj(quat(R)) (quat* = target_quat[b] normalised, xyzw, quat(R) as
 *     drmb200_fk_jacobian returns it), negated if its w < 0;  e_rot = 2 atan2(s, w) / s q_err.xyz, s = |q_err.xyz| (0 if
 *     s == 0): the world-frame rotation vector of R* R^T.  target_quat == NULL: position only, e and J are the 3
 *     position rows.  E = |e|^2; done = |e_pos| <= pos_tol && |e_rot| <= rot_tol.
 *   max_iters times, skipping rows that are done: Cholesky of A = J J^T + lambda I (a pivot <= 0 or not finite rejects the
 *   step); q' = clamp(q + J^T A^-1 e), evaluated as above; accept iff E' < E (then q, J, e, E <- the trial's and
 *   lambda <- max(lambda / 2, 1e-5)), else lambda <- min(4 lambda, 1e5).
 * Outputs at the returned q: q [B, n_dofs], pos_err / rot_err [B] (|e_pos|, |e_rot|; rot_err = 0 for position only),
 * converged [B] (0 / 1: done) and damping_out [B] (the final lambda).  K iterations in one call are bit-identical to K
 * calls with max_iters = 1 that pass q and damping_out on.  Joints off the root -> ee path never move.  The suggested
 * damping_init is 1e-2.  Inputs: q0 [B, n_dofs], target_pos [B, 3], target_quat [B, 4] or NULL, lower / upper [n_dofs]
 * (both or neither), damping_in [B] or NULL.  Device pointers, caller-allocated outputs that must not alias inputs; no
 * allocation, no synchronisation (graph-capturable).  batch == 0 is a no-op.  DRMB200_EINVAL for a model without movable
 * joints, an ee path without movable joints, max_iters < 0, negative tolerances, one limit pointer without the other or
 * damping_init <= 0; DRMB200_ELIMIT when a 32-row CTA needs more than 227 KB of shared memory (14 n + 7 floats per row).
 */
int drmb200_inverse_kinematics(const drmb200_topology_t* topo, int32_t ee_link, const float* table,
                               const float* q0, const float* target_pos, const float* target_quat,
                               const float* lower, const float* upper, const float* damping_in,
                               int64_t batch, int32_t max_iters, float damping_init, float pos_tol, float rot_tol,
                               float* q, float* pos_err, float* rot_err, uint8_t* converged, float* damping_out,
                               void* cuda_stream);

/*
 * Inverse kinematics of SEVERAL links at once (fingertips of a hand, an arm and its hand): one Levenberg-Marquardt solve over
 * the stacked errors of every link per row, all iterations in ONE launch (csrc/inverse_kinematics_multi.cu).  The links share
 * the joints on the common part of their root paths, so they are moved together, which no set of single-link solves does.
 *   ee_links [n_ee]  host array of distinct link indices, 1 <= n_ee <= 8, each with a movable joint on its root path.
 *   U = the movable joints on the union of the root -> link paths, n_u = |U|; M = 3 n_ee (position) or 6 n_ee (pose).
 * Per row b, in fp32:
 *   q <- clamp(q0[b]) and lambda <- damping_in[b] (damping_init when NULL), as drmb200_inverse_kinematics; evaluate at q:
 *   for every link e its pose and Jacobian (as drmb200_fk_jacobian_multi returns them) and its errors e_pos,e and e_rot,e
 *   (as drmb200_inverse_kinematics computes them: normalised target, w < 0 flip, atan2 rotation vector).  e and J [M, n_u]
 *   are stacked link by link: rows [6e, 6e + 3) position, [6e + 3, 6e + 6) rotation (3 position rows per link for position
 *   only).  E = sum over e in link order of (|e_pos,e|^2 + |e_rot,e|^2); done = every link has |e_pos,e| <= pos_tol and
 *   |e_rot,e| <= rot_tol.
 *   max_iters times, skipping rows that are done, one damped least-squares step in the smaller space:
 *     M <= n_u (task space):  A = J J^T + lambda I_M,   dq = J^T A^-1 e;
 *     M >  n_u (joint space): A = J^T J + lambda I_nu,  dq = A^-1 J^T e   (equal to the above: push-through identity);
 *   Cholesky of A with the rejection rule of drmb200_inverse_kinematics; q' = clamp(q + dq) on U, evaluated as above; accept
 *   iff E' < E, with the same damping update (halve, floor 1e-5 / times 4, cap 1e5).
 * Outputs at the returned q: q [B, n_dofs], pos_err / rot_err [n_ee, B] (rot_err = 0 for position only), converged [B] and
 * damping_out [B].  K iterations in one call are bit-identical to K calls with max_iters = 1 that pass q and damping_out on;
 * with n_ee = 1 and M <= n_u the result is bit-identical to drmb200_inverse_kinematics of that link.  Joints outside U never
 * move.  Inputs: q0 [B, n_dofs], target_pos [n_ee, B, 3], target_quat [n_ee, B, 4] or NULL (the [n_ee, B, ...] blocks of
 * drmb200_fk_jacobian_multi, so its output at a goal configuration is a valid target), lower / upper [n_dofs] (both or
 * neither), damping_in [B] or NULL.  Device pointers, caller-allocated outputs that must not alias inputs; no allocation,
 * no synchronisation (graph-capturable).  batch == 0 is a no-op.  DRMB200_ELIMIT for n_ee outside [1, 8] or when a one-row
 * CTA needs more than 227 KB of shared memory; DRMB200_EINVAL for a link requested twice, a link without a movable joint on
 * its root path (the root included) and the argument errors of drmb200_inverse_kinematics.
 */
int drmb200_inverse_kinematics_multi(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links,
                                     const float* table, const float* q0, const float* target_pos,
                                     const float* target_quat, const float* lower, const float* upper,
                                     const float* damping_in, int64_t batch, int32_t max_iters, float damping_init,
                                     float pos_tol, float rot_tol, float* q, float* pos_err, float* rot_err,
                                     uint8_t* converged, float* damping_out, void* cuda_stream);

/*
 * Operational-space dynamics of SEVERAL links, one launch (csrc/operational_space.cu).  Per row b, for the model, the state
 * (q, qd), the applied joint forces f, flags (DRMB200_GRAVITY, DRMB200_DAMPING as for drmb200_forward_dynamics) and the
 * distinct links ee_links [n_ee] (host array, 1 <= n_ee <= 8):
 *   J [M, n_dofs]  every link's geometric Jacobian as drmb200_fk_jacobian returns it (link frame origin, world frame, the 3
 *                  linear rows over the 3 angular rows), stacked in list order: M = 6 n_ee; position_only != 0 keeps the
 *                  linear rows, M = 3 n_ee.  A link without a movable joint on its root path, the root included, has zero rows.
 *   qdd            what drmb200_forward_dynamics computes at (q, qd, f) with `flags`.
 *   G [n, n]       G[:, j] = forward dynamics at (q, 0, e_j) without gravity or damping (the dqdd_df of
 *                  drmb200_forward_dynamics_derivatives): H^-1 for symmetric inertias; for a non-symmetric inertia matrix the
 *                  result follows the articulated-body arithmetic, not H^-1.
 * Outputs, caller-allocated, fp32, row-major; NULL skips one (all NULL: nothing is launched):
 *   inv_inertia        [B, M, M]  J G J^T, off-diagonal blocks of links sharing joints included, not symmetrised
 *   velocity           [B, M]     J qd
 *   bias_acceleration  [B, M]     Jdot qd = sum_k d(J qd)/dq_k qd_k: the classical acceleration of each link origin (and the
 *                                 angular acceleration) at qdd = 0
 *   acceleration       [B, M]     J qdd + Jdot qd, the true world-frame acceleration; gravity enters only through qdd
 * The articulated-body algorithm is affine in f, so acceleration(f + J^T F) = acceleration(f) + inv_inertia F for any F in
 * R^M.  Inputs: q, qd, f [B, n_dofs], table; device pointers, outputs must not alias inputs.  No allocation, no
 * synchronisation (graph-capturable).  batch == 0 is a no-op.  DRMB200_EINVAL for n_ee outside [1, 8], a link index out of
 * range, a link requested twice, a negative batch or a null input; DRMB200_ELIMIT for more live branch points than the
 * forward-dynamics kernel handles or when a one-row CTA needs more than 227 KB of shared memory.
 */
int drmb200_operational_space_dynamics(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links,
                                       const float* table, const float* q, const float* qd, const float* f,
                                       int64_t batch, uint32_t flags, int32_t position_only, float* inv_inertia,
                                       float* acceleration, float* velocity, float* bias_acceleration,
                                       void* cuda_stream);

/*
 * Contact dynamics and contact impulses of bilateral rigid contacts at SEVERAL links, one launch each
 * (csrc/contact_dynamics.cu).  Per row b, for the model, the distinct links ee_links [n_ee] (host array, 1 <= n_ee <= 8),
 * position_only and a regularisation mu = `regularization` >= 0:
 *   J [M, n_dofs]  the stacked geometric Jacobians exactly as drmb200_operational_space_dynamics builds them (link frame
 *                  origin, world frame, 3 linear rows over 3 angular rows, M = 6 n_ee; only the linear rows, M = 3 n_ee, with
 *                  position_only != 0).
 *   G [n, n]       the same dqdd_df as there: the articulated-body algorithm at (q, 0, e_j) without gravity or damping; H^-1
 *                  for a symmetric inertia, the articulated-body arithmetic for a non-symmetric inertia_mat.
 *   A [M, M]       J G J^T + mu I_M: the operational-space inv_inertia plus mu on the diagonal.
 * Contact dynamics (drmb200_contact_dynamics), with the call's flags (DRMB200_GRAVITY, DRMB200_DAMPING):
 *   b        = J qdd_free + Jdot qd, qdd_free = forward dynamics at (q, qd, f): the operational-space `acceleration`;
 *   lambda   solves A lambda = a_ref - b, a_ref [B, M] the desired constraint-space acceleration (accel_ref; NULL: 0);
 *   qdd      [B, n]  qdd_free + G J^T lambda (= forward dynamics at (q, qd, f + J^T lambda): the ABA is affine in f);
 *   force    [B, M]  lambda: the stacked world-frame force applied at each link origin (and torque, in pose mode), the
 *                    convention of the operational-space acceleration(f + J^T F).
 *   Hence J qdd + Jdot qd = a_ref - mu lambda.
 * Contact impulse (drmb200_contact_impulse), no flags and no f: gravity, damping and applied forces do not act during an
 * instantaneous impulse:
 *   Lambda   solves A Lambda = v_ref - J qd, v_ref [B, M] the desired post-impact constraint velocity (velocity_ref; NULL:
 *            0, a perfectly inelastic impact; restitution e is v_ref = -e J qd);
 *   qd_plus  [B, n]  qd + G J^T Lambda;
 *   impulse  [B, M]  Lambda.
 *   Hence J qd_plus = v_ref - mu Lambda.
 * The solve: Jacobi equilibration s_k = |A_kk|^-1/2, then Gaussian elimination with partial pivoting on S A S (ties go to
 * the lower row index) and back substitution; the solution is S y.  A row is UNSOLVED when some A_kk is zero or not finite
 * or when a pivot of S A S is not finite or has magnitude <= 1e-5 (CONTACT_PIVOT_MIN, compiled in): it gets solved[b] = 0
 * and NaN in both outputs; a solved row gets solved[b] = 1.  The equilibration makes the threshold independent of units:
 * pose rows mix m/s^2 per N with rad/s^2 per N m.  Redundant constraint sets (more independent rows than the joints can
 * satisfy, e.g. 4 pose fingertips on iiwa7_allegro, M = 24 > 23 joints, or the planar 2-link arm in pose mode) are
 * unsolved at mu = 0 and need mu > 0.
 * Outputs, caller-allocated, fp32 / uint8, row-major, must not alias inputs; force / impulse may be NULL (skipped), qdd /
 * qd_plus and solved are required.  Inputs: q, qd, f [B, n_dofs], table; device pointers.  No allocation, no
 * synchronisation (graph-capturable).  batch == 0 is a no-op (no launch).  DRMB200_EINVAL for n_ee outside [1, 8], a link
 * index out of range, a link given twice, a link with no movable joint on its root path (the root included: its rows are
 * zero and never solvable), a negative or non-finite regularization, a null required pointer (batch > 0: empty tensors may
 * have null data) or a negative batch;
 * DRMB200_ELIMIT for more live branch points than the forward-dynamics kernel handles or, naming the bytes, when a one-row
 * CTA needs more than 227 KB of shared memory.
 */
int drmb200_contact_dynamics(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                             const float* q, const float* qd, const float* f, const float* accel_ref, int64_t batch,
                             uint32_t flags, int32_t position_only, float regularization,
                             float* qdd, float* force, uint8_t* solved, void* cuda_stream);
int drmb200_contact_impulse(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                            const float* q, const float* qd, const float* velocity_ref, int64_t batch,
                            int32_t position_only, float regularization,
                            float* qd_plus, float* impulse, uint8_t* solved, void* cuda_stream);

/*
 * Adjoints of drmb200_contact_dynamics and drmb200_contact_impulse (csrc/contact_backward.cu).  Given the forward's inputs, its
 * outputs qdd / qd_plus [B, n], force / impulse [B, M] and solved [B], and the upstream gradients g_qdd / g_qd_plus [B, n]
 * and g_force / g_impulse [B, M] (NULL: zero), per row, with J, G, A = J G J^T + mu I and qdd_free as stated above:
 *   lambda is defined implicitly by qdd = FD(q, qd, tau_c), tau_c = f + J^T lambda, and J qdd + Jdot qd = a_ref - mu lambda.
 *   Differentiating that equation:
 *     s      = g_force + J G^T g_qdd                  (G is not assumed symmetric)
 *     nu     solves A^T nu = s
 *     g^     = g_qdd - J^T nu;                        accel_ref_grad = nu
 *     (q1, qd1, theta1, tau^) = the adjoint of drmb200_forward_dynamics at (q, qd, tau_c) with upstream g^, the call's flags;
 *                                                      f_grad = tau^
 *     phi(q, qd; theta) = lambda^T J(q) tau^ - nu^T (J(q) qdd + Jdot(q, qd) qd)   with lambda, nu, tau^, qdd held constant
 *     q_grad = q1 + dphi/dq,  qd_grad = qd1 + dphi/dqd,  table_grad += theta1 + dphi/dtheta (the kinematic F, r columns)
 *   The impulse is the same with qdd -> qd_plus and lambda -> Lambda: the forward-dynamics adjoint runs at (q, 0, J^T Lambda)
 *   without flags, phi has no Jdot term (J qd_plus only), qd_grad = g^ and velocity_ref_grad = nu.
 * A^T nu = s is solved on the forward's factorisation: with S = diag(|A_kk|^-1/2), A~ = S A S and P A~ = L U by the forward's
 * elimination (the same float operations, so the same pivots and the same solved decision, bit for bit), A~^T y = S s and
 * nu = S y.  mu is not differentiated.  A row contributes only when the forward's solved[b] is set and the backward's own
 * factorisation (which repeats the forward's, so it decides the same) succeeds; every other row contributes exactly zero
 * to every gradient, whatever its upstream gradient and even when its inputs are not finite: its q_grad, qd_grad, f_grad,
 * accel_ref_grad / velocity_ref_grad rows are 0 and it adds nothing to table_grad.
 * Outputs, caller-allocated, fp32, must not alias inputs; each may be NULL: q_grad, qd_grad, f_grad [B, n],
 * accel_ref_grad / velocity_ref_grad [B, M], and table_grad [n_links, 28], which is ACCUMULATED into (a sum over the batch,
 * bitwise reproducible).  `workspace` must hold drmb200_contact_backward_workspace_bytes(topo, n_ee, ee_links,
 * position_only, batch) bytes.  Three stages in stream order: one launch of the contact adjoint kernel (nu, g^, tau_c); then,
 * when any of q_grad, qd_grad, f_grad, table_grad is wanted, the forward-dynamics adjoint (one launch, plus its reduction
 * with table_grad); then, when any of q_grad, qd_grad (dynamics only) or table_grad is wanted, one launch of the kinematic
 * adjoint kernel (plus its reduction with table_grad).  At most 5 launches; nothing is allocated or synchronised
 * (graph-capturable).  batch == 0 is a no-op.  Errors: those of the forward (checked before any launch), a null required
 * pointer (batch > 0) or workspace; DRMB200_ELIMIT, naming the bytes, when one row of either adjoint kernel needs more than
 * 227 KB of shared memory.
 */
int64_t drmb200_contact_backward_workspace_bytes(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links,
                                                 int32_t position_only, int64_t batch);
int drmb200_contact_dynamics_backward(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                      const float* q, const float* qd, const float* f, const float* accel_ref, const float* qdd,
                                      const float* force, const uint8_t* solved, int64_t batch, uint32_t flags,
                                      int32_t position_only, float regularization, const float* g_qdd, const float* g_force,
                                      float* q_grad, float* qd_grad, float* f_grad, float* accel_ref_grad, float* table_grad,
                                      void* workspace, void* cuda_stream);
int drmb200_contact_impulse_backward(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                                     const float* q, const float* qd, const float* velocity_ref, const float* qd_plus,
                                     const float* impulse, const uint8_t* solved, int64_t batch, int32_t position_only,
                                     float regularization, const float* g_qd_plus, const float* g_impulse, float* q_grad,
                                     float* qd_grad, float* velocity_ref_grad, float* table_grad, void* workspace,
                                     void* cuda_stream);

/*
 * Contact-constrained rollouts: T steps of semi-implicit Euler over drmb200_contact_dynamics with Baumgarte stabilisation,
 * ONE launch (csrc/contact_rollout.cu).  The links ee_links [n_ee] (host array, 1 <= n_ee <= 8), position_only, M = 3 n_ee or
 * 6 n_ee, mu = regularization >= 0 and the flags (DRMB200_GRAVITY, DRMB200_DAMPING) are those of drmb200_contact_dynamics;
 * dt is the step and omega = stabilization >= 0 (finite) the stabilisation rate.  Targets per link and row: a position p*
 * and, in pose mode, an orientation quat* (xyzw, normalised in the kernel as the IK kernels do); when none are given they
 * are the links' poses at q0, taken from the kernel's own walk at step 0.
 * From (q_0, qd_0) = (q0, qd0), step t = 0 ... T-1, in fp32:
 *   1. walk at (q_t, qd_t) as drmb200_operational_space_dynamics does: J, v = J qd, Jdot qd and every link's pose (p_l, R_l);
 *   2. e [M]: per link p_l - p*_l and, in pose mode, the world-frame rotation vector of R_l R*_l^T, the shorter way round
 *      (minus the rotation error of drmb200_inverse_kinematics, so that de/dt ~ omega_l, the angular rows of J qd);
 *   3. a_ref = -(2 omega) v - (omega^2) e, with 2 omega and omega^2 each rounded once, every product and the difference
 *      rounded once; omega == 0 forms no term: a_ref = 0 exactly and the step is drmb200_contact_dynamics(accel_ref = NULL);
 *   4. (qdd_t, lambda_t, ok_t) = drmb200_contact_dynamics(q_t, qd_t, f[t], a_ref), the same device code in the same order;
 *   5. qd_{t+1} = qd_t + dt * qdd_t;  q_{t+1} = q_t + dt * qd_{t+1}, every product and sum rounded separately.
 * With DRMB200_DAMPING the damping torque -d qd_t enters qdd_t explicitly, so the integrate is stable only for dt below
 * about 2 I / d (I a joint's effective inertia); light, strongly damped links need a far smaller step (the Allegro
 * fingers diverge within ten steps at dt = 1 ms and at 0.1 ms).  DRMB200_IMPLICIT_DAMPING (with DRMB200_DAMPING) takes
 * the damping implicitly: G and qdd_free become those of drmb200_forward_dynamics_implicit_damping with h = dt (pivots
 * d + dt damping in the ABA and in every unit-response sweep), so A = J G J^T + mu I follows; the step is stable in the
 * damping at any dt.
 * Outputs, time-major, caller-allocated, must not alias inputs: q [T, B, n] (q[t] = q_{t+1}), qd [T, B, n], qdd [T, B, n]
 * (qdd_t) or NULL, force [T, B, M] (lambda_t) or NULL, accel_ref [T, B, M] (the a_ref of step t) or NULL, solved [B] uint8
 * (the AND of ok_t over all steps).  An unsolved step gives NaN in qdd and lambda, so the row's state is NaN from then on;
 * other rows are unaffected.  Inputs: q0, qd0 [B, n], f [T, B, n] (required), target_pos [n_ee, B, 3] and, in pose mode,
 * target_quat [n_ee, B, 4] (both or neither; NULL in position mode), table; device pointers.  No allocation, no
 * synchronisation (graph-capturable).  batch == 0 or n_steps == 0 is a no-op (no launch).  DRMB200_EINVAL for the argument
 * errors of drmb200_contact_dynamics, n_steps < 0, a negative or non-finite stabilization, a target_quat in position mode
 * or only one of the two targets in pose mode; DRMB200_ELIMIT for more live branch points than the forward-dynamics kernel
 * handles or, naming the bytes, when a one-row CTA needs more than 227 KB of shared memory.
 */
int drmb200_contact_rollout(const drmb200_topology_t* topo, int32_t n_ee, const int32_t* ee_links, const float* table,
                            const float* q0, const float* qd0, const float* f, const float* target_pos,
                            const float* target_quat, int64_t batch, int32_t n_steps, float dt, uint32_t flags,
                            int32_t position_only, float regularization, float stabilization, float* q, float* qd, float* qdd,
                            float* force, float* accel_ref, uint8_t* solved, void* cuda_stream);

/*
 * The joint-torque regressor of the inertial parameters and dampings, one launch (csrc/dynamics_regressor.cu).  tau is
 * linear in every link's table entries 12:26 (I_o 9 row-major | mc 3 | m | damping), so for any table
 *   tau_i(q, qd, qdd) = sum_{l, k} Y[b, i, l, k] * table[l, 12 + k]         (Y . pi = tau)
 * where tau is exactly what drmb200_inverse_dynamics computes with the same table, flags and inputs.
 *   Y [B, n_dofs, n_links, 14], fp32, row-major:  Y[b, i, l, k] = d tau_i / d table[l, 12 + k], columns in the table's
 *     order; the entries of I_o are independent columns (non-symmetric I_o included: adding the I_o[a][b] and I_o[b][a]
 *     columns gives the usual symmetric 10-parameter form).  Every link has its own 14 columns: a fixed link's parameters
 *     reach tau through its movable ancestor, so its columns are not zero.  Exact zeros: the root's columns, the columns of
 *     links outside the subtree of dof i's link, the damping column of fixed links and, without DRMB200_DAMPING, every
 *     damping column.  With DRMB200_DAMPING, Y[b, dof(l), l, 13] = qd[b, dof(l)].  DRMB200_GRAVITY enters through the base
 *     acceleration, as in RNEA.
 * The regressor needs a column per table row, so it always walks the full (unfolded) tree: there is no _prefolded variant
 * and the "rnea_fold" option does not affect it.  Inputs: q, qd, qdd [B, n_dofs], table; device pointers, a
 * caller-allocated output that must not alias the inputs.  No allocation, no synchronisation (graph-capturable).
 * batch == 0 and models without movable joints are a no-op.  DRMB200_EINVAL for a null pointer or a negative batch;
 * DRMB200_ELIMIT for more live branch points than the tree program holds (as drmb200_inverse_dynamics) and, naming the
 * bytes needed, when one configuration per CTA needs more than 227 KB of shared memory (56 n_dofs n_links B of output each).
 */
int drmb200_dynamics_regressor(const drmb200_topology_t* topo, const float* table,
                               const float* q, const float* qd, const float* qdd,
                               int64_t batch, uint32_t flags, float* Y, void* cuda_stream);

/*
 * Whole-body quantities of a configuration, one launch (csrc/energy_momentum.cu).  They hold for any link table: learnable,
 * fused and non-symmetric I_o included.  For every link i, root included:
 *   (R_i, p_i) is its world pose and (w_i, v_i) its body-frame spatial velocity, exactly as drmb200_kinematic_state returns
 *   them; m_i = table[i, 24], mc_i = table[i, 21:24] and I_o,i = table[i, 12:21] (row-major, not symmetrised); M = sum_i m_i.
 *   For a movable link j, z_j is its world joint axis and p_j its origin, as in the Jacobian; sub(j) is link j and its
 *   descendants.  (f_lin, f_ang) = I_i V_i = (m v - mc x w, I_o w + mc x v), the reference's multiply_motion_vec.
 * Outputs, caller-allocated, fp32, row-major:
 *   kinetic       [B]        sum_i 1/2 m_i |v_i|^2 + 1/2 w_i^T I_o,i w_i + v_i . (w_i x mc_i)  (= 1/2 sum_i <V_i, I_i V_i>)
 *   potential     [B]        9.81 sum_i (m_i p_i,z + (R_i mc_i)_z): gravity is (0, 0, -9.81), the same as the DRMB200_GRAVITY
 *                            base acceleration; zero at z = 0
 *   momentum      [B, n]     momentum[dof(j)] = z_j . sum_{i in sub(j)} (R_i f_ang,i + (p_i - p_j) x R_i f_lin,i).  This equals
 *                            H(q) qd for the H of drmb200_mass_matrix, for any table
 *   com           [B, 3]     sum_i (m_i p_i + R_i mc_i) / M
 *   com_velocity  [B, 3]     sum_i R_i (m_i v_i + w_i x mc_i) / M, world frame
 *   com_jacobian  [B, 3, n]  column dof(j) = z_j x (sum_{i in sub(j)} (m_i p_i + R_i mc_i) - (sum_{i in sub(j)} m_i) p_j) / M,
 *                            so com_velocity = com_jacobian qd; a joint whose subtree is massless gets an exactly zero column
 * If M == 0 exactly, com, com_velocity and com_jacobian are written as zeros, not NaN.  kinetic = 1/2 qd . momentum holds
 * mathematically; only the symmetric part of I_o enters kinetic.
 * NULL skips an output (all NULL: nothing is launched).  qd [B, n_dofs] may be NULL only when kinetic, momentum and
 * com_velocity are all NULL; the other outputs do not depend on it and are bit-identical either way.  It always walks the
 * full (unfolded) tree: there is no _prefolded variant and "rnea_fold" does not affect it.  Inputs: q [B, n_dofs], table;
 * device pointers, outputs must not alias inputs.  No allocation, no synchronisation (graph-capturable).  batch == 0 is a
 * no-op.  DRMB200_EINVAL for a null table or q, a null qd that is needed, or a negative batch; DRMB200_ELIMIT for more
 * live branch points than the tree program holds and, naming the bytes, when a one-row CTA needs more than 227 KB of shared
 * memory (about 16 n_links + 4 n_dofs floats per row: no model within DRMB200_MAX_LINKS reaches it).
 */
int drmb200_energy_momentum(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                            int64_t batch, float* kinetic, float* potential, float* momentum, float* com,
                            float* com_velocity, float* com_jacobian, void* cuda_stream);

/*
 * World pose (and body-frame spatial velocity) of EVERY link in one launch: replaces update_kinematic_state
 * (robot_model.py:140-195) and, with `quats`, compute_forward_kinematics_all_links (robot_model.py:198-221).
 * Outputs are link-major / component-major so that stores coalesce:
 *   poses [n_links, 12, B]  rows 0..8 = R (row-major), 9..11 = p        (NULL to skip)
 *   quats [n_links,  4, B]  xyzw                                        (NULL to skip)
 *   vels  [n_links,  6, B]  ang(3), lin(3) in the link frame; needs qd  (NULL to skip)
 */
int drmb200_kinematic_state(const drmb200_topology_t* topo, const float* table, const float* q, const float* qd,
                            int64_t batch, float* poses, float* quats, float* vels, void* cuda_stream);

/*
 * Link-parameter rows -> link table, and its adjoint (device pointers, asynchronous).
 *   raw       [n_links, DRMB200_RAW_STRIDE]: rpy(3) | trans(3) | mass | com(3) | inertia_mat(9, at the COM) | damping
 *             -- the values the reference keeps in per-link modules (rigid_body.py:47-49,
 *             spatial_vector_algebra.py:312-314); for fixed joints pass the construction-time origin.
 *   table     [n_links, 28] as documented above (F = Rz Ry Rx, Io = I_c + m S(c)S(c)^T, mc = m c).
 * The backward maps table_grad [n_links, 28] to raw_grad [n_links, 20].  These replace ~60 small torch ops
 * (and ~100 autograd nodes) per call when link parameters are being learned.
 */
#define DRMB200_RAW_STRIDE 20
int drmb200_build_link_table(const float* raw, int32_t n_links, float* table, void* cuda_stream);
int drmb200_build_link_table_backward(const float* raw, const float* table_grad, int32_t n_links,
                                      float* raw_grad, void* cuda_stream);

/*
 * Fused parametrisation (BASELINE config 5): every learnable entry of the raw block is a function of ONE flat device vector,
 *   raw[k] = const_raw[k] (src[k] < 0) | flat[src[k]] (kind[k] == 0) | flat[src[k]]^2 + off[k] (kind[k] == 1),
 * which covers the reference's UnconstrainedScalar / UnconstrainedTensor / PositiveScalar modules
 * (rigid_body_params.py:14-56).  Several raw entries may read one flat entry (a parameter tied across links).
 * Forward: one launch (raw rows are written to raw_out for the backward, then the table as above).
 * Backward: table_grad -> flat_grad [n_flat] (two tiny launches; raw_grad_scratch [n_links, 20] is workspace).  The
 * inverse of src is passed as linked lists: first_reader[s] (n_flat entries) is the lowest raw index k with src[k] == s and
 * next_reader[k] (n_links * DRMB200_RAW_STRIDE entries) the next higher one, -1 for none; flat_grad[s] is the sum over that
 * list in that order, so it is bitwise repeatable, and zero for an entry nothing reads.
 * All pointers are device pointers; src / kind / off have n_links * DRMB200_RAW_STRIDE entries.
 */
int drmb200_build_link_table_fused(const float* const_raw, const float* flat, const int32_t* src, const int32_t* kind,
                                   const float* off, int32_t n_links, float* raw_out, float* table, void* cuda_stream);
int drmb200_build_link_table_fused_backward(const float* raw, const float* table_grad, const float* flat,
                                            const int32_t* first_reader, const int32_t* next_reader, const int32_t* kind,
                                            int32_t n_links, int32_t n_flat, float* raw_grad_scratch, float* flat_grad,
                                            void* cuda_stream);

/*
 * Host-buffer variant of drmb200_fk_jacobian: q and the outputs are HOST pointers (pinned memory
 * gives full PCIe bandwidth; pageable memory works).  `table` is still a device pointer (it is
 * < 8 KB and lives with the model).  With page-locked buffers (cudaHostAlloc / cudaHostRegister / torch pin_memory)
 * the kernel is launched ONCE on their device aliases and its TMA copies read / write host memory directly over PCIe
 * (transfer fused into the compute kernel); with pageable buffers the call splits the batch into chunks and overlaps
 * H2D / kernel / D2H on internal streams of `device`.  Either way it returns once all outputs are on the host.
 */
int drmb200_fk_jacobian_host(const drmb200_topology_t* topo, int32_t ee_link, int32_t device,
                             const float* table, const float* q_host, int64_t batch,
                             float* pos_host, float* quat_host,
                             float* jac_lin_host, float* jac_ang_host);

/*
 * The one exchange step of the data path (parameter learning on a sharded batch, BASELINE config 5): SUM all-reduce of the
 * flat link-parameter gradient over NVLink peer memory FUSED with the Adam update -- one kernel, no NCCL call, graph
 * capturable.  One process per GPU; the reference has no distributed code, this is new surface (csrc/comm.cu).
 *   drmb200_comm_create   allocates this rank's inbox on the current device and returns its 64-byte CUDA IPC handle;
 *   drmb200_comm_connect  takes the handles of ALL ranks (world * 64 bytes, in rank order; exchanged by the host, e.g.
 *                         with one torch.distributed all_gather) and maps the peers' inboxes;
 *   drmb200_allreduce_adam  param [n] (in place), grad [n] (this rank's shard gradient), exp_avg / exp_avg_sq [n] Adam state;
 *                         every rank must launch it once per step; all ranks end up with bit-identical parameters
 *                         (rank-ordered sum).  torch.optim.Adam arithmetic (no weight decay / amsgrad).
 *   drmb200_comm_error    1 if a peer failed to arrive within ~2 s (the kernel never spins forever), -1 on a CUDA error.
 */
typedef struct drmb200_comm drmb200_comm_t;
int drmb200_comm_create(int32_t rank, int32_t world, int32_t max_floats, drmb200_comm_t** comm, void* ipc_handle_out);
int drmb200_comm_connect(drmb200_comm_t* comm, const void* all_ipc_handles);
int drmb200_comm_destroy(drmb200_comm_t* comm);
int drmb200_comm_error(drmb200_comm_t* comm);
int drmb200_allreduce_adam(drmb200_comm_t* comm, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                           int32_t n, float lr, float beta1, float beta2, float eps, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* DRM_B200_H */
