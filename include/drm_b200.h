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
 * (rigid_body_params.py:14-56).  Forward: one launch (raw rows are written to raw_out for the backward, then the table as
 * above).  Backward: table_grad -> flat_grad [n_flat] (two tiny launches; raw_grad_scratch [n_links, 20] is workspace).
 * All pointers are device pointers; src / kind / off have n_links * DRMB200_RAW_STRIDE entries.
 */
int drmb200_build_link_table_fused(const float* const_raw, const float* flat, const int32_t* src, const int32_t* kind,
                                   const float* off, int32_t n_links, float* raw_out, float* table, void* cuda_stream);
int drmb200_build_link_table_fused_backward(const float* raw, const float* table_grad, const float* flat,
                                            const int32_t* src, const int32_t* kind, int32_t n_links, int32_t n_flat,
                                            float* raw_grad_scratch, float* flat_grad, void* cuda_stream);

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
