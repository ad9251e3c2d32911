"""
ctypes binding of the C-ABI library + torch.autograd plumbing
================================================================
``libdrm_b200.so`` (``csrc/``, declared in ``include/drm_b200.h``) is the product: hand-written
sm_90a kernels behind an ``extern "C"`` interface with plain pointers.  This module loads it with
ctypes (no torch types cross the boundary -- only ``tensor.data_ptr()`` and the raw handle of the
current CUDA stream) and wraps the forward / backward entry points in ``torch.autograd.Function``s so
that the reference's parameter-learning examples keep training.

There is NO fallback: if the library is missing, or tensors are not on a CUDA device, every
compute entry raises ``RuntimeError``.
"""
import ctypes
import os

import torch

from .link_table import Topology

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libdrm_b200.so")
_lib = None

GRAVITY = 1
DAMPING = 2
INERTIAL_GRADS_ONLY = 4      # backward hint: no kinematic link parameter is learnable (see include/drm_b200.h)

_c_float_p = ctypes.c_void_p      # raw device / host addresses
_SIGNATURES = {
    "drmb200_version": (ctypes.c_int, []),
    "drmb200_last_error": (ctypes.c_char_p, []),
    "drmb200_launch_count": (ctypes.c_int64, []),
    "drmb200_set_option": (ctypes.c_int, [ctypes.c_char_p, ctypes.c_int]),
    "drmb200_get_option": (ctypes.c_int, [ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]),
    "drmb200_fk_jacobian": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, _c_float_p, _c_float_p,
                                           ctypes.c_int64, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                           ctypes.c_void_p]),
    "drmb200_fk_jacobian_multi": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32),
                                                 _c_float_p, _c_float_p, ctypes.c_int64, _c_float_p, _c_float_p, _c_float_p,
                                                 _c_float_p, ctypes.c_void_p]),
    "drmb200_table_grad_workspace_bytes": (ctypes.c_int64, [ctypes.POINTER(Topology), ctypes.c_int64]),
    "drmb200_fk_jacobian_backward": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, _c_float_p, _c_float_p,
                                                    ctypes.c_int64, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                    _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_inverse_dynamics": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p,
                                                ctypes.c_void_p]),
    "drmb200_folded_table_rows": (ctypes.c_int64, [ctypes.POINTER(Topology)]),
    "drmb200_fold_link_table": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_inverse_dynamics_prefolded": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                          ctypes.c_int64, ctypes.c_uint32, _c_float_p, ctypes.c_void_p]),
    "drmb200_mass_matrix_prefolded": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, ctypes.c_int64, _c_float_p,
                                                     ctypes.c_void_p]),
    "drmb200_forward_dynamics_prefolded": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                          ctypes.c_int64, ctypes.c_uint32, _c_float_p, ctypes.c_void_p]),
    "drmb200_dynamic_state": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                             ctypes.c_int64, ctypes.c_uint32, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                             ctypes.c_void_p]),
    "drmb200_inverse_dynamics_backward": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                         _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p,
                                                         _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                         ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_forward_dynamics": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p,
                                                ctypes.c_void_p]),
    "drmb200_mass_matrix": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, ctypes.c_int64, _c_float_p,
                                           ctypes.c_void_p]),
    "drmb200_forward_dynamics_backward_workspace_bytes": (ctypes.c_int64, [ctypes.POINTER(Topology), ctypes.c_int64]),
    "drmb200_forward_dynamics_backward": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                         _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p,
                                                         _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                         ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_kinematic_state": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64,
                                               _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_build_link_table": (ctypes.c_int, [_c_float_p, ctypes.c_int32, _c_float_p, ctypes.c_void_p]),
    "drmb200_build_link_table_backward": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int32, _c_float_p,
                                                         ctypes.c_void_p]),
    "drmb200_build_link_table_fused": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_void_p, _c_float_p,
                                                      ctypes.c_int32, _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_build_link_table_fused_backward": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                                               ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, _c_float_p,
                                                               _c_float_p, ctypes.c_void_p]),
    "drmb200_comm_create": (ctypes.c_int, [ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.POINTER(ctypes.c_void_p),
                                           ctypes.c_void_p]),
    "drmb200_comm_connect": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_comm_destroy": (ctypes.c_int, [ctypes.c_void_p]),
    "drmb200_comm_error": (ctypes.c_int, [ctypes.c_void_p]),
    "drmb200_allreduce_adam": (ctypes.c_int, [ctypes.c_void_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int32,
                                              ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "drmb200_fk_jacobian_host": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.c_int32, _c_float_p,
                                                _c_float_p, ctypes.c_int64, _c_float_p, _c_float_p, _c_float_p,
                                                _c_float_p]),
}


def library_path():
    return _LIB_PATH


def declared_symbols():
    return sorted(_SIGNATURES)


def lib():
    """Load (once) and return the C-ABI library; raise if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise RuntimeError(
                f"{_LIB_PATH} not found: the CUDA engine has not been built "
                "(run `python -c 'import __graft_entry__ as g; g.build()'` or `make -C "
                "differentiable_robot_model_b200/csrc`). There is no CPU fallback."
            )
        handle = ctypes.CDLL(_LIB_PATH)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(handle, name)      # AttributeError if the library lacks a declared symbol
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = handle
    return _lib


def _check(rc, what):
    if rc != 0:
        msg = lib().drmb200_last_error()
        raise RuntimeError(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _NoGuard:
    def __enter__(self):
        return None

    def __exit__(self, *exc):
        return False


_NO_GUARD = _NoGuard()


def _on(device):
    """Context that makes `device` current for a launch.  A no-op object when it already is (the usual case): entering
    torch.cuda.device() costs microseconds of host time per call, a large share of a batch-1 call."""
    if device.index is None or device.index == torch.cuda.current_device():
        return _NO_GUARD
    return torch.cuda.device(device)


def _require_cuda(*tensors):
    first = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(
                "the engine computes on CUDA tensors only (got a tensor on "
                f"{t.device}); there is no CPU fallback"
            )
        if t.dtype != torch.float32:
            raise RuntimeError(f"the engine is fp32-only like the reference (got {t.dtype})")
        if first is None:
            first = t.device
        elif t.device != first:
            raise RuntimeError(f"all tensors of one call must live on the same GPU (got {first} and {t.device})")


def launch_count():
    return int(lib().drmb200_launch_count())


def set_option(name, value):
    _check(lib().drmb200_set_option(name.encode(), int(value)), "drmb200_set_option")


def get_option(name):
    value = ctypes.c_int(0)
    _check(lib().drmb200_get_option(name.encode(), ctypes.byref(value)), "drmb200_get_option")
    return int(value.value)


# ------------------------------------------------------------------------------------------------
# raw (non-differentiable) launches
# ------------------------------------------------------------------------------------------------
def fk_jacobian_raw(topo, ee_link, table, q, want_pos=True, want_quat=True, want_jac=True, out=None):
    _require_cuda(table, q)
    q = q.contiguous()
    B, n = q.shape
    dev = q.device
    if out is not None:
        pos, quat, jlin, jang = out
    else:
        pos = torch.empty((B, 3), device=dev, dtype=torch.float32) if want_pos else None
        quat = torch.empty((B, 4), device=dev, dtype=torch.float32) if want_quat else None
        jlin = torch.empty((B, 3, n), device=dev, dtype=torch.float32) if want_jac else None
        jang = torch.empty((B, 3, n), device=dev, dtype=torch.float32) if want_jac else None
    with _on(dev):
        rc = lib().drmb200_fk_jacobian(ctypes.byref(topo), ee_link, _ptr(table), _ptr(q), B, _ptr(pos), _ptr(quat),
                                       _ptr(jlin), _ptr(jang), _stream())
    _check(rc, "drmb200_fk_jacobian")
    return pos, quat, jlin, jang


def fk_jacobian_multi_raw(topo, ee_links, table, q, want_pos=True, want_quat=True, want_jac=True, out=None):
    """FK (+ Jacobians) of several links in ONE tree walk (drmb200_fk_jacobian_multi): stacked [n_ee, B, ...] outputs."""
    _require_cuda(table, q)
    q = q.contiguous()
    B, n = q.shape
    dev, E = q.device, len(ee_links)
    if out is not None:
        pos, quat, jlin, jang = out
    else:
        pos = torch.empty((E, B, 3), device=dev, dtype=torch.float32) if want_pos else None
        quat = torch.empty((E, B, 4), device=dev, dtype=torch.float32) if want_quat else None
        jlin = torch.empty((E, B, 3, n), device=dev, dtype=torch.float32) if want_jac else None
        jang = torch.empty((E, B, 3, n), device=dev, dtype=torch.float32) if want_jac else None
    links = (ctypes.c_int32 * E)(*[int(l) for l in ee_links])
    with _on(dev):
        rc = lib().drmb200_fk_jacobian_multi(ctypes.byref(topo), E, links, _ptr(table), _ptr(q), B, _ptr(pos), _ptr(quat),
                                             _ptr(jlin), _ptr(jang), _stream())
    _check(rc, "drmb200_fk_jacobian_multi")
    return pos, quat, jlin, jang


def fold_link_table(topo, table):
    """Folded canonical rows [n_red, 28] of a link table (drmb200_fold_link_table), or None if there is nothing to fold.
    For tables that do not change between launches: drmb200_inverse_dynamics_prefolded reads them with a plain copy instead
    of folding the fixed links once per CTA."""
    _require_cuda(table)
    rows = int(lib().drmb200_folded_table_rows(ctypes.byref(topo)))
    if rows <= 0:
        return None
    folded = torch.empty((rows, 28), device=table.device, dtype=torch.float32)
    with _on(table.device):
        rc = lib().drmb200_fold_link_table(ctypes.byref(topo), _ptr(table.contiguous()), _ptr(folded), _stream())
    _check(rc, "drmb200_fold_link_table")
    return folded


def inverse_dynamics_raw(topo, table, q, qd, qdd, flags, out=None, folded=None):
    """tau [B, n].  `folded`: rows from fold_link_table(topo, table) for a table that has not changed since."""
    _require_cuda(table, q, qd, qdd, folded)
    q, qd, qdd = q.contiguous(), qd.contiguous(), qdd.contiguous()
    B, n = q.shape
    tau = out if out is not None else torch.empty((B, n), device=q.device, dtype=torch.float32)
    with _on(q.device):
        if folded is not None:
            rc = lib().drmb200_inverse_dynamics_prefolded(ctypes.byref(topo), _ptr(folded), _ptr(q), _ptr(qd), _ptr(qdd), B,
                                                          flags & 3, _ptr(tau), _stream())
        else:
            rc = lib().drmb200_inverse_dynamics(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(qdd), B,
                                                flags, _ptr(tau), _stream())
    _check(rc, "drmb200_inverse_dynamics")
    return tau


def forward_dynamics_raw(topo, table, q, qd, f, flags, out=None, folded=None):
    """Articulated-body algorithm, one launch (drmb200_forward_dynamics; `folded`: rows of fold_link_table for an unchanged table)."""
    _require_cuda(table, q, qd, f, folded)
    q, qd, f = q.contiguous(), qd.contiguous(), f.contiguous()
    B, n = q.shape
    qdd = out if out is not None else torch.empty((B, n), device=q.device, dtype=torch.float32)
    with _on(q.device):
        if folded is not None:
            rc = lib().drmb200_forward_dynamics_prefolded(ctypes.byref(topo), _ptr(folded), _ptr(q), _ptr(qd), _ptr(f), B,
                                                          flags, _ptr(qdd), _stream())
        else:
            rc = lib().drmb200_forward_dynamics(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B,
                                                flags, _ptr(qdd), _stream())
    _check(rc, "drmb200_forward_dynamics")
    return qdd


def kinematic_state_raw(topo, table, q, qd=None, want_poses=True, want_quats=False):
    """Poses [N,12,B] (+ quaternions [N,4,B], + velocities [N,6,B] when qd is given) of every link, one launch."""
    _require_cuda(table, q, qd)
    q = q.contiguous()
    qd = None if qd is None else qd.contiguous()
    B, N, dev = q.shape[0], topo.n_links, q.device
    poses = torch.empty((N, 12, B), device=dev, dtype=torch.float32) if want_poses else None
    quats = torch.empty((N, 4, B), device=dev, dtype=torch.float32) if want_quats else None
    vels = torch.empty((N, 6, B), device=dev, dtype=torch.float32) if qd is not None else None
    with _on(dev):
        rc = lib().drmb200_kinematic_state(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), B, _ptr(poses), _ptr(quats),
                                           _ptr(vels), _stream())
    _check(rc, "drmb200_kinematic_state")
    return poses, quats, vels


def dynamic_state_raw(topo, table, q, qd, qdd, flags, want_tau=True):
    """Inverse dynamics + per-link (vel, acc, force) blocks [N, 6, B] in one launch (drmb200_dynamic_state)."""
    _require_cuda(table, q, qd, qdd)
    q, qd, qdd = q.contiguous(), qd.contiguous(), qdd.contiguous()
    B, n = q.shape
    N, dev = topo.n_links, q.device
    tau = torch.empty((B, n), device=dev, dtype=torch.float32) if want_tau else None
    vels, accs, forces = (torch.empty((N, 6, B), device=dev, dtype=torch.float32) for _ in range(3))
    with _on(dev):
        rc = lib().drmb200_dynamic_state(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(qdd), B, flags, _ptr(tau),
                                         _ptr(vels), _ptr(accs), _ptr(forces), _stream())
    _check(rc, "drmb200_dynamic_state")
    return tau, vels, accs, forces


def fk_jacobian_host(topo, ee_link, device_index, table, q_host, pos, quat, jlin, jang):
    """Host-buffer FK+Jacobian (H2D / kernel / D2H pipelined inside the library)."""
    _require_cuda(table)
    B = q_host.shape[0]
    n = topo.n_dofs
    for name, t, shape in (("q", q_host, (B, n)), ("pos", pos, (B, 3)), ("quat", quat, (B, 4)),
                           ("jac_lin", jlin, (B, 3, n)), ("jac_ang", jang, (B, 3, n))):
        if t is None:
            if name == "q":
                raise RuntimeError("q_host is required")
            continue
        if t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != shape:
            raise RuntimeError(f"{name}: expected a contiguous fp32 CPU tensor of shape {shape}, got "
                               f"{t.dtype} {tuple(t.shape)} on {t.device} (contiguous={t.is_contiguous()})")
    if table.device.index != device_index:
        raise RuntimeError(f"table lives on {table.device}, the call targets cuda:{device_index}")
    # the library launches on its own non-blocking stream: everything queued on torch's current stream of that device
    # (e.g. the kernel that built `table`) must have completed first
    torch.cuda.current_stream(table.device).synchronize()
    rc = lib().drmb200_fk_jacobian_host(ctypes.byref(topo), ee_link, device_index, _ptr(table), _ptr(q_host), B,
                                        _ptr(pos), _ptr(quat), _ptr(jlin), _ptr(jang))
    _check(rc, "drmb200_fk_jacobian_host")


def _workspace(topo, batch, device):
    nbytes = int(lib().drmb200_table_grad_workspace_bytes(ctypes.byref(topo), batch))
    return torch.empty((max(nbytes, 4) + 3) // 4, device=device, dtype=torch.float32)


# ------------------------------------------------------------------------------------------------
# autograd
# ------------------------------------------------------------------------------------------------
class BuildLinkTableFunction(torch.autograd.Function):
    """raw link parameters [n_links, 20] -> link table [n_links, 28] (csrc/table.cu), one launch each way."""

    @staticmethod
    def forward(ctx, raw):
        _require_cuda(raw)
        raw = raw.contiguous()
        n_links = raw.shape[0]
        table = torch.empty((n_links, 28), device=raw.device, dtype=torch.float32)
        with _on(raw.device):
            rc = lib().drmb200_build_link_table(_ptr(raw), n_links, _ptr(table), _stream())
        _check(rc, "drmb200_build_link_table")
        ctx.save_for_backward(raw)
        return table

    @staticmethod
    def backward(ctx, g_table):
        (raw,) = ctx.saved_tensors
        g_table = g_table.contiguous()
        _require_cuda(g_table)
        g_raw = torch.empty_like(raw)
        with _on(raw.device):
            rc = lib().drmb200_build_link_table_backward(_ptr(raw), _ptr(g_table), raw.shape[0], _ptr(g_raw), _stream())
        _check(rc, "drmb200_build_link_table_backward")
        return g_raw



class FusedTableFunction(torch.autograd.Function):
    """flat link-parameter vector [P] -> link table [n_links, 28] in ONE launch (drmb200_build_link_table_fused): the
    per-(link, parameter) parametrisation modules are applied inside the kernel through an index / kind / offset map.
    Backward: table_grad -> flat_grad, two tiny launches.  One leaf, one AccumulateGrad node, one optimiser tensor."""

    @staticmethod
    def forward(ctx, flat, const_raw, src, kind, off):
        _require_cuda(flat, const_raw, off)
        flat = flat.contiguous()
        n_links = const_raw.shape[0]
        raw = torch.empty_like(const_raw)
        table = torch.empty((n_links, 28), device=flat.device, dtype=torch.float32)
        with _on(flat.device):
            rc = lib().drmb200_build_link_table_fused(_ptr(const_raw), _ptr(flat), _ptr(src), _ptr(kind), _ptr(off), n_links,
                                                      _ptr(raw), _ptr(table), _stream())
        _check(rc, "drmb200_build_link_table_fused")
        ctx.save_for_backward(flat, raw, src, kind)
        return table

    @staticmethod
    def backward(ctx, g_table):
        flat, raw, src, kind = ctx.saved_tensors
        g_table = g_table.contiguous()
        _require_cuda(g_table)
        g_flat = torch.empty_like(flat)
        scratch = torch.empty_like(raw)
        with _on(flat.device):
            rc = lib().drmb200_build_link_table_fused_backward(_ptr(raw), _ptr(g_table), _ptr(flat), _ptr(src), _ptr(kind),
                                                               raw.shape[0], flat.numel(), _ptr(scratch), _ptr(g_flat),
                                                               _stream())
        _check(rc, "drmb200_build_link_table_fused_backward")
        return g_flat, None, None, None, None


class FkJacobianFunction(torch.autograd.Function):
    """(table, q) -> (pos, quat, jac_lin, jac_ang); analytic backward kernel (SURVEY.md Appendix B.1)."""

    @staticmethod
    def forward(ctx, table, q, topo, ee_link, want_pos, want_quat, want_jac):
        table, q = table.contiguous(), q.contiguous()
        pos, quat, jlin, jang = fk_jacobian_raw(topo, ee_link, table, q, want_pos, want_quat, want_jac)
        ctx.save_for_backward(table, q)
        ctx.topo, ctx.ee_link = topo, ee_link
        return pos, quat, jlin, jang           # skipped outputs are None

    @staticmethod
    def backward(ctx, g_pos, g_quat, g_jlin, g_jang):
        table, q = ctx.saved_tensors
        need_table, need_q = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        B, n = q.shape
        g = [None if t is None else t.contiguous() for t in (g_pos, g_quat, g_jlin, g_jang)]
        _require_cuda(*g)
        q_grad = torch.empty_like(q) if need_q else None
        table_grad = torch.zeros_like(table) if need_table else None
        ws = _workspace(ctx.topo, B, q.device)
        with _on(q.device):
            rc = lib().drmb200_fk_jacobian_backward(ctypes.byref(ctx.topo), ctx.ee_link, _ptr(table), _ptr(q), B,
                                                    _ptr(g[0]), _ptr(g[1]), _ptr(g[2]), _ptr(g[3]), _ptr(q_grad),
                                                    _ptr(table_grad), _ptr(ws), _stream())
        _check(rc, "drmb200_fk_jacobian_backward")
        return table_grad, q_grad, None, None, None, None, None


class FkJacobianMultiFunction(torch.autograd.Function):
    """(table, q) -> stacked (pos, quat, jac_lin, jac_ang) of several links: one tree-walk launch forward; the adjoint is
    the sum of the single-link adjoints, one launch of the FK backward kernel per link with a non-zero upstream gradient
    (q_grad summed, table_grad accumulated in place by the kernel)."""

    @staticmethod
    def forward(ctx, table, q, topo, ee_links, want_pos, want_quat, want_jac):
        table, q = table.contiguous(), q.contiguous()
        outs = fk_jacobian_multi_raw(topo, ee_links, table, q, want_pos, want_quat, want_jac)
        ctx.save_for_backward(table, q)
        ctx.topo, ctx.ee_links = topo, tuple(ee_links)
        return outs

    @staticmethod
    def backward(ctx, g_pos, g_quat, g_jlin, g_jang):
        table, q = ctx.saved_tensors
        need_table, need_q = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        B, n = q.shape
        table_grad = torch.zeros_like(table) if need_table else None
        q_grad = torch.zeros_like(q) if need_q else None
        ws = _workspace(ctx.topo, B, q.device)
        for e, link in enumerate(ctx.ee_links):
            g = [None if t is None else t[e].contiguous() for t in (g_pos, g_quat, g_jlin, g_jang)]
            if all(t is None for t in g):
                continue
            _require_cuda(*g)
            q_grad_e = torch.empty_like(q) if need_q else None
            with _on(q.device):
                rc = lib().drmb200_fk_jacobian_backward(ctypes.byref(ctx.topo), int(link), _ptr(table), _ptr(q), B,
                                                        _ptr(g[0]), _ptr(g[1]), _ptr(g[2]), _ptr(g[3]), _ptr(q_grad_e),
                                                        _ptr(table_grad), _ptr(ws), _stream())
            _check(rc, "drmb200_fk_jacobian_backward")
            if need_q:
                q_grad += q_grad_e
        return table_grad, q_grad, None, None, None, None, None


class AllLinksFkFunction(torch.autograd.Function):
    """(table, q) -> (pos [N, B, 3], quat [N, B, 4]) of EVERY link: one launch of the all-links kernel forward; the adjoint
    is the sum of the single-link adjoints (one FK backward launch per link whose outputs received a gradient)."""

    @staticmethod
    def forward(ctx, table, q, topo):
        table, q = table.contiguous(), q.contiguous()
        poses, quats, _ = kinematic_state_raw(topo, table, q, None, want_poses=True, want_quats=True)
        ctx.save_for_backward(table, q)
        ctx.topo = topo
        pos = poses[:, 9:12].transpose(1, 2).contiguous()       # [N, B, 3]
        quat = quats.transpose(1, 2).contiguous()               # [N, B, 4]
        return pos, quat

    @staticmethod
    def backward(ctx, g_pos, g_quat):
        table, q = ctx.saved_tensors
        need_table, need_q = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        B, n = q.shape
        N = ctx.topo.n_links
        table_grad = torch.zeros_like(table) if need_table else None
        q_grad = torch.zeros_like(q) if need_q else None
        ws = _workspace(ctx.topo, B, q.device)
        # links whose outputs received no gradient are skipped (one host read of N flags)
        used = torch.zeros(N, dtype=torch.bool, device=q.device)
        if g_pos is not None:
            used |= g_pos.reshape(N, -1).ne(0).any(dim=1)
        if g_quat is not None:
            used |= g_quat.reshape(N, -1).ne(0).any(dim=1)
        for link in torch.nonzero(used).flatten().tolist():
            if link == 0:
                continue                                         # the root pose is constant
            gp = None if g_pos is None else g_pos[link].contiguous()
            gq = None if g_quat is None else g_quat[link].contiguous()
            _require_cuda(gp, gq)
            q_grad_l = torch.empty_like(q) if need_q else None
            with _on(q.device):
                rc = lib().drmb200_fk_jacobian_backward(ctypes.byref(ctx.topo), int(link), _ptr(table), _ptr(q), B, _ptr(gp),
                                                        _ptr(gq), None, None, _ptr(q_grad_l), _ptr(table_grad), _ptr(ws),
                                                        _stream())
            _check(rc, "drmb200_fk_jacobian_backward")
            if need_q:
                q_grad += q_grad_l
        return table_grad, q_grad, None


class InverseDynamicsFunction(torch.autograd.Function):
    """(table, q, qd, qdd) -> tau; analytic RNEA adjoint kernel (SURVEY.md Appendix B.2)."""

    @staticmethod
    def forward(ctx, table, q, qd, qdd, topo, flags, folded=None):
        table, q, qd, qdd = table.contiguous(), q.contiguous(), qd.contiguous(), qdd.contiguous()
        tau = inverse_dynamics_raw(topo, table, q, qd, qdd, flags, folded=folded)
        ctx.save_for_backward(table, q, qd, qdd)
        ctx.topo, ctx.flags = topo, flags
        return tau

    @staticmethod
    def backward(ctx, g_tau):
        table, q, qd, qdd = ctx.saved_tensors
        need = ctx.needs_input_grad
        B, n = q.shape
        g_tau = g_tau.contiguous()
        _require_cuda(g_tau)
        table_grad = torch.zeros_like(table) if need[0] else None
        q_grad = torch.empty_like(q) if need[1] else None
        qd_grad = torch.empty_like(q) if need[2] else None
        qdd_grad = torch.empty_like(q) if need[3] else None
        ws = _workspace(ctx.topo, B, q.device)
        flags = ctx.flags
        if need[1] or need[2] or need[3] or not need[0]:
            flags &= ~INERTIAL_GRADS_ONLY                   # the single-sweep kernel only produces table columns
        with _on(q.device):
            rc = lib().drmb200_inverse_dynamics_backward(
                ctypes.byref(ctx.topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(qdd), B, flags, _ptr(g_tau), _ptr(q_grad), _ptr(qd_grad), _ptr(qdd_grad),
                _ptr(table_grad), _ptr(ws), _stream())
        _check(rc, "drmb200_inverse_dynamics_backward")
        return table_grad, q_grad, qd_grad, qdd_grad, None, None, None


class ForwardDynamicsFunction(torch.autograd.Function):
    """(table, q, qd, f) -> qdd; articulated-body kernel forward, analytic adjoint kernel backward."""

    @staticmethod
    def forward(ctx, table, q, qd, f, topo, flags, folded=None):
        table, q, qd, f = table.contiguous(), q.contiguous(), qd.contiguous(), f.contiguous()
        qdd = forward_dynamics_raw(topo, table, q, qd, f, flags, folded=folded)
        ctx.save_for_backward(table, q, qd, f)
        ctx.topo, ctx.flags = topo, flags
        return qdd

    @staticmethod
    def backward(ctx, g_qdd):
        table, q, qd, f = ctx.saved_tensors
        need = ctx.needs_input_grad
        B, n = q.shape
        g_qdd = g_qdd.contiguous()
        _require_cuda(g_qdd)
        table_grad = torch.zeros_like(table) if need[0] else None
        q_grad = torch.empty_like(q) if need[1] else None
        qd_grad = torch.empty_like(q) if need[2] else None
        f_grad = torch.empty_like(q) if need[3] else None
        nbytes = int(lib().drmb200_forward_dynamics_backward_workspace_bytes(ctypes.byref(ctx.topo), B))
        ws = torch.empty((nbytes + 3) // 4, device=q.device, dtype=torch.float32)
        with _on(q.device):
            rc = lib().drmb200_forward_dynamics_backward(
                ctypes.byref(ctx.topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B, ctx.flags, _ptr(g_qdd), _ptr(q_grad), _ptr(qd_grad),
                _ptr(f_grad), _ptr(table_grad), _ptr(ws), _stream())
        _check(rc, "drmb200_forward_dynamics_backward")
        return table_grad, q_grad, qd_grad, f_grad, None, None, None


def mass_matrix_raw(topo, table, q, out=None, folded=None):
    """Joint-space inertia matrix [B, n, n], one launch (drmb200_mass_matrix; `folded`: rows of fold_link_table)."""
    _require_cuda(table, q, folded)
    q = q.contiguous()
    B, n = q.shape
    H = out if out is not None else torch.empty((B, n, n), device=q.device, dtype=torch.float32)
    with _on(q.device):
        if folded is not None:
            rc = lib().drmb200_mass_matrix_prefolded(ctypes.byref(topo), _ptr(folded), _ptr(q), B, _ptr(H), _stream())
        else:
            rc = lib().drmb200_mass_matrix(ctypes.byref(topo), _ptr(table), _ptr(q), B, _ptr(H), _stream())
    _check(rc, "drmb200_mass_matrix")
    return H


class MassMatrixFunction(torch.autograd.Function):
    """(table, q) -> H [B, n, n].  Forward: the mass-matrix kernel.  Backward: column j of H is the inverse-dynamics
    torque for (q, qd = 0, qdd = e_j) without gravity or damping, so the adjoint is ONE launch of the RNEA adjoint
    kernel over the n stacked unit-acceleration batches (q_grad summed over the stack, table_grad as is)."""

    @staticmethod
    def forward(ctx, table, q, topo, folded=None):
        table, q = table.contiguous(), q.contiguous()
        H = mass_matrix_raw(topo, table, q, folded=folded)
        ctx.save_for_backward(table, q)
        ctx.topo = topo
        return H

    @staticmethod
    def backward(ctx, g_H):
        table, q = ctx.saved_tensors
        need_table, need_q = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        B, n = q.shape
        _require_cuda(g_H)
        qs = q.repeat(n, 1)                                            # slab j = the batch with qdd = e_j
        zeros = torch.zeros_like(qs)
        qdd = zeros.view(n, B, n).clone()
        idx = torch.arange(n, device=q.device)
        qdd[idx, :, idx] = 1.0
        g_tau = g_H.permute(2, 0, 1).contiguous().view(n * B, n)       # slab j: dL/dH[:, :, j]
        table_grad = torch.zeros_like(table) if need_table else None
        q_grad = torch.empty_like(qs) if need_q else None
        ws = _workspace(ctx.topo, n * B, q.device)
        with _on(q.device):
            rc = lib().drmb200_inverse_dynamics_backward(
                ctypes.byref(ctx.topo), _ptr(table), _ptr(qs), _ptr(zeros), _ptr(qdd.view(n * B, n)), n * B, 0, _ptr(g_tau),
                _ptr(q_grad), None, None, _ptr(table_grad), _ptr(ws), _stream())
        _check(rc, "drmb200_inverse_dynamics_backward")
        return table_grad, (q_grad.view(n, B, n).sum(0) if need_q else None), None, None
