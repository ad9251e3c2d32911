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
IMPLICIT_DAMPING = 8         # rollouts: the damping torque taken at the end-of-step velocity (see include/drm_b200.h)
IMPLICIT_GAINS = 16          # PD rollout: the PD law taken at the end-of-step state, stable PD (see include/drm_b200.h)

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
    "drmb200_forward_dynamics_implicit_damping": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                                 _c_float_p, ctypes.c_int64, ctypes.c_uint32, ctypes.c_float,
                                                                 _c_float_p, ctypes.c_void_p]),
    "drmb200_forward_dynamics_implicit_damping_backward": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p,
                                                                          _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_uint32,
                                                                          ctypes.c_float, _c_float_p, _c_float_p, _c_float_p,
                                                                          _c_float_p, _c_float_p, ctypes.c_void_p,
                                                                          ctypes.c_void_p]),
    "drmb200_forward_dynamics_rollout": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                        ctypes.c_int64, ctypes.c_int32, ctypes.c_float, ctypes.c_uint32,
                                                        _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_forward_dynamics_rollout_backward_workspace_bytes": (ctypes.c_int64, [ctypes.POINTER(Topology), ctypes.c_int64]),
    "drmb200_forward_dynamics_rollout_backward": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                                 _c_float_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_float,
                                                                 ctypes.c_uint32, _c_float_p, _c_float_p, _c_float_p,
                                                                 _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                                 _c_float_p, ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_pd_rollout": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                          _c_float_p, _c_float_p, _c_float_p, ctypes.c_int32, _c_float_p, ctypes.c_int64,
                                          ctypes.c_int32, ctypes.c_float, ctypes.c_uint32, _c_float_p, _c_float_p, _c_float_p,
                                          _c_float_p, ctypes.c_void_p]),
    "drmb200_pd_rollout_backward_workspace_bytes": (ctypes.c_int64, [ctypes.POINTER(Topology), ctypes.c_int64]),
    "drmb200_pd_rollout_backward": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                   _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int32, _c_float_p,
                                                   ctypes.c_int64, ctypes.c_int32, ctypes.c_float, ctypes.c_uint32, _c_float_p,
                                                   _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                   _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                   _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_inverse_dynamics_derivatives": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                            _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p, _c_float_p,
                                                            ctypes.c_void_p]),
    "drmb200_inverse_dynamics_derivatives_prefolded": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                                      _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p,
                                                                      _c_float_p, ctypes.c_void_p]),
    "drmb200_forward_dynamics_derivatives": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                            _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p, _c_float_p,
                                                            _c_float_p, ctypes.c_void_p]),
    "drmb200_forward_dynamics_derivatives_prefolded": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p,
                                                                      _c_float_p, ctypes.c_int64, ctypes.c_uint32, _c_float_p,
                                                                      _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_inverse_kinematics": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, _c_float_p, _c_float_p, _c_float_p,
                                                  _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int32,
                                                  ctypes.c_float, ctypes.c_float, ctypes.c_float, _c_float_p, _c_float_p,
                                                  _c_float_p, ctypes.c_void_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_inverse_kinematics_multi": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32),
                                                        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                        _c_float_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_float, ctypes.c_float,
                                                        ctypes.c_float, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                                        _c_float_p, ctypes.c_void_p]),
    "drmb200_operational_space_dynamics": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32,
                                                          ctypes.POINTER(ctypes.c_int32), _c_float_p, _c_float_p, _c_float_p,
                                                          _c_float_p, ctypes.c_int64, ctypes.c_uint32, ctypes.c_int32,
                                                          _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_contact_dynamics": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32),
                                                _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64,
                                                ctypes.c_uint32, ctypes.c_int32, ctypes.c_float, _c_float_p, _c_float_p,
                                                ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_contact_impulse": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32),
                                               _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64, ctypes.c_int32,
                                               ctypes.c_float, _c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_contact_backward_workspace_bytes": (ctypes.c_int64, [ctypes.POINTER(Topology), ctypes.c_int32,
                                                                  ctypes.POINTER(ctypes.c_int32), ctypes.c_int32, ctypes.c_int64]),
    "drmb200_contact_dynamics_backward": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32),
                                                         _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                         _c_float_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint32,
                                                         ctypes.c_int32, ctypes.c_float, _c_float_p, _c_float_p, _c_float_p,
                                                         _c_float_p, _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                                         ctypes.c_void_p]),
    "drmb200_contact_impulse_backward": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32),
                                                        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_float,
                                                        _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                        ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_contact_rollout": (ctypes.c_int, [ctypes.POINTER(Topology), ctypes.c_int32, ctypes.POINTER(ctypes.c_int32),
                                               _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                               ctypes.c_int64, ctypes.c_int32, ctypes.c_float, ctypes.c_uint32, ctypes.c_int32,
                                               ctypes.c_float, ctypes.c_float, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                               _c_float_p, ctypes.c_void_p, ctypes.c_void_p]),
    "drmb200_dynamics_regressor": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                                  ctypes.c_int64, ctypes.c_uint32, _c_float_p, ctypes.c_void_p]),
    "drmb200_energy_momentum": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64,
                                               _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p, _c_float_p,
                                               ctypes.c_void_p]),
    "drmb200_kinematic_state": (ctypes.c_int, [ctypes.POINTER(Topology), _c_float_p, _c_float_p, _c_float_p, ctypes.c_int64,
                                               _c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_build_link_table": (ctypes.c_int, [_c_float_p, ctypes.c_int32, _c_float_p, ctypes.c_void_p]),
    "drmb200_build_link_table_backward": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_int32, _c_float_p,
                                                         ctypes.c_void_p]),
    "drmb200_build_link_table_fused": (ctypes.c_int, [_c_float_p, _c_float_p, ctypes.c_void_p, ctypes.c_void_p, _c_float_p,
                                                      ctypes.c_int32, _c_float_p, _c_float_p, ctypes.c_void_p]),
    "drmb200_build_link_table_fused_backward": (ctypes.c_int, [_c_float_p, _c_float_p, _c_float_p, ctypes.c_void_p,
                                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                                               _c_float_p, _c_float_p, ctypes.c_void_p]),
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


def forward_dynamics_raw(topo, table, q, qd, f, flags, out=None, folded=None, implicit_dt=None):
    """Articulated-body algorithm, one launch (drmb200_forward_dynamics; `folded`: rows of fold_link_table for an unchanged table).
    implicit_dt: implicit damping with that step (drmb200_forward_dynamics_implicit_damping, on the unfolded table)."""
    _require_cuda(table, q, qd, f, folded)
    q, qd, f = q.contiguous(), qd.contiguous(), f.contiguous()
    B, n = q.shape
    qdd = out if out is not None else torch.empty((B, n), device=q.device, dtype=torch.float32)
    with _on(q.device):
        if implicit_dt is not None:
            rc = lib().drmb200_forward_dynamics_implicit_damping(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B,
                                                                 flags, ctypes.c_float(implicit_dt), _ptr(qdd), _stream())
            _check(rc, "drmb200_forward_dynamics_implicit_damping")
            return qdd
        if folded is not None:
            rc = lib().drmb200_forward_dynamics_prefolded(ctypes.byref(topo), _ptr(folded), _ptr(q), _ptr(qd), _ptr(f), B,
                                                          flags, _ptr(qdd), _stream())
        else:
            rc = lib().drmb200_forward_dynamics(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B,
                                                flags, _ptr(qdd), _stream())
    _check(rc, "drmb200_forward_dynamics")
    return qdd


def inverse_dynamics_derivatives_raw(topo, table, q, qd, qdd, flags, folded=None, want_dq=True, want_dqd=True):
    """(dtau_dq, dtau_dqd) [B, n, n], out[b, i, j] = d tau_i / d x_j, one launch (drmb200_inverse_dynamics_derivatives;
    `folded`: rows of fold_link_table for an unchanged table).  A matrix that is not wanted is None."""
    _require_cuda(table, q, qd, qdd, folded)
    q, qd, qdd = q.contiguous(), qd.contiguous(), qdd.contiguous()
    B, n = q.shape
    dq = torch.empty((B, n, n), device=q.device, dtype=torch.float32) if want_dq else None
    dqd = torch.empty((B, n, n), device=q.device, dtype=torch.float32) if want_dqd else None
    with _on(q.device):
        if folded is not None:
            rc = lib().drmb200_inverse_dynamics_derivatives_prefolded(ctypes.byref(topo), _ptr(folded), _ptr(q), _ptr(qd), _ptr(qdd),
                                                                      B, flags & 3, _ptr(dq), _ptr(dqd), _stream())
        else:
            rc = lib().drmb200_inverse_dynamics_derivatives(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(qdd), B,
                                                            flags & 3, _ptr(dq), _ptr(dqd), _stream())
    _check(rc, "drmb200_inverse_dynamics_derivatives")
    return dq, dqd


def forward_dynamics_derivatives_raw(topo, table, q, qd, f, flags, folded=None, want_dq=True, want_dqd=True, want_df=True):
    """(dqdd_dq, dqdd_dqd, dqdd_df) [B, n, n], out[b, i, j] = d qdd_i / d x_j, one launch
    (drmb200_forward_dynamics_derivatives; `folded`: rows of fold_link_table for an unchanged table)."""
    _require_cuda(table, q, qd, f, folded)
    q, qd, f = q.contiguous(), qd.contiguous(), f.contiguous()
    B, n = q.shape
    outs = [torch.empty((B, n, n), device=q.device, dtype=torch.float32) if want else None
            for want in (want_dq, want_dqd, want_df)]
    with _on(q.device):
        if folded is not None:
            rc = lib().drmb200_forward_dynamics_derivatives_prefolded(ctypes.byref(topo), _ptr(folded), _ptr(q), _ptr(qd), _ptr(f),
                                                                      B, flags & 3, *[_ptr(o) for o in outs], _stream())
        else:
            rc = lib().drmb200_forward_dynamics_derivatives(ctypes.byref(topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B,
                                                            flags & 3, *[_ptr(o) for o in outs], _stream())
    _check(rc, "drmb200_forward_dynamics_derivatives")
    return tuple(outs)


def dynamics_regressor_raw(topo, table, q, qd, qdd, flags, out=None):
    """Y [B, n, n_links, 14], Y[b, i, l, k] = d tau_i / d table[l, 12 + k], so that einsum("bilk,lk->bi", Y, table[:, 12:26])
    is the inverse dynamics of the same inputs; one launch (drmb200_dynamics_regressor, always on the unfolded table)."""
    _require_cuda(table, q, qd, qdd, out)
    q, qd, qdd = q.contiguous(), qd.contiguous(), qdd.contiguous()
    B, n = q.shape
    Y = out if out is not None else torch.empty((B, n, topo.n_links, 14), device=q.device, dtype=torch.float32)
    with _on(q.device):
        rc = lib().drmb200_dynamics_regressor(ctypes.byref(topo), _ptr(table.contiguous()), _ptr(q), _ptr(qd), _ptr(qdd), B,
                                              flags & 3, _ptr(Y), _stream())
    _check(rc, "drmb200_dynamics_regressor")
    return Y


def energy_momentum_raw(topo, table, q, qd=None, want_kinetic=True, want_potential=True, want_momentum=True, want_com=True,
                        want_com_velocity=True, want_com_jacobian=True):
    """(kinetic [B], potential [B], momentum [B, n], com [B, 3], com_velocity [B, 3], com_jacobian [B, 3, n]), one launch
    (drmb200_energy_momentum, always on the unfolded table).  An output not wanted is None; without qd the velocity-dependent
    ones (kinetic, momentum, com_velocity) are None as well."""
    _require_cuda(table, q, qd)
    q = q.contiguous()
    qd = None if qd is None else qd.contiguous()
    B, n = q.shape
    dev = q.device
    has_qd = qd is not None
    shapes = ((B,), (B,), (B, n), (B, 3), (B, 3), (B, 3, n))
    wants = (want_kinetic and has_qd, want_potential, want_momentum and has_qd, want_com, want_com_velocity and has_qd,
             want_com_jacobian)
    outs = [torch.empty(s, device=dev, dtype=torch.float32) if w else None for s, w in zip(shapes, wants)]
    with _on(dev):
        rc = lib().drmb200_energy_momentum(ctypes.byref(topo), _ptr(table.contiguous()), _ptr(q), _ptr(qd), B,
                                           *[_ptr(o) for o in outs], _stream())
    _check(rc, "drmb200_energy_momentum")
    return tuple(outs)


def forward_dynamics_rollout_raw(topo, table, q0, qd0, f, dt, flags, want_qdd=True):
    """(q, qd, qdd) [T, B, n] of T semi-implicit Euler steps over the articulated-body algorithm, one launch
    (drmb200_forward_dynamics_rollout); qdd is None unless want_qdd."""
    _require_cuda(table, q0, qd0, f)
    q0, qd0, f = q0.contiguous(), qd0.contiguous(), f.contiguous()
    T, B, n = f.shape
    dev = q0.device
    q = torch.empty((T, B, n), device=dev, dtype=torch.float32)
    qd = torch.empty((T, B, n), device=dev, dtype=torch.float32)
    qdd = torch.empty((T, B, n), device=dev, dtype=torch.float32) if want_qdd else None
    with _on(dev):
        rc = lib().drmb200_forward_dynamics_rollout(ctypes.byref(topo), _ptr(table), _ptr(q0), _ptr(qd0), _ptr(f), B, T,
                                                    ctypes.c_float(dt), flags, _ptr(q), _ptr(qd), _ptr(qdd), _stream())
    _check(rc, "drmb200_forward_dynamics_rollout")
    return q, qd, qdd


def pd_rollout_raw(topo, table, q0, qd0, q_ref, kp, kd, dt, flags, qd_ref=None, f=None, effort_limit=None, want_qdd=True):
    """(q, qd, qdd, tau) [T, B, n] of T semi-implicit Euler steps over the articulated-body algorithm driven by the PD law
    tau = clamp(f + kp (q_ref - q) + kd (qd_ref - qd), -effort_limit, effort_limit), one launch (drmb200_pd_rollout;
    IMPLICIT_GAINS in flags: the law at the end-of-step state).  kp / kd both [n] (shared) or both [B, n] (per row); qd_ref,
    f, effort_limit may be None; qdd is None unless want_qdd."""
    _require_cuda(table, q0, qd0, q_ref, kp, kd, qd_ref, f, effort_limit)
    if kp.shape != kd.shape:      # one gains_per_row flag describes both buffers
        raise RuntimeError(f"kp and kd must have the same shape (got {tuple(kp.shape)} and {tuple(kd.shape)})")
    q0, qd0, q_ref, kp, kd = (t.contiguous() for t in (q0, qd0, q_ref, kp, kd))
    qd_ref, f, effort_limit = (None if t is None else t.contiguous() for t in (qd_ref, f, effort_limit))
    T, B, n = q_ref.shape
    dev = q0.device
    q, qd, tau = (torch.empty((T, B, n), device=dev, dtype=torch.float32) for _ in range(3))
    qdd = torch.empty((T, B, n), device=dev, dtype=torch.float32) if want_qdd else None
    with _on(dev):
        rc = lib().drmb200_pd_rollout(ctypes.byref(topo), _ptr(table), _ptr(q0), _ptr(qd0), _ptr(q_ref), _ptr(qd_ref), _ptr(f),
                                      _ptr(kp), _ptr(kd), 1 if kp.ndim == 2 else 0, _ptr(effort_limit), B, T, ctypes.c_float(dt),
                                      flags, _ptr(q), _ptr(qd), _ptr(qdd), _ptr(tau), _stream())
    _check(rc, "drmb200_pd_rollout")
    return q, qd, qdd, tau


IK_DAMPING_INIT = 1e-2       # suggested initial Levenberg-Marquardt damping (include/drm_b200.h)
IK_DAMPING_MIN = 1e-5        # compiled into csrc/inverse_kinematics.cu
IK_DAMPING_MAX = 1e5


def inverse_kinematics_raw(topo, ee_link, table, q0, target_pos, target_quat=None, lower=None, upper=None, damping=None,
                           max_iters=100, damping_init=IK_DAMPING_INIT, pos_tol=1e-4, rot_tol=1e-3):
    """Levenberg-Marquardt inverse kinematics of link `ee_link`, all iterations in one launch (drmb200_inverse_kinematics).
    q0 [B, n], target_pos [B, 3], target_quat [B, 4] xyzw or None (position only), lower / upper [n] or None, damping [B]
    or None (damping_init for every row).  Returns (q [B, n], pos_err [B], rot_err [B], converged [B] bool, damping [B])."""
    _require_cuda(table, q0, target_pos, target_quat, lower, upper, damping)
    q0, target_pos = q0.contiguous(), target_pos.contiguous()
    target_quat = None if target_quat is None else target_quat.contiguous()
    lower = None if lower is None else lower.contiguous()
    upper = None if upper is None else upper.contiguous()
    damping = None if damping is None else damping.contiguous()
    B, n = q0.shape
    dev = q0.device
    q = torch.empty((B, n), device=dev, dtype=torch.float32)
    pos_err = torch.empty(B, device=dev, dtype=torch.float32)
    rot_err = torch.empty(B, device=dev, dtype=torch.float32)
    converged = torch.empty(B, device=dev, dtype=torch.uint8)
    damping_out = torch.empty(B, device=dev, dtype=torch.float32)
    with _on(dev):
        rc = lib().drmb200_inverse_kinematics(ctypes.byref(topo), ee_link, _ptr(table), _ptr(q0), _ptr(target_pos),
                                              _ptr(target_quat), _ptr(lower), _ptr(upper), _ptr(damping), B, int(max_iters),
                                              ctypes.c_float(damping_init), ctypes.c_float(pos_tol), ctypes.c_float(rot_tol),
                                              _ptr(q), _ptr(pos_err), _ptr(rot_err), _ptr(converged), _ptr(damping_out),
                                              _stream())
    _check(rc, "drmb200_inverse_kinematics")
    return q, pos_err, rot_err, converged.view(torch.bool), damping_out


def inverse_kinematics_multi_raw(topo, ee_links, table, q0, target_pos, target_quat=None, lower=None, upper=None, damping=None,
                                 max_iters=100, damping_init=IK_DAMPING_INIT, pos_tol=1e-4, rot_tol=1e-3):
    """Levenberg-Marquardt inverse kinematics of several links at once, one solve over their stacked errors, all iterations
    in one launch (drmb200_inverse_kinematics_multi).  q0 [B, n], target_pos [n_ee, B, 3], target_quat [n_ee, B, 4] xyzw or
    None (position only), lower / upper [n] or None, damping [B] or None.  Returns (q [B, n], pos_err [n_ee, B],
    rot_err [n_ee, B], converged [B] bool, damping [B])."""
    _require_cuda(table, q0, target_pos, target_quat, lower, upper, damping)
    q0, target_pos = q0.contiguous(), target_pos.contiguous()
    target_quat = None if target_quat is None else target_quat.contiguous()
    lower = None if lower is None else lower.contiguous()
    upper = None if upper is None else upper.contiguous()
    damping = None if damping is None else damping.contiguous()
    B, n = q0.shape
    dev, E = q0.device, len(ee_links)
    q = torch.empty((B, n), device=dev, dtype=torch.float32)
    pos_err = torch.empty((E, B), device=dev, dtype=torch.float32)
    rot_err = torch.empty((E, B), device=dev, dtype=torch.float32)
    converged = torch.empty(B, device=dev, dtype=torch.uint8)
    damping_out = torch.empty(B, device=dev, dtype=torch.float32)
    links = (ctypes.c_int32 * max(E, 1))(*[int(l) for l in ee_links])
    with _on(dev):
        rc = lib().drmb200_inverse_kinematics_multi(ctypes.byref(topo), E, links, _ptr(table), _ptr(q0), _ptr(target_pos),
                                                    _ptr(target_quat), _ptr(lower), _ptr(upper), _ptr(damping), B,
                                                    int(max_iters), ctypes.c_float(damping_init), ctypes.c_float(pos_tol),
                                                    ctypes.c_float(rot_tol), _ptr(q), _ptr(pos_err), _ptr(rot_err),
                                                    _ptr(converged), _ptr(damping_out), _stream())
    _check(rc, "drmb200_inverse_kinematics_multi")
    return q, pos_err, rot_err, converged.view(torch.bool), damping_out


def operational_space_dynamics_raw(topo, ee_links, table, q, qd, f, flags, position_only=False, want_inv_inertia=True,
                                   want_acceleration=True, want_velocity=True, want_bias=True):
    """(inv_inertia [B, M, M], acceleration [B, M], velocity [B, M], bias_acceleration [B, M]) of the links `ee_links`,
    M = 6 len(ee_links) (3 with position_only), one launch (drmb200_operational_space_dynamics); an output not wanted is
    None."""
    _require_cuda(table, q, qd, f)
    q, qd, f = q.contiguous(), qd.contiguous(), f.contiguous()
    B = q.shape[0]
    E = len(ee_links)
    M = (3 if position_only else 6) * E
    dev = q.device
    inv = torch.empty((B, M, M), device=dev, dtype=torch.float32) if want_inv_inertia else None
    vecs = [torch.empty((B, M), device=dev, dtype=torch.float32) if want else None
            for want in (want_acceleration, want_velocity, want_bias)]
    links = (ctypes.c_int32 * max(E, 1))(*[int(l) for l in ee_links])
    with _on(dev):
        rc = lib().drmb200_operational_space_dynamics(ctypes.byref(topo), E, links, _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B,
                                                      flags & 3, 1 if position_only else 0, _ptr(inv),
                                                      *[_ptr(v) for v in vecs], _stream())
    _check(rc, "drmb200_operational_space_dynamics")
    return (inv, *vecs)


CONTACT_PIVOT_MIN = 1e-5     # compiled into csrc/contact_dynamics.cu: smallest pivot of the equilibrated system that solves


def contact_dynamics_raw(topo, ee_links, table, q, qd, f, flags, accel_ref=None, position_only=False, regularization=0.0,
                         want_force=True):
    """(qdd [B, n], force [B, M] or None, solved [B] bool) of rigid contacts at the links `ee_links`, M = 6 len(ee_links)
    (3 with position_only), one launch (drmb200_contact_dynamics).  accel_ref [B, M] or None (0)."""
    _require_cuda(table, q, qd, f, accel_ref)
    q, qd, f = q.contiguous(), qd.contiguous(), f.contiguous()
    accel_ref = None if accel_ref is None else accel_ref.contiguous()
    B, n = q.shape
    E = len(ee_links)
    M = (3 if position_only else 6) * E
    if accel_ref is not None and tuple(accel_ref.shape) != (B, M):
        raise RuntimeError(f"accel_ref: expected shape {(B, M)}, got {tuple(accel_ref.shape)}")
    dev = q.device
    qdd = torch.empty((B, n), device=dev, dtype=torch.float32)
    force = torch.empty((B, M), device=dev, dtype=torch.float32) if want_force else None
    solved = torch.empty(B, device=dev, dtype=torch.uint8)
    links = (ctypes.c_int32 * max(E, 1))(*[int(l) for l in ee_links])
    with _on(dev):
        rc = lib().drmb200_contact_dynamics(ctypes.byref(topo), E, links, _ptr(table), _ptr(q), _ptr(qd), _ptr(f),
                                            _ptr(accel_ref), B, flags & 3, 1 if position_only else 0,
                                            ctypes.c_float(regularization), _ptr(qdd), _ptr(force), _ptr(solved), _stream())
    _check(rc, "drmb200_contact_dynamics")
    return qdd, force, solved.view(torch.bool)


def contact_impulse_raw(topo, ee_links, table, q, qd, velocity_ref=None, position_only=False, regularization=0.0,
                        want_impulse=True):
    """(qd_plus [B, n], impulse [B, M] or None, solved [B] bool) of an impact at the links `ee_links`, M = 6 len(ee_links)
    (3 with position_only), one launch (drmb200_contact_impulse).  velocity_ref [B, M] or None (0: inelastic)."""
    _require_cuda(table, q, qd, velocity_ref)
    q, qd = q.contiguous(), qd.contiguous()
    velocity_ref = None if velocity_ref is None else velocity_ref.contiguous()
    B, n = q.shape
    E = len(ee_links)
    M = (3 if position_only else 6) * E
    if velocity_ref is not None and tuple(velocity_ref.shape) != (B, M):
        raise RuntimeError(f"velocity_ref: expected shape {(B, M)}, got {tuple(velocity_ref.shape)}")
    dev = q.device
    qd_plus = torch.empty((B, n), device=dev, dtype=torch.float32)
    impulse = torch.empty((B, M), device=dev, dtype=torch.float32) if want_impulse else None
    solved = torch.empty(B, device=dev, dtype=torch.uint8)
    links = (ctypes.c_int32 * max(E, 1))(*[int(l) for l in ee_links])
    with _on(dev):
        rc = lib().drmb200_contact_impulse(ctypes.byref(topo), E, links, _ptr(table), _ptr(q), _ptr(qd), _ptr(velocity_ref), B,
                                           1 if position_only else 0, ctypes.c_float(regularization), _ptr(qd_plus),
                                           _ptr(impulse), _ptr(solved), _stream())
    _check(rc, "drmb200_contact_impulse")
    return qd_plus, impulse, solved.view(torch.bool)


def _contact_workspace(topo, links, position_only, batch, device):
    nbytes = int(lib().drmb200_contact_backward_workspace_bytes(ctypes.byref(topo), len(links), links,
                                                               1 if position_only else 0, batch))
    return torch.empty((max(nbytes, 4) + 3) // 4, device=device, dtype=torch.float32)


def contact_dynamics_backward_raw(topo, ee_links, table, q, qd, f, qdd, force, solved, flags, g_qdd=None, g_force=None,
                                  accel_ref=None, position_only=False, regularization=0.0, want_q=True, want_qd=True,
                                  want_f=True, want_accel_ref=True, want_table=True):
    """(q_grad, qd_grad, f_grad [B, n], accel_ref_grad [B, M], table_grad [n_links, 28]) of drmb200_contact_dynamics at the
    forward's outputs (qdd, force, solved) for the upstream gradients g_qdd [B, n] / g_force [B, M] (None: zero), in at most
    five launches (drmb200_contact_dynamics_backward); an output not wanted is None.  Unsolved rows get zero gradients."""
    _require_cuda(table, q, qd, f, qdd, force, g_qdd, g_force, accel_ref)
    table, q, qd, f, qdd, force = (t.contiguous() for t in (table, q, qd, f, qdd, force))
    g_qdd, g_force, accel_ref = (None if t is None else t.contiguous() for t in (g_qdd, g_force, accel_ref))
    solved = solved.contiguous().view(torch.uint8)
    B, n = q.shape
    E = len(ee_links)
    M = (3 if position_only else 6) * E
    dev = q.device
    outs = [torch.empty((B, n), device=dev, dtype=torch.float32) if w else None for w in (want_q, want_qd, want_f)]
    ref_grad = torch.empty((B, M), device=dev, dtype=torch.float32) if want_accel_ref else None
    table_grad = torch.zeros_like(table) if want_table else None
    links = (ctypes.c_int32 * max(E, 1))(*[int(l) for l in ee_links])
    ws = _contact_workspace(topo, links, position_only, B, dev)
    with _on(dev):
        rc = lib().drmb200_contact_dynamics_backward(ctypes.byref(topo), E, links, _ptr(table), _ptr(q), _ptr(qd), _ptr(f),
                                                     _ptr(accel_ref), _ptr(qdd), _ptr(force), _ptr(solved), B, flags & 3,
                                                     1 if position_only else 0, ctypes.c_float(regularization), _ptr(g_qdd),
                                                     _ptr(g_force), *[_ptr(t) for t in outs], _ptr(ref_grad), _ptr(table_grad),
                                                     _ptr(ws), _stream())
    _check(rc, "drmb200_contact_dynamics_backward")
    return (*outs, ref_grad, table_grad)


def contact_impulse_backward_raw(topo, ee_links, table, q, qd, qd_plus, impulse, solved, g_qd_plus=None, g_impulse=None,
                                 velocity_ref=None, position_only=False, regularization=0.0, want_q=True, want_qd=True,
                                 want_velocity_ref=True, want_table=True):
    """(q_grad, qd_grad [B, n], velocity_ref_grad [B, M], table_grad [n_links, 28]) of drmb200_contact_impulse at the
    forward's outputs for the upstream gradients g_qd_plus [B, n] / g_impulse [B, M] (None: zero), in at most five launches
    (drmb200_contact_impulse_backward); an output not wanted is None.  Unsolved rows get zero gradients."""
    _require_cuda(table, q, qd, qd_plus, impulse, g_qd_plus, g_impulse, velocity_ref)
    table, q, qd, qd_plus, impulse = (t.contiguous() for t in (table, q, qd, qd_plus, impulse))
    g_qd_plus, g_impulse, velocity_ref = (None if t is None else t.contiguous() for t in (g_qd_plus, g_impulse, velocity_ref))
    solved = solved.contiguous().view(torch.uint8)
    B, n = q.shape
    E = len(ee_links)
    M = (3 if position_only else 6) * E
    dev = q.device
    outs = [torch.empty((B, n), device=dev, dtype=torch.float32) if w else None for w in (want_q, want_qd)]
    ref_grad = torch.empty((B, M), device=dev, dtype=torch.float32) if want_velocity_ref else None
    table_grad = torch.zeros_like(table) if want_table else None
    links = (ctypes.c_int32 * max(E, 1))(*[int(l) for l in ee_links])
    ws = _contact_workspace(topo, links, position_only, B, dev)
    with _on(dev):
        rc = lib().drmb200_contact_impulse_backward(ctypes.byref(topo), E, links, _ptr(table), _ptr(q), _ptr(qd),
                                                    _ptr(velocity_ref), _ptr(qd_plus), _ptr(impulse), _ptr(solved), B,
                                                    1 if position_only else 0, ctypes.c_float(regularization), _ptr(g_qd_plus),
                                                    _ptr(g_impulse), *[_ptr(t) for t in outs], _ptr(ref_grad),
                                                    _ptr(table_grad), _ptr(ws), _stream())
    _check(rc, "drmb200_contact_impulse_backward")
    return (*outs, ref_grad, table_grad)


def contact_rollout_raw(topo, ee_links, table, q0, qd0, f, dt, flags, target_pos=None, target_quat=None, position_only=False,
                        regularization=0.0, stabilization=0.0, want_qdd=True, want_force=True, want_accel_ref=False):
    """(q, qd, qdd [T, B, n], force [T, B, M], accel_ref [T, B, M], solved [B] bool) of T semi-implicit Euler steps of the
    contact dynamics at the links `ee_links` with Baumgarte rate `stabilization`, one launch (drmb200_contact_rollout).
    f [T, B, n]; target_pos [n_ee, B, 3] / target_quat [n_ee, B, 4] or None (the poses at q0).  qdd / force / accel_ref are
    None unless wanted."""
    _require_cuda(table, q0, qd0, f, target_pos, target_quat)
    q0, qd0, f = q0.contiguous(), qd0.contiguous(), f.contiguous()
    target_pos = None if target_pos is None else target_pos.contiguous()
    target_quat = None if target_quat is None else target_quat.contiguous()
    T, B, n = f.shape
    E = len(ee_links)
    M = (3 if position_only else 6) * E
    dev = q0.device
    q, qd = (torch.empty((T, B, n), device=dev, dtype=torch.float32) for _ in range(2))
    qdd = torch.empty((T, B, n), device=dev, dtype=torch.float32) if want_qdd else None
    force = torch.empty((T, B, M), device=dev, dtype=torch.float32) if want_force else None
    accel_ref = torch.empty((T, B, M), device=dev, dtype=torch.float32) if want_accel_ref else None
    solved = torch.empty(B, device=dev, dtype=torch.uint8)
    links = (ctypes.c_int32 * max(E, 1))(*[int(l) for l in ee_links])
    with _on(dev):
        rc = lib().drmb200_contact_rollout(ctypes.byref(topo), E, links, _ptr(table), _ptr(q0), _ptr(qd0), _ptr(f),
                                           _ptr(target_pos), _ptr(target_quat), B, T, ctypes.c_float(dt),
                                           flags & (GRAVITY | DAMPING | IMPLICIT_DAMPING),
                                           1 if position_only else 0, ctypes.c_float(regularization),
                                           ctypes.c_float(stabilization), _ptr(q), _ptr(qd), _ptr(qdd), _ptr(force),
                                           _ptr(accel_ref), _ptr(solved), _stream())
    _check(rc, "drmb200_contact_rollout")
    return q, qd, qdd, force, accel_ref, solved.view(torch.bool)


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
SECOND_ORDER_UNSUPPORTED = (
    "second-order derivatives through the engine's kernels are not supported: the analytic backward kernels are "
    "first-order only (their gradients carry no graph of their own). Differentiate the kinematic Jacobian outputs "
    "(compute_endeffector_jacobian / compute_fk_and_jacobian) or use compute_inverse_dynamics_derivatives / "
    "compute_forward_dynamics_derivatives instead.")


class _FirstOrderOnly(torch.autograd.Function):
    """Identity on a gradient returned by a kernel backward under ``create_graph=True``.  Its inputs include the primals
    of that backward and its upstream gradients, so the result requires grad and sits on the path from them; its backward
    raises.  Without it torch treats the kernel's gradient as a constant, and a Hessian or a gradient penalty silently
    gets zeros where the second-order term should be."""

    @staticmethod
    def forward(ctx, grad, *depends_on):
        return grad.view_as(grad)

    @staticmethod
    def backward(ctx, *_):
        raise RuntimeError(SECOND_ORDER_UNSUPPORTED)


def first_order_only(grads, depends_on):
    """``grads`` (a tuple, None entries allowed) unchanged outside ``create_graph``; under it (grad mode on inside a
    backward), each gradient wrapped so that differentiating it raises, provided any tensor of ``depends_on`` requires
    grad -- otherwise no second-order path exists and nothing is wrapped."""
    if not torch.is_grad_enabled():
        return grads
    deps = [t for t in depends_on if isinstance(t, torch.Tensor) and t.requires_grad]
    if not deps:
        return grads
    return tuple(g if g is None else _FirstOrderOnly.apply(g, *deps) for g in grads)


class BuildLinkTableFunction(torch.autograd.Function):
    """raw link parameters [n_links, 20] -> link table [n_links, 28] (csrc/table.cu), one launch each way."""

    @staticmethod
    def forward(ctx, raw):
        _require_cuda(raw)
        ctx.save_for_backward(raw)
        raw = raw.contiguous()
        n_links = raw.shape[0]
        table = torch.empty((n_links, 28), device=raw.device, dtype=torch.float32)
        with _on(raw.device):
            rc = lib().drmb200_build_link_table(_ptr(raw), n_links, _ptr(table), _stream())
        _check(rc, "drmb200_build_link_table")
        return table

    @staticmethod
    def backward(ctx, g_table):
        saved = ctx.saved_tensors
        raw = saved[0].contiguous()
        g_table = g_table.contiguous()
        _require_cuda(g_table)
        g_raw = torch.empty_like(raw)
        with _on(raw.device):
            rc = lib().drmb200_build_link_table_backward(_ptr(raw), _ptr(g_table), raw.shape[0], _ptr(g_raw), _stream())
        _check(rc, "drmb200_build_link_table_backward")
        return first_order_only((g_raw,), saved + (g_table,))[0]



class FusedTableFunction(torch.autograd.Function):
    """flat link-parameter vector [P] -> link table [n_links, 28] in ONE launch (drmb200_build_link_table_fused): the
    per-(link, parameter) parametrisation modules are applied inside the kernel through an index / kind / offset map.
    Backward: table_grad -> flat_grad, two tiny launches; a flat entry read by several raw entries (a tied parameter) gets
    the sum of their gradients in a fixed order.  One leaf, one AccumulateGrad node, one optimiser tensor."""

    @staticmethod
    def forward(ctx, flat, const_raw, src, kind, off, first_reader, next_reader):
        _require_cuda(flat, const_raw, off)
        flat_in = flat
        flat = flat.contiguous()
        n_links = const_raw.shape[0]
        raw = torch.empty_like(const_raw)
        table = torch.empty((n_links, 28), device=flat.device, dtype=torch.float32)
        with _on(flat.device):
            rc = lib().drmb200_build_link_table_fused(_ptr(const_raw), _ptr(flat), _ptr(src), _ptr(kind), _ptr(off), n_links,
                                                      _ptr(raw), _ptr(table), _stream())
        _check(rc, "drmb200_build_link_table_fused")
        ctx.save_for_backward(flat_in, raw, kind, first_reader, next_reader)
        return table

    @staticmethod
    def backward(ctx, g_table):
        flat_in, raw, kind, first_reader, next_reader = ctx.saved_tensors
        flat = flat_in.contiguous()
        g_table = g_table.contiguous()
        _require_cuda(g_table)
        g_flat = torch.empty_like(flat)
        scratch = torch.empty_like(raw)
        with _on(flat.device):
            rc = lib().drmb200_build_link_table_fused_backward(_ptr(raw), _ptr(g_table), _ptr(flat), _ptr(first_reader),
                                                               _ptr(next_reader), _ptr(kind), raw.shape[0], flat.numel(),
                                                               _ptr(scratch), _ptr(g_flat), _stream())
        _check(rc, "drmb200_build_link_table_fused_backward")
        return first_order_only((g_flat,), (flat_in, g_table)) + (None,) * 6


class FkJacobianFunction(torch.autograd.Function):
    """(table, q) -> (pos, quat, jac_lin, jac_ang); analytic backward kernel (SURVEY.md Appendix B.1)."""

    @staticmethod
    def forward(ctx, table, q, topo, ee_link, want_pos, want_quat, want_jac):
        ctx.save_for_backward(table, q)  # as given, not the contiguous copies: first_order_only links to them
        table, q = table.contiguous(), q.contiguous()
        pos, quat, jlin, jang = fk_jacobian_raw(topo, ee_link, table, q, want_pos, want_quat, want_jac)
        ctx.topo, ctx.ee_link = topo, ee_link
        return pos, quat, jlin, jang           # skipped outputs are None

    @staticmethod
    def backward(ctx, g_pos, g_quat, g_jlin, g_jang):
        saved = ctx.saved_tensors
        table, q = (t.contiguous() for t in saved)
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
        return first_order_only((table_grad, q_grad), saved + (g_pos, g_quat, g_jlin, g_jang)) + (None,) * 5


class FkJacobianMultiFunction(torch.autograd.Function):
    """(table, q) -> stacked (pos, quat, jac_lin, jac_ang) of several links: one tree-walk launch forward; the adjoint is
    the sum of the single-link adjoints, one launch of the FK backward kernel per link with a non-zero upstream gradient
    (q_grad summed, table_grad accumulated in place by the kernel)."""

    @staticmethod
    def forward(ctx, table, q, topo, ee_links, want_pos, want_quat, want_jac):
        ctx.save_for_backward(table, q)  # as given, not the contiguous copies: first_order_only links to them
        table, q = table.contiguous(), q.contiguous()
        outs = fk_jacobian_multi_raw(topo, ee_links, table, q, want_pos, want_quat, want_jac)
        ctx.topo, ctx.ee_links = topo, tuple(ee_links)
        return outs

    @staticmethod
    def backward(ctx, g_pos, g_quat, g_jlin, g_jang):
        saved = ctx.saved_tensors
        table, q = (t.contiguous() for t in saved)
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
        return first_order_only((table_grad, q_grad), saved + (g_pos, g_quat, g_jlin, g_jang)) + (None,) * 5


class AllLinksFkFunction(torch.autograd.Function):
    """(table, q) -> (pos [N, B, 3], quat [N, B, 4]) of EVERY link: one launch of the all-links kernel forward; the adjoint
    is the sum of the single-link adjoints (one FK backward launch per link whose outputs received a gradient)."""

    @staticmethod
    def forward(ctx, table, q, topo):
        ctx.save_for_backward(table, q)  # as given, not the contiguous copies: first_order_only links to them
        table, q = table.contiguous(), q.contiguous()
        poses, quats, _ = kinematic_state_raw(topo, table, q, None, want_poses=True, want_quats=True)
        ctx.topo = topo
        pos = poses[:, 9:12].transpose(1, 2).contiguous()       # [N, B, 3]
        quat = quats.transpose(1, 2).contiguous()               # [N, B, 4]
        return pos, quat

    @staticmethod
    def backward(ctx, g_pos, g_quat):
        saved = ctx.saved_tensors
        table, q = (t.contiguous() for t in saved)
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
        return first_order_only((table_grad, q_grad), saved + (g_pos, g_quat)) + (None,)


class InverseDynamicsFunction(torch.autograd.Function):
    """(table, q, qd, qdd) -> tau; analytic RNEA adjoint kernel (SURVEY.md Appendix B.2)."""

    @staticmethod
    def forward(ctx, table, q, qd, qdd, topo, flags, folded=None):
        ctx.save_for_backward(table, q, qd, qdd)  # as given, not the contiguous copies: first_order_only links to them
        table, q, qd, qdd = table.contiguous(), q.contiguous(), qd.contiguous(), qdd.contiguous()
        tau = inverse_dynamics_raw(topo, table, q, qd, qdd, flags, folded=folded)
        ctx.topo, ctx.flags = topo, flags
        return tau

    @staticmethod
    def backward(ctx, g_tau):
        saved = ctx.saved_tensors
        table, q, qd, qdd = (t.contiguous() for t in saved)
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
        return first_order_only((table_grad, q_grad, qd_grad, qdd_grad), saved + (g_tau,)) + (None,) * 3


class ForwardDynamicsFunction(torch.autograd.Function):
    """(table, q, qd, f) -> qdd; articulated-body kernel forward, analytic adjoint kernel backward.  implicit_dt: implicit
    damping with that step (not differentiated)."""

    @staticmethod
    def forward(ctx, table, q, qd, f, topo, flags, folded=None, implicit_dt=None):
        ctx.save_for_backward(table, q, qd, f)  # as given, not the contiguous copies: first_order_only links to them
        table, q, qd, f = table.contiguous(), q.contiguous(), qd.contiguous(), f.contiguous()
        qdd = forward_dynamics_raw(topo, table, q, qd, f, flags, folded=folded, implicit_dt=implicit_dt)
        ctx.topo, ctx.flags, ctx.implicit_dt = topo, flags, implicit_dt
        return qdd

    @staticmethod
    def backward(ctx, g_qdd):
        saved = ctx.saved_tensors
        table, q, qd, f = (t.contiguous() for t in saved)
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
            if ctx.implicit_dt is not None:
                rc = lib().drmb200_forward_dynamics_implicit_damping_backward(
                    ctypes.byref(ctx.topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B, ctx.flags, ctypes.c_float(ctx.implicit_dt),
                    _ptr(g_qdd), _ptr(q_grad), _ptr(qd_grad), _ptr(f_grad), _ptr(table_grad), _ptr(ws), _stream())
                _check(rc, "drmb200_forward_dynamics_implicit_damping_backward")
            else:
                rc = lib().drmb200_forward_dynamics_backward(
                    ctypes.byref(ctx.topo), _ptr(table), _ptr(q), _ptr(qd), _ptr(f), B, ctx.flags, _ptr(g_qdd), _ptr(q_grad), _ptr(qd_grad),
                    _ptr(f_grad), _ptr(table_grad), _ptr(ws), _stream())
                _check(rc, "drmb200_forward_dynamics_backward")
        return first_order_only((table_grad, q_grad, qd_grad, f_grad), saved + (g_qdd,)) + (None,) * 4


class ForwardDynamicsRolloutFunction(torch.autograd.Function):
    """(table, q0, qd0, f) -> (q, qd, qdd) of a forward-dynamics rollout; one rollout launch forward, the ABA adjoint
    stepped in reverse time backward (drmb200_forward_dynamics_rollout_backward)."""

    @staticmethod
    def forward(ctx, table, q0, qd0, f, topo, flags, dt):
        inputs = (table, q0, qd0, f)  # as given, not the contiguous copies: first_order_only links to them
        table, q0, qd0, f = table.contiguous(), q0.contiguous(), qd0.contiguous(), f.contiguous()
        q, qd, qdd = forward_dynamics_rollout_raw(topo, table, q0, qd0, f, dt, flags)
        ctx.save_for_backward(*inputs, q, qd)
        ctx.topo, ctx.flags, ctx.dt = topo, flags, dt
        return q, qd, qdd

    @staticmethod
    def backward(ctx, g_q, g_qd, g_qdd):
        saved = ctx.saved_tensors
        table, q0, qd0, f = (t.contiguous() for t in saved[:4])
        q, qd = saved[4:]
        need = ctx.needs_input_grad
        T, B, n = f.shape
        g = [None if t is None else t.contiguous() for t in (g_q, g_qd, g_qdd)]
        _require_cuda(*g)
        table_grad = torch.zeros_like(table) if need[0] else None
        alloc = torch.zeros_like if T == 0 else torch.empty_like       # zero steps: the state passes through unchanged
        q0_grad = alloc(q0) if need[1] else None
        qd0_grad = alloc(q0) if need[2] else None
        f_grad = torch.empty_like(f) if need[3] else None
        nbytes = int(lib().drmb200_forward_dynamics_rollout_backward_workspace_bytes(ctypes.byref(ctx.topo), B))
        ws = torch.empty((max(nbytes, 4) + 3) // 4, device=q0.device, dtype=torch.float32)
        with _on(q0.device):
            rc = lib().drmb200_forward_dynamics_rollout_backward(
                ctypes.byref(ctx.topo), _ptr(table), _ptr(q0), _ptr(qd0), _ptr(f), B, T, ctypes.c_float(ctx.dt), ctx.flags,
                _ptr(q), _ptr(qd), _ptr(g[0]), _ptr(g[1]), _ptr(g[2]), _ptr(q0_grad), _ptr(qd0_grad), _ptr(f_grad),
                _ptr(table_grad), _ptr(ws), _stream())
        _check(rc, "drmb200_forward_dynamics_rollout_backward")
        return first_order_only((table_grad, q0_grad, qd0_grad, f_grad), saved[:4] + (g_q, g_qd, g_qdd)) + (None,) * 3


class PDRolloutFunction(torch.autograd.Function):
    """(table, q0, qd0, q_ref, qd_ref, f, kp, kd) -> (q, qd, qdd, tau) of a PD-controlled rollout; one launch forward, the ABA
    adjoint stepped in reverse time with the feedback folded into the element-wise step backward
    (drmb200_pd_rollout_backward).  qd_ref / f may be None; not differentiable in dt or effort_limit.  The kernel returns
    the gains' gradients per row; a shared gain's is their sum over rows, a fixed-order torch reduction."""

    @staticmethod
    def forward(ctx, table, q0, qd0, q_ref, qd_ref, f, kp, kd, topo, flags, dt, effort_limit):
        inputs = (table, q0, qd0, q_ref, qd_ref, f, kp, kd)  # as given: first_order_only links to them
        q, qd, qdd, tau = pd_rollout_raw(topo, table.contiguous(), q0, qd0, q_ref, kp, kd, dt, flags, qd_ref, f, effort_limit)
        ctx.has = tuple(t is not None for t in inputs)
        ctx.save_for_backward(*[t for t in inputs if t is not None], effort_limit, q, qd, tau)
        ctx.topo, ctx.flags, ctx.dt = topo, flags, dt
        return q, qd, qdd, tau

    @staticmethod
    def backward(ctx, g_q, g_qd, g_qdd, g_tau):
        saved = list(ctx.saved_tensors)
        given = [saved.pop(0) if has else None for has in ctx.has]
        effort_limit, q, qd, tau = saved
        table, q0, qd0, q_ref, qd_ref, f, kp, kd = (None if t is None else t.contiguous() for t in given)
        need = ctx.needs_input_grad
        T, B, n = q_ref.shape
        g = [None if t is None else t.contiguous() for t in (g_q, g_qd, g_qdd, g_tau)]
        _require_cuda(*g)
        per_row = kp.ndim == 2
        table_grad = torch.zeros_like(table) if need[0] else None
        alloc = torch.zeros_like if T == 0 else torch.empty_like       # zero steps: nothing reaches the inputs
        q0_grad = alloc(q0) if need[1] else None
        qd0_grad = alloc(q0) if need[2] else None
        q_ref_grad = torch.empty_like(q_ref) if need[3] else None
        qd_ref_grad = torch.empty_like(q_ref) if need[4] else None
        f_grad = torch.empty_like(q_ref) if need[5] else None
        kp_rows = alloc(q0) if need[6] else None                       # [B, n] per row, whichever the gains' shape
        kd_rows = alloc(q0) if need[7] else None
        nbytes = int(lib().drmb200_pd_rollout_backward_workspace_bytes(ctypes.byref(ctx.topo), B))
        ws = torch.empty((max(nbytes, 4) + 3) // 4, device=q0.device, dtype=torch.float32)
        with _on(q0.device):
            rc = lib().drmb200_pd_rollout_backward(
                ctypes.byref(ctx.topo), _ptr(table), _ptr(q0), _ptr(qd0), _ptr(q_ref), _ptr(qd_ref), _ptr(f), _ptr(kp), _ptr(kd),
                1 if per_row else 0, _ptr(effort_limit), B, T, ctypes.c_float(ctx.dt), ctx.flags, _ptr(q), _ptr(qd), _ptr(tau),
                _ptr(g[0]), _ptr(g[1]), _ptr(g[2]), _ptr(g[3]), _ptr(q0_grad), _ptr(qd0_grad), _ptr(q_ref_grad),
                _ptr(qd_ref_grad), _ptr(f_grad), _ptr(kp_rows), _ptr(kd_rows), _ptr(table_grad), _ptr(ws), _stream())
        _check(rc, "drmb200_pd_rollout_backward")
        kp_grad = kp_rows if per_row or kp_rows is None else kp_rows.sum(0)
        kd_grad = kd_rows if per_row or kd_rows is None else kd_rows.sum(0)
        grads = (table_grad, q0_grad, qd0_grad, q_ref_grad, qd_ref_grad, f_grad, kp_grad, kd_grad)
        deps = tuple(t for t in given if t is not None) + (g_q, g_qd, g_qdd, g_tau)
        return first_order_only(grads, deps) + (None,) * 4


class ContactDynamicsFunction(torch.autograd.Function):
    """(table, q, qd, f, accel_ref) -> (qdd, force, solved) of rigid contacts at several links: the single
    drmb200_contact_dynamics launch forward (the same outputs, bit for bit), drmb200_contact_dynamics_backward backward.
    ``solved`` is not differentiable; unsolved rows get zero gradients."""

    @staticmethod
    def forward(ctx, table, q, qd, f, accel_ref, topo, ee_links, flags, position_only, regularization):
        inputs = (table, q, qd, f, accel_ref)  # as given, not the contiguous copies: first_order_only links to them
        qdd, force, solved = contact_dynamics_raw(topo, ee_links, table.contiguous(), q, qd, f, flags, accel_ref,
                                                  position_only, regularization)
        ctx.save_for_backward(*inputs, qdd, force, solved)
        ctx.topo, ctx.ee_links, ctx.flags = topo, tuple(ee_links), flags
        ctx.position_only, ctx.regularization = position_only, regularization
        ctx.mark_non_differentiable(solved)
        return qdd, force, solved

    @staticmethod
    def backward(ctx, g_qdd, g_force, _g_solved):
        saved = ctx.saved_tensors
        table, q, qd, f, accel_ref, qdd, force, solved = saved
        need = ctx.needs_input_grad
        grads = contact_dynamics_backward_raw(ctx.topo, ctx.ee_links, table, q, qd, f, qdd, force, solved, ctx.flags, g_qdd,
                                              g_force, accel_ref, ctx.position_only, ctx.regularization, want_q=need[1],
                                              want_qd=need[2], want_f=need[3], want_accel_ref=need[4], want_table=need[0])
        q_grad, qd_grad, f_grad, ref_grad, table_grad = grads
        return first_order_only((table_grad, q_grad, qd_grad, f_grad, ref_grad),
                                saved[:5] + (g_qdd, g_force)) + (None,) * 5


class ContactImpulseFunction(torch.autograd.Function):
    """(table, q, qd, velocity_ref) -> (qd_plus, impulse, solved) of an impact at several links: the single
    drmb200_contact_impulse launch forward (the same outputs, bit for bit), drmb200_contact_impulse_backward backward.
    ``solved`` is not differentiable; unsolved rows get zero gradients."""

    @staticmethod
    def forward(ctx, table, q, qd, velocity_ref, topo, ee_links, position_only, regularization):
        inputs = (table, q, qd, velocity_ref)  # as given, not the contiguous copies: first_order_only links to them
        qd_plus, impulse, solved = contact_impulse_raw(topo, ee_links, table.contiguous(), q, qd, velocity_ref, position_only,
                                                       regularization)
        ctx.save_for_backward(*inputs, qd_plus, impulse, solved)
        ctx.topo, ctx.ee_links = topo, tuple(ee_links)
        ctx.position_only, ctx.regularization = position_only, regularization
        ctx.mark_non_differentiable(solved)
        return qd_plus, impulse, solved

    @staticmethod
    def backward(ctx, g_qd_plus, g_impulse, _g_solved):
        saved = ctx.saved_tensors
        table, q, qd, velocity_ref, qd_plus, impulse, solved = saved
        need = ctx.needs_input_grad
        q_grad, qd_grad, ref_grad, table_grad = contact_impulse_backward_raw(
            ctx.topo, ctx.ee_links, table, q, qd, qd_plus, impulse, solved, g_qd_plus, g_impulse, velocity_ref,
            ctx.position_only, ctx.regularization, want_q=need[1], want_qd=need[2], want_velocity_ref=need[3],
            want_table=need[0])
        return first_order_only((table_grad, q_grad, qd_grad, ref_grad), saved[:4] + (g_qd_plus, g_impulse)) + (None,) * 4


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
        ctx.save_for_backward(table, q)  # as given, not the contiguous copies: first_order_only links to them
        table, q = table.contiguous(), q.contiguous()
        H = mass_matrix_raw(topo, table, q, folded=folded)
        ctx.topo = topo
        return H

    @staticmethod
    def backward(ctx, g_H):
        saved = ctx.saved_tensors
        table, q = (t.contiguous() for t in saved)
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
        q_grad = q_grad.view(n, B, n).sum(0) if need_q else None
        return first_order_only((table_grad, q_grad), saved + (g_H,)) + (None,) * 2
