"""GPU: parity of the CUDA engine (called through the Python API -> ctypes -> C ABI) with

  * the golden vectors produced by the reference itself (tests/golden/*.npz, every shipped URDF);
  * the fp64 CPU oracle (oracle/drm_oracle.py) on seeded inputs at sizes it finishes in seconds;
  * size-independent properties at BASELINE.json's full batch sizes.

Tolerances: FK / Jacobian  allclose(rtol=1e-5, atol=1e-6) -- the reference's own atol
(tests/test_kinematics_dynamics.py:265-274, 314-323) and north_star's 1e-5 relative;
inverse dynamics atol=1e-5 (tests/test_kinematics_dynamics.py:373-377).
"""
import ctypes

import numpy as np
import pytest
import torch

from conftest import assert_close, canon_quat, load_golden, urdf_path
import differentiable_robot_model_b200 as drm
from differentiable_robot_model_b200 import engine
from oracle import drm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gpu_model(stem):
    return drm.DifferentiableRobotModel(urdf_path(stem), stem, device=DEV)


def cuda(a):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device=DEV)


@pytest.fixture(params=[(1, 0, 0, 1), (0, 0, 0, 1), (1, 1, 64, 1), (1, 0, 256, 0), (1, 0, 0, 2), (0, 0, 64, 2)],
                ids=["tma_bulk_packed", "coop_copy_packed", "unrolled_tile64", "tile256_scalar", "two_configs_per_thread",
                     "two_configs_coop_tile64"])
def fk_variant(request):
    """Every staging / unrolling / tile / packed-arithmetic variant of the FK kernel must give the same parity."""
    variant, unroll, tile, packed = request.param
    engine.set_option("fk_variant", variant)
    engine.set_option("fk_unroll", unroll)
    engine.set_option("fk_tile", tile)
    engine.set_option("fk_packed", packed)
    yield request.param
    engine.set_option("fk_variant", 1)
    engine.set_option("fk_unroll", 2)       # auto
    engine.set_option("fk_tile", 0)
    engine.set_option("fk_packed", 1)


# ------------------------------------------------------------------------------------------------
# golden vectors (reference outputs), every shipped URDF
# ------------------------------------------------------------------------------------------------
def test_fk_jacobian_matches_reference_golden(robot_stem, fk_variant):
    g = load_golden(robot_stem)
    m = gpu_model(robot_stem)
    q = cuda(g["q"])
    m._link_table()                                  # constant model: built once (one launch), then cached
    launches = engine.launch_count()
    for link in g["fk_links"].tolist():
        pos, quat = m.compute_forward_kinematics(q, link)
        jl, ja = m.compute_endeffector_jacobian(q, link)
        fpos, fquat, fjl, fja = m.compute_fk_and_jacobian(q, link)
        assert_close(pos.cpu().numpy(), g[f"pos.{link}"], what=f"pos {link}")
        assert_close(canon_quat(quat.cpu().numpy()), canon_quat(g[f"quat.{link}"]), what=f"quat {link}")
        assert_close(jl.cpu().numpy(), g[f"jlin.{link}"], what=f"jlin {link}")
        assert_close(ja.cpu().numpy(), g[f"jang.{link}"], what=f"jang {link}")
        # the fused op is the same kernel with all outputs enabled: bit-identical
        for a, b in ((pos, fpos), (quat, fquat), (jl, fjl), (ja, fja)):
            assert torch.equal(a, b)
        # raw sign convention of the quaternion (away from branch boundaries)
        same = np.abs(quat.cpu().numpy() - g[f"quat.{link}"]).max(axis=1) < 1e-5
        assert same.mean() >= 0.85
    assert engine.launch_count() - launches == 3 * len(g["fk_links"])


@pytest.fixture(params=[(1, 1, 0), (0, 1, 0), (1, 0, 0), (0, 0, 0), (1, 1, 64), (1, 1, 128), (0, 0, 128)],
                ids=["packed_folded", "scalar_folded", "packed_every_link", "scalar_every_link", "packed_folded_tile64",
                     "packed_folded_tile128", "scalar_every_link_tile128"])
def rnea_variant(request):
    """Both arithmetic variants of the inverse-dynamics kernel, with fixed links folded into their movable ancestors
    (default) and with one step per link like the reference, must give the same parity.  The tile ("rnea_tile") is
    picked by batch size (64 rows below 32 768 configurations); forcing 128 runs the small and ragged batches here with
    the large-batch tile."""
    packed, fold, tile = request.param
    try:
        engine.set_option("rnea_packed", packed)
        engine.set_option("rnea_fold", fold)
        engine.set_option("rnea_tile", tile)
        yield request.param
    finally:
        engine.set_option("rnea_packed", 1)
        engine.set_option("rnea_fold", 1)
        engine.set_option("rnea_tile", 0)


def test_inverse_dynamics_matches_reference_golden(robot_stem, rnea_variant):
    g = load_golden(robot_stem)
    m = gpu_model(robot_stem)
    q, qd, qdd = cuda(g["q"]), cuda(g["qd"]), cuda(g["qdd"])
    for grav in (0, 1):
        for damp in (0, 1):
            tau = m.compute_inverse_dynamics(q, qd, qdd, include_gravity=bool(grav), use_damping=bool(damp))
            assert_close(tau.cpu().numpy(), g[f"tau.g{grav}d{damp}"], rtol=1e-5, atol=1e-5, what=f"tau g{grav}d{damp}")
    nle = m.compute_non_linear_effects(q, qd)
    ref = m.compute_inverse_dynamics(q, qd, torch.zeros_like(q))
    assert torch.equal(nle, ref)


# ------------------------------------------------------------------------------------------------
# fp64 oracle on seeded batches (ragged sizes exercise partial tiles and the non-bulk tail path)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", [1, 3, 255, 256, 257, 1001, 4099])
def test_fk_jacobian_matches_oracle(batch, fk_variant):
    for stem, link in (("iiwa7", "iiwa_link_ee"), ("allegro_hand_description_left", "link_15.0_tip"),
                       ("iiwa7_allegro", "link_3.0_tip")):
        robot = O.load_robot(urdf_path(stem), torch.float64)
        q, _, _ = O.sample_inputs(robot, batch, seed=batch)
        m = gpu_model(stem)
        pos, quat, jl, ja = m.compute_fk_and_jacobian(q.to(DEV), link)
        o_pos, o_quat = O.forward_kinematics(robot, q.double(), link)
        o_jl, o_ja = O.jacobian(robot, q.double(), link)
        assert_close(pos.cpu().numpy(), o_pos.numpy(), what=f"{stem} pos")
        assert_close(canon_quat(quat.cpu().numpy()), canon_quat(o_quat.numpy()), what=f"{stem} quat")
        assert_close(jl.cpu().numpy(), o_jl.numpy(), what=f"{stem} jlin")
        assert_close(ja.cpu().numpy(), o_ja.numpy(), what=f"{stem} jang")


@pytest.mark.parametrize("batch", [1, 5, 127, 128, 129, 1003])
def test_inverse_dynamics_matches_oracle(batch, rnea_variant):
    for stem in ("panda_no_gripper", "iiwa7", "allegro_hand_description_left", "trifinger_edu", "jaco_clean",
                 "iiwa7_allegro"):
        robot = O.load_robot(urdf_path(stem), torch.float64)
        q, qd, qdd = O.sample_inputs(robot, batch, seed=100 + batch)
        m = gpu_model(stem)
        tau = m.compute_inverse_dynamics(q.to(DEV), qd.to(DEV), qdd.to(DEV))
        o_tau = O.inverse_dynamics(robot, q.double(), qd.double(), qdd.double())
        scale = float(o_tau.abs().max())
        assert_close(tau.cpu().numpy(), o_tau.numpy(), rtol=1e-5, atol=max(1e-5, 2e-6 * scale), what=f"{stem} tau")


# ------------------------------------------------------------------------------------------------
# edge cases
# ------------------------------------------------------------------------------------------------
def test_empty_batch_and_1d_inputs(fk_variant):
    m = gpu_model("iiwa7")
    pos, quat, jl, ja = m.compute_fk_and_jacobian(torch.zeros(0, 7, device=DEV), "iiwa_link_ee")
    assert pos.shape == (0, 3) and quat.shape == (0, 4) and jl.shape == (0, 3, 7) and ja.shape == (0, 3, 7)
    tau = m.compute_inverse_dynamics(*(torch.zeros(0, 7, device=DEV),) * 3)
    assert tau.shape == (0, 7)
    # 1-D input -> outputs with the batch dimension removed (robot_model.py:58-62)
    q1 = torch.linspace(-1, 1, 7, device=DEV)
    pos, quat = m.compute_forward_kinematics(q1, "iiwa_link_ee")
    jl, ja = m.compute_endeffector_jacobian(q1, "iiwa_link_ee")
    tau = m.compute_inverse_dynamics(q1, q1, q1)
    assert pos.shape == (3,) and quat.shape == (4,) and jl.shape == (3, 7) and ja.shape == (3, 7) and tau.shape == (7,)
    pos2, _ = m.compute_forward_kinematics(q1[None], "iiwa_link_ee")
    assert torch.equal(pos, pos2[0])
    # zero pose known answer: 0.15+0.19+0.21+0.19+0.21+0.19+0.081+0.045 = 1.266 (SURVEY.md 8c)
    pos0, quat0 = m.compute_forward_kinematics(torch.zeros(7, device=DEV), "iiwa_link_ee")
    assert_close(pos0.cpu().numpy(), [0, 0, 1.266], what="zero pose")
    assert_close(quat0.cpu().numpy(), [0, 0, 0, 1], what="zero quat")


def test_root_link_and_mid_chain_links():
    m = gpu_model("iiwa7")
    q = torch.rand(33, 7, device=DEV)
    pos, quat, jl, ja = m.compute_fk_and_jacobian(q, "iiwa_link_0")         # the root: identity, zero Jacobian
    assert torch.equal(pos, torch.zeros_like(pos)) and torch.equal(jl, torch.zeros_like(jl))
    assert torch.equal(quat, torch.tensor([0.0, 0, 0, 1], device=DEV).expand(33, 4))
    _, _, jl, ja = m.compute_fk_and_jacobian(q, "iiwa_link_3")              # columns 3..6 are off the path
    assert torch.equal(jl[:, :, 3:], torch.zeros_like(jl[:, :, 3:])) and torch.equal(ja[:, :, 3:], torch.zeros_like(ja[:, :, 3:]))
    assert float(ja[:, :, :3].abs().sum()) > 0


def test_unaligned_and_noncontiguous_inputs(fk_variant):
    m = gpu_model("iiwa7")
    base = torch.rand(1030, 7, device=DEV) * 4 - 2
    want = m.compute_fk_and_jacobian(base[1:1025].clone(), "iiwa_link_ee")
    got = m.compute_fk_and_jacobian(base[1:1025], "iiwa_link_ee")          # data_ptr offset 28 B: not 16-B aligned
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    wide = torch.rand(513, 14, device=DEV)
    got = m.compute_fk_and_jacobian(wide[:, ::2], "iiwa_link_ee")           # non-contiguous view
    want = m.compute_fk_and_jacobian(wide[:, ::2].contiguous(), "iiwa_link_ee")
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    t1 = m.compute_inverse_dynamics(base[1:1025], base[2:1026], base[3:1027])
    t2 = m.compute_inverse_dynamics(base[1:1025].clone(), base[2:1026].clone(), base[3:1027].clone())
    assert torch.equal(t1, t2)


def test_large_joint_angles_use_accurate_range_reduction():
    m = gpu_model("iiwa7")
    robot = O.load_robot(urdf_path("iiwa7"), torch.float64)
    q = (torch.rand(512, 7, dtype=torch.float64) * 2 - 1) * 200.0          # far outside the joint limits
    q32 = q.to(torch.float32)
    pos, quat, jl, ja = m.compute_fk_and_jacobian(q32.to(DEV), "iiwa_link_ee")
    o_pos, _ = O.forward_kinematics(robot, q32.double(), "iiwa_link_ee")
    o_jl, o_ja = O.jacobian(robot, q32.double(), "iiwa_link_ee")
    assert_close(pos.cpu().numpy(), o_pos.numpy(), atol=3e-6, what="pos, |q| <= 200 rad")
    assert_close(jl.cpu().numpy(), o_jl.numpy(), atol=3e-6, what="jlin, |q| <= 200 rad")
    huge = torch.full((4, 7), 3.0e6, device=DEV)                            # slow-path (Payne-Hanek) branch
    pos, _ = m.compute_forward_kinematics(huge, "iiwa_link_ee")
    o_pos, _ = O.forward_kinematics(robot, huge.cpu().double(), "iiwa_link_ee")
    assert_close(pos.cpu().numpy(), o_pos.numpy(), atol=3e-6, what="pos, q = 3e6 rad")


def test_device_and_argument_errors():
    m = gpu_model("iiwa7")
    with pytest.raises(AssertionError):                       # CPU tensor into a CUDA model (robot_model.py:38-40)
        m.compute_forward_kinematics(torch.zeros(3, 7), "iiwa_link_ee")
    with pytest.raises(AssertionError):
        m.compute_inverse_dynamics(torch.zeros(3, 7, device=DEV), torch.zeros(3, 6, device=DEV), torch.zeros(3, 7, device=DEV))
    with pytest.raises(KeyError):
        m.compute_endeffector_jacobian(torch.zeros(3, 7, device=DEV), "nope")
    with pytest.raises(RuntimeError, match="fp32-only"):
        m.compute_forward_kinematics(torch.zeros(3, 7, device=DEV, dtype=torch.float64), "iiwa_link_ee")
    # C ABI error codes surface as RuntimeError with the library's message
    with pytest.raises(RuntimeError, match="ee_link"):
        engine.fk_jacobian_raw(m._topology, 77, m._link_table(), torch.zeros(3, 7, device=DEV))


# ------------------------------------------------------------------------------------------------
# size-independent properties at the BASELINE.json batch sizes
# ------------------------------------------------------------------------------------------------
def test_full_size_fk_jacobian_properties():
    """Config 2: Kuka iiwa FK + Jacobian, batch 65 536."""
    m = gpu_model("iiwa7")
    robot = O.load_robot(urdf_path("iiwa7"), torch.float64)
    B = 65536
    q, _, _ = O.sample_inputs(robot, B, seed=7)
    q = q.to(DEV)
    pos, quat, jl, ja = m.compute_fk_and_jacobian(q, "iiwa_link_ee")
    assert torch.isfinite(pos).all() and torch.isfinite(jl).all()
    # unit quaternions, unit joint axes
    assert float((quat.norm(dim=1) - 1).abs().max()) < 2e-6
    assert float((ja.norm(dim=1) - 1).abs().max()) < 2e-6
    # 2 pi periodicity of every revolute joint
    pos2, quat2, jl2, ja2 = m.compute_fk_and_jacobian(q + 2 * np.pi, "iiwa_link_ee")
    assert float((pos - pos2).abs().max()) < 5e-6 and float((jl - jl2).abs().max()) < 5e-6
    # tiling independence: any sub-batch gives bit-identical rows (a checksum of checksums)
    idx = torch.randperm(B, device=DEV)[:10007]
    sub = m.compute_fk_and_jacobian(q[idx], "iiwa_link_ee")
    for full, part in zip((pos, quat, jl, ja), sub):
        assert torch.equal(full[idx], part)
    # the linear Jacobian is the derivative of the position: central differences along a random direction
    d = torch.randn(B, 7, device=DEV)
    h = 1e-3
    pp, _ = m.compute_forward_kinematics(q + h * d, "iiwa_link_ee")
    pm, _ = m.compute_forward_kinematics(q - h * d, "iiwa_link_ee")
    fd = (pp - pm) / (2 * h)
    an = torch.einsum("bij,bj->bi", jl, d)
    assert float((fd - an).abs().max()) < 2e-3 * float(an.abs().max())
    # spot-check 2048 rows against the fp64 oracle
    rows = idx[:2048].cpu()
    o_pos, o_quat = O.forward_kinematics(robot, q.cpu().double()[rows], "iiwa_link_ee")
    o_jl, o_ja = O.jacobian(robot, q.cpu().double()[rows], "iiwa_link_ee")
    assert_close(pos.cpu().numpy()[rows], o_pos.numpy(), what="pos")
    assert_close(canon_quat(quat.cpu().numpy()[rows]), canon_quat(o_quat.numpy()), what="quat")
    assert_close(jl.cpu().numpy()[rows], o_jl.numpy(), what="jlin")
    assert_close(ja.cpu().numpy()[rows], o_ja.numpy(), what="jang")


def test_full_size_inverse_dynamics_properties():
    """Config 3: Franka Panda RNEA, batch 65 536."""
    m = gpu_model("panda_no_gripper")
    robot = O.load_robot(urdf_path("panda_no_gripper"), torch.float64)
    B = 65536
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, B, seed=11))
    tau = m.compute_inverse_dynamics(q, qd, qdd)
    assert torch.isfinite(tau).all()
    # tau is affine in qdd: tau(a) + tau(b) - tau(0) == tau(a + b)
    a, b = torch.randn_like(qdd), torch.randn_like(qdd)
    t = lambda x: m.compute_inverse_dynamics(q, qd, x)  # noqa: E731
    lhs, rhs = t(a) + t(b) - t(torch.zeros_like(a)), t(a + b)
    assert float((lhs - rhs).abs().max()) < 2e-4 * max(1.0, float(rhs.abs().max()))
    # damping enters as damping * qd; gravity term is velocity independent
    d_on = m.compute_inverse_dynamics(q, qd, qdd, use_damping=True)
    d_off = m.compute_inverse_dynamics(q, qd, qdd, use_damping=False)
    damp = torch.stack([b_.get_joint_damping_const().reshape(()) for b_ in (m._bodies[i] for i in m._controlled_joints)])
    assert float((d_on - d_off - damp * qd).abs().max()) < 1e-5
    # the mass matrix extracted column by column is symmetric positive definite
    z = torch.zeros_like(q[:4096])
    g_ = m.compute_inverse_dynamics(q[:4096], z, z)
    cols = []
    for j in range(7):
        e = z.clone(); e[:, j] = 1.0
        cols.append(m.compute_inverse_dynamics(q[:4096], z, e) - g_)
    H = torch.stack(cols, dim=2)
    assert float((H - H.transpose(1, 2)).abs().max()) < 1e-4
    assert float(torch.linalg.eigvalsh(H.double().cpu()).min()) > 0
    # tiling independence + oracle spot check
    idx = torch.randperm(B, device=DEV)[:5003]
    assert torch.equal(tau[idx], m.compute_inverse_dynamics(q[idx], qd[idx], qdd[idx]))
    rows = idx[:1024].cpu()
    o_tau = O.inverse_dynamics(robot, q.cpu().double()[rows], qd.cpu().double()[rows], qdd.cpu().double()[rows])
    assert_close(tau.cpu().numpy()[rows], o_tau.numpy(), rtol=1e-5, atol=max(1e-5, 2e-6 * float(o_tau.abs().max())), what="tau")


@pytest.mark.parametrize("mode", ["fused_pinned", "staged_pinned", "pageable"])
def test_host_buffer_entry_point_matches_device_path(mode):
    """Page-locked buffers: one launch whose TMA copies read / write host memory directly (default) or the staged
    H2D -> kernel -> D2H pipeline; pageable buffers always take the staged pipeline.  All bit-identical to the device path."""
    m = gpu_model("iiwa7")
    B = 150001                                               # several pipeline chunks + a ragged tail
    pin = (lambda t: t.pin_memory()) if mode != "pageable" else (lambda t: t)
    q_host = pin(torch.rand(B, 7) * 4 - 2)
    outs = [pin(torch.zeros(B, 3)), pin(torch.zeros(B, 4)), pin(torch.zeros(B, 3, 7)), pin(torch.zeros(B, 3, 7))]
    engine.set_option("host_fused", 0 if mode == "staged_pinned" else 1)
    table = m._link_table()
    try:
        launches = engine.launch_count()
        engine.fk_jacobian_host(m._topology, m._name_to_idx_map["iiwa_link_ee"], 0, table, q_host, *outs)
        if mode == "fused_pinned":
            assert engine.launch_count() - launches == 1
    finally:
        engine.set_option("host_fused", 1)
    want = m.compute_fk_and_jacobian(q_host.to(DEV), "iiwa_link_ee")
    for got, w in zip(outs, want):
        assert torch.equal(got, w.cpu())


# ------------------------------------------------------------------------------------------------
# programmatic dependent launch (fk_pdl = 2): launches overlap their predecessors; results must not change
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def pdl_mode():
    engine.set_option("fk_pdl", 2)
    yield
    engine.set_option("fk_pdl", 0)


def _fk_reference_runs(m, ee, qs):
    engine.set_option("fk_pdl", 0)
    want = [[t.clone() for t in engine.fk_jacobian_raw(m._topology, ee, m._link_table(), q)] for q in qs]
    torch.cuda.synchronize()
    return want


@pytest.mark.parametrize("batch", [65536, 40000, 4099])
def test_pdl_chain_of_independent_batches_is_bit_identical(batch, pdl_mode):
    """A stream of back-to-back FK launches over rotating buffers, eagerly and replayed from a CUDA graph, with the
    launches overlapping (batch >= ~30 k takes the PDL path, smaller ones fall back): outputs == ordinary launches."""
    m = gpu_model("iiwa7")
    ee = m._name_to_idx_map["iiwa_link_ee"]
    robot = O.load_robot(urdf_path("iiwa7"), torch.float32)
    qs = [O.sample_inputs(robot, batch, seed=40 + i)[0].to(DEV) for i in range(6)]
    want = _fk_reference_runs(m, ee, qs)
    engine.set_option("fk_pdl", 2)
    table = m._link_table()
    outs = [tuple(torch.zeros_like(t) for t in w) for w in want]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for rep in range(3):
            for i, q in enumerate(qs):
                engine.fk_jacobian_raw(m._topology, ee, table, q, out=outs[i])
        stream.synchronize()
        for w, o in zip(want, outs):
            for a, b in zip(w, o):
                assert torch.equal(a, b)
                b.zero_()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            for rep in range(4):
                for i, q in enumerate(qs):
                    engine.fk_jacobian_raw(m._topology, ee, table, q, out=outs[i])
        for _ in range(3):
            g.replay()
        stream.synchronize()
    for w, o in zip(want, outs):
        for a, b in zip(w, o):
            assert torch.equal(a, b)


def test_pdl_falls_back_when_a_launch_reads_its_predecessors_output(pdl_mode):
    """Launch k+1 takes the J_lin block that launch k is still writing as its q: stream order must hold."""
    m = gpu_model("iiwa7")
    ee = m._name_to_idx_map["iiwa_link_ee"]
    robot = O.load_robot(urdf_path("iiwa7"), torch.float32)
    B = 65536
    q0 = O.sample_inputs(robot, B, seed=77)[0].to(DEV)
    table = m._link_table()

    def chain():
        cur, res = q0, []
        for _ in range(4):
            pos, quat, jl, ja = engine.fk_jacobian_raw(m._topology, ee, table, cur)
            res.append((pos, quat, jl, ja))
            cur = jl.view(3 * B, 7)[:B]                 # the first B rows of the block just written, as joint angles
        torch.cuda.synchronize()
        return res

    engine.set_option("fk_pdl", 0)
    want = chain()
    engine.set_option("fk_pdl", 2)
    for _ in range(3):
        got = chain()
        for w, g_ in zip(want, got):
            for a, b in zip(w, g_):
                assert torch.equal(a, b)


def test_default_constructed_model_computes():
    """The reference's default-constructed model computes (on its default device, robot_model.py:100-104); here the
    default device is the current CUDA device."""
    m = drm.DifferentiableKUKAiiwa()
    assert m._device.type == "cuda"
    g = load_golden("iiwa7")
    pos, quat = m.compute_forward_kinematics(cuda(g["q"]), "iiwa_link_ee")
    assert_close(pos.cpu().numpy(), g["pos.iiwa_link_ee"], what="pos")


# ------------------------------------------------------------------------------------------------
# 1024-row reference batches, raw quaternion sign on all four branches of get_quaternion
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stem", ["large_iiwa7", "large_panda_no_gripper", "large_allegro_left"])
def test_large_reference_batches_with_raw_quaternion_sign(stem, fk_variant):
    from conftest import LARGE_GOLDEN, quat_branch_margin
    g = load_golden(stem)
    m = gpu_model(LARGE_GOLDEN[stem])
    q, qd, qdd = cuda(g["q"]), cuda(g["qd"]), cuda(g["qdd"])
    for link in g["links"].tolist():
        pos, quat, jl, ja = m.compute_fk_and_jacobian(q, link)
        assert_close(pos.cpu().numpy(), g[f"pos.{link}"], what=f"{stem} pos {link}")
        assert_close(jl.cpu().numpy(), g[f"jlin.{link}"], what=f"{stem} jlin {link}")
        assert_close(ja.cpu().numpy(), g[f"jang.{link}"], what=f"{stem} jang {link}")
        # the RAW quaternion (sign included) wherever the rotation is clear of a branch boundary of
        # spatial_vector_algebra.py:118-128; the remaining rows up to sign
        clear = quat_branch_margin(g[f"R.{link}"]) > 1e-3
        assert_close(quat.cpu().numpy()[clear], g[f"quat.{link}"][clear], atol=2e-6, what=f"{stem} raw quat {link}")
        assert_close(canon_quat(quat.cpu().numpy()), canon_quat(g[f"quat.{link}"]), atol=2e-6, what=f"{stem} quat {link}")
    if stem != "large_allegro_left":
        branch = g["branch"]
        clear = quat_branch_margin(g[f"R.{g['links'][0]}"]) > 1e-3
        assert min(int((clear & (branch == b)).sum()) for b in range(4)) >= 40      # each branch asserted with raw sign
    tau = m.compute_inverse_dynamics(q, qd, qdd)
    assert_close(tau.cpu().numpy(), g["tau"], atol=1e-5, what=f"{stem} tau")


def test_folded_inverse_dynamics_follows_learnable_parameters_of_fixed_links():
    """Folding recomputes the composite bodies from the CURRENT table on every launch: learnable inertial parameters of a
    link behind a fixed joint (iiwa_link_ee) and learnable origins of movable links change tau exactly as without folding."""
    from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar, UnconstrainedTensor
    robot = O.load_robot(urdf_path("iiwa7"), torch.float32)
    q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, 777, seed=5))
    m = gpu_model("iiwa7")
    m.make_link_param_learnable("iiwa_link_ee", "mass", UnconstrainedScalar(init_val=torch.tensor([2.5])))
    m.make_link_param_learnable("iiwa_link_ee", "com", UnconstrainedTensor(1, 3, init_tensor=torch.tensor([[0.05, -0.02, 0.1]])))
    m.make_link_param_learnable("iiwa_link_ee", "inertia_mat", UnconstrainedTensor(3, 3, init_tensor=torch.tensor([[0.02, 0.003, -0.001], [0.001, 0.03, 0.002], [0.004, -0.002, 0.01]])))
    m.make_link_param_learnable("iiwa_link_6", "trans", UnconstrainedTensor(1, 3, init_tensor=torch.tensor([[0.01, 0.05, 0.2]])))
    with torch.no_grad():
        engine.set_option("rnea_fold", 0)
        want = m.compute_inverse_dynamics(q, qd, qdd)
        engine.set_option("rnea_fold", 1)
        got = m.compute_inverse_dynamics(q, qd, qdd)
    scale = float(want.abs().max())
    assert_close(got.cpu().numpy() / scale, want.cpu().numpy() / scale, rtol=1e-5, atol=2e-6, what="tau folded vs every link")
    base = gpu_model("iiwa7").compute_inverse_dynamics(q, qd, qdd)
    assert float((got - base).abs().max()) > 1e-2 * scale          # the fixed link's parameters do matter


@pytest.mark.parametrize("stem", ["iiwa7", "panda", "allegro_hand_description_left", "iiwa7_allegro", "trifinger_edu", "jaco"])
def test_folding_fixed_links_does_not_change_mass_matrix_or_forward_dynamics(stem):
    """The mass-matrix and articulated-body kernels walk only the movable links too ("rnea_fold"); one step per link
    (the reference's loop) must give the same numbers up to rounding."""
    robot = O.load_robot(urdf_path(stem), torch.float32)
    q, qd, _ = (t.to(DEV) for t in O.sample_inputs(robot, 300, seed=8))
    f = torch.randn(300, q.shape[1], generator=torch.Generator().manual_seed(1)).to(DEV)
    m = gpu_model(stem)
    out = {}
    for fold in (0, 1):
        engine.set_option("rnea_fold", fold)
        with torch.no_grad():
            out[fold] = (m.compute_lagrangian_inertia_matrix(q), m.compute_forward_dynamics(q, qd, f, use_damping=True))
    engine.set_option("rnea_fold", 1)
    for a, b, what in zip(out[1], out[0], ("H", "qdd")):
        scale = float(b.abs().max())
        assert_close(a.cpu().numpy() / scale, b.cpu().numpy() / scale, rtol=2e-5, atol=5e-6, what=f"{stem} {what} folded vs every link")


@pytest.mark.parametrize("stem", ["iiwa7", "panda_no_gripper", "allegro_hand_description_left", "iiwa7_allegro", "jaco"])
def test_prefolded_table_gives_the_same_torques_bit_for_bit(stem):
    """A constant model folds its table ONCE (drmb200_fold_link_table) and launches drmb200_inverse_dynamics_prefolded; the
    kernel then copies the rows instead of folding them per CTA: same arithmetic, same bits."""
    m = gpu_model(stem)
    robot = O.load_robot(urdf_path(stem), torch.float32)
    for batch in (37, 4099, 40000):
        q, qd, qdd = (t.to(DEV) for t in O.sample_inputs(robot, batch, seed=batch))
        folded = engine.fold_link_table(m._topology, m._link_table())
        assert folded is not None and folded.shape[1] == 28
        a = engine.inverse_dynamics_raw(m._topology, m._link_table(), q, qd, qdd, 3)
        b = engine.inverse_dynamics_raw(m._topology, m._link_table(), q, qd, qdd, 3, folded=folded)
        assert torch.equal(a, b)
        assert torch.equal(m.compute_inverse_dynamics(q, qd, qdd), a)          # the model takes the prefolded path by itself
    launches = engine.launch_count()
    m.compute_inverse_dynamics(q, qd, qdd)
    assert engine.launch_count() - launches == 1                               # folded once, not per call
