"""GPU parity of the fused crop producer (csrc/fp_crop.cu) and the depth filters (csrc/fp_depth.cu)
against the CPU oracle (oracle/geometry.py, raster.py, pipeline.py).

Bars:
  * crop window (integer-valued edges): bit-exact;
  * raster coverage / triangle choice: the oracle uses the same fixed-point rule, so rendered-crop
    validity masks must agree on >= 99.9 % of pixels (a vertex whose projection differs in the last
    fp32 bit may flip a 1/256-px snap);
  * values on agreeing pixels: 2e-4 abs (fp32 interpolation order differs), rgb 2e-3;
  * observed crop (nearest/bilinear resampling): >= 99.8 % of pixels within tolerance (nearest-neighbour
    ties at x.5 are decided by the last bit of kornia's coordinate chain);
  * depth filters: 1e-6 abs.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from oracle import pipeline

    mesh = synth.make_mesh(3)
    pose = np.eye(4)
    pose[:3, :3] = synth.random_rotation(0)
    pose[:3, 3] = [0.02, -0.01, 0.6]
    rgb, depth, mask = synth.make_scene(mesh.visual.image, pose)
    d = synth.mesh_diameter(mesh.vertices)
    mt = pipeline.mesh_tensors(mesh)
    e = Engine()
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt["uv"], tex=mt["tex"])
    poses = np.stack([pose, pose, pose, pose]).astype(np.float32)
    poses[1, :3, 3] += [0.01, 0.0, 0.02]
    poses[2, :3, :3] = synth.random_rotation(7)
    poses[3, :3, 3] = [0.25, 0.18, 0.5]  # partially outside the frame
    return dict(e=e, mesh=mesh, mt=mt, rgb=rgb, depth=depth, K=synth.DEFAULT_K, d=d, poses=poses)


def _compare(got, ref, what, min_agree, atol):
    got, ref = got.float().cpu(), ref.float().cpu()
    ok = (got - ref).abs() <= atol
    frac = ok.float().mean().item()
    assert frac >= min_agree, f"{what}: only {frac * 100:.3f}% of values within {atol}"


@pytest.mark.parametrize("mode", [0, 1])
def test_crops_match_oracle(scene, mode):
    from oracle import geometry, pipeline

    e = scene["e"]
    e.set_frame(scene["rgb"], scene["depth"], scene["K"], filter_depth=False)
    _, dbg, win = e.make_crops(scene["poses"], mode=mode, want_dbg=True)
    xyz = geometry.depth2xyzmap(scene["depth"], scene["K"])
    A, B, owin = pipeline.make_crops(scene["poses"], scene["mt"], scene["rgb"], scene["depth"], xyz, scene["K"], scene["d"], mode)
    w = win.cpu().numpy()
    np.testing.assert_array_equal(w[:, 0], owin["left"])
    np.testing.assert_array_equal(w[:, 1], owin["top"])
    np.testing.assert_array_equal(w[:, 2], owin["sx"])
    np.testing.assert_array_equal(w[:, 3], owin["sy"])
    gA = dbg[:, 0].permute(0, 3, 1, 2)  # (N,6,160,160)
    gB = dbg[:, 1].permute(0, 3, 1, 2)
    # coverage of the rendered crop
    cov_g = (gA[:, 3:].abs().sum(1) > 0).cpu()
    cov_o = A[:, 3:].abs().sum(1) > 0
    agree = (cov_g == cov_o).float().mean().item()
    assert agree >= 0.999, f"raster coverage agreement {agree}"
    both = (cov_g & cov_o)[:, None].expand(-1, 3, -1, -1)
    assert ((gA[:, 3:].cpu() - A[:, 3:]).abs()[both] <= 2e-4).float().mean().item() >= 0.9995
    assert ((gA[:, :3].cpu() - A[:, :3]).abs()[both] <= 2e-3).float().mean().item() >= 0.999
    _compare(gB[:, :3], B[:, :3], "observed rgb", 0.998, 2e-3)
    _compare(gB[:, 3:], B[:, 3:], "observed xyz", 0.998, 2e-4)


def test_fp16_crop_buffer_layout(scene):
    """The fp16 buffer the stem convolution reads: [2N][166 rows][even | odd columns][84 pairs][8]; interior =
    crops, border = zeros."""
    from foundationpose_b200 import packing

    e = scene["e"]
    e.set_frame(scene["rgb"], scene["depth"], scene["K"], filter_depth=False)
    crops, dbg, _ = e.make_crops(scene["poses"], mode=0, want_dbg=True)
    N = len(scene["poses"])
    assert crops.shape == (2 * N, 166, 2, 84, 8)
    canvas = packing.unpad_image_c8(crops)
    inner = canvas[:, 3:163, 3:163, :6].float()
    ref = torch.cat([dbg[:, 0], dbg[:, 1]], 0)
    assert (inner - ref).abs().max().item() <= 2e-3
    assert canvas[:, :3].abs().max().item() == 0 and canvas[:, 163:].abs().max().item() == 0
    assert canvas[:, :, :3].abs().max().item() == 0 and canvas[:, :, 163:].abs().max().item() == 0
    assert canvas[..., 6:].abs().max().item() == 0


def test_depth_filters(scene):
    from foundationpose_b200.engine import op_depth_filter
    from oracle import geometry

    depth = scene["depth"].copy()
    rng = np.random.default_rng(3)
    depth[rng.random(depth.shape) < 0.05] = 0  # holes
    depth[100:110, 200:260] += 0.05  # a step
    dg = torch.from_numpy(depth).cuda()
    er = op_depth_filter(dg, 0)
    ref_er = geometry.erode_depth(depth)
    np.testing.assert_allclose(er.cpu().numpy(), ref_er, atol=1e-6, rtol=0)
    bl = op_depth_filter(er, 1)
    ref_bl = geometry.bilateral_filter_depth(ref_er)
    np.testing.assert_allclose(bl.cpu().numpy(), ref_bl, atol=2e-6, rtol=0)


def test_set_frame_filters_and_xyz(scene):
    from oracle import geometry

    e = scene["e"]
    e.set_frame(scene["rgb"], scene["depth"], scene["K"], filter_depth=True)
    d, xyz = e.get_depth()
    ref = geometry.bilateral_filter_depth(geometry.erode_depth(scene["depth"]))
    np.testing.assert_allclose(d.cpu().numpy(), ref, atol=2e-6, rtol=0)
    np.testing.assert_allclose(xyz.cpu().numpy(), geometry.depth2xyzmap(ref, scene["K"]), atol=1e-6, rtol=0)


def test_pose_update(scene):
    from oracle import geometry

    g = torch.Generator().manual_seed(2)
    poses = torch.from_numpy(scene["poses"]).clone()
    trans = torch.randn(4, 3, generator=g) * 0.3
    rot = torch.randn(4, 3, generator=g)
    rot[0] = 0  # exercises the eps clamp of so3_exp_map
    # slot 0 holds the scene's mesh (diameter d); the context keeps the default rot_normalizer
    out, _, _ = scene["e"].op_pose_update(poses.cuda(), trans.cuda(), rot.cuda())
    ref, _, _ = geometry.pose_update(poses, trans, rot, scene["d"], 0.3490658503988659)
    np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), atol=2e-6, rtol=0)


def test_start_poses_match_host_guess_translation(scene):
    """Device-side guess_translation (exact masked median via radix select) vs the host restatement of
    estimater.py:137-156, odd and even valid counts, empty mask, no valid depth."""
    from foundationpose_b200 import hypotheses, synth

    e = scene["e"]
    e.set_frame(scene["rgb"], scene["depth"], scene["K"], filter_depth=True)
    depth_f = e.get_depth()[0].cpu().numpy()
    grid = torch.from_numpy(hypotheses.make_rotation_grid()).cuda()
    _, _, mask = synth.make_scene(scene["mesh"].visual.image, scene["poses"][0].astype(np.float64))
    masks = [mask.copy(), mask.copy(), np.zeros_like(mask), mask.copy()]
    vs, us = np.where(masks[1])
    masks[1][vs[0], us[0]] = False  # flips the parity of the valid count
    depths_zero = [False, False, False, True]
    for m, dz in zip(masks, depths_zero):
        if dz:
            e.set_frame(scene["rgb"], np.zeros_like(scene["depth"]), scene["K"], filter_depth=True)
            dref = np.zeros_like(depth_f)
        else:
            e.set_frame(scene["rgb"], scene["depth"], scene["K"], filter_depth=True)
            dref = depth_f
        poses, info = e.start_poses(m, grid)
        ref_t = hypotheses.guess_translation(dref, m, scene["K"])
        info = info.cpu().numpy()
        np.testing.assert_allclose(info[:3], ref_t, atol=1e-6, rtol=0)
        assert int(info[3]) == int((m & (dref >= 0.001)).sum())
        p = poses.cpu().numpy()
        np.testing.assert_array_equal(p[:, :3, :3], grid.cpu().numpy()[:, :3, :3])
        np.testing.assert_allclose(p[:, :3, 3], np.tile(ref_t.astype(np.float32), (252, 1)), atol=1e-6, rtol=0)


def test_other_frame_size_and_intrinsics():
    """The path is not specialised to 640x480: a 1280x720 frame with its own intrinsics, crops vs the oracle."""
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from oracle import geometry, pipeline

    mesh = synth.make_mesh(2)
    K = np.array([[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1.0]])
    pose = np.eye(4)
    pose[:3, :3] = synth.random_rotation(4)
    pose[:3, 3] = [-0.15, 0.08, 0.7]
    rgb, depth, mask = synth.make_scene(mesh.visual.image, pose, K=K, H=720, W=1280)
    d = synth.mesh_diameter(mesh.vertices)
    mt = pipeline.mesh_tensors(mesh)
    e = Engine()
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt["uv"], tex=mt["tex"])
    e.set_frame(rgb, depth, K, filter_depth=False)
    poses = np.stack([pose, pose]).astype(np.float32)
    poses[1, :3, 3] = [0.62, 0.3, 0.72]  # crop window partly outside the frame
    xyz = geometry.depth2xyzmap(depth, K)
    for mode in (0, 1):
        _, dbg, win = e.make_crops(poses, mode=mode, want_dbg=True)
        A, B, owin = pipeline.make_crops(poses, mt, rgb, depth, xyz, K, d, mode)
        np.testing.assert_array_equal(win.cpu().numpy()[:, 0], owin["left"])
        np.testing.assert_array_equal(win.cpu().numpy()[:, 3], owin["sy"])
        gA = dbg[:, 0].permute(0, 3, 1, 2)
        gB = dbg[:, 1].permute(0, 3, 1, 2)
        _compare(gA[:, 3:], A[:, 3:], "rendered xyz", 0.999, 2e-4)
        _compare(gA[:, :3], A[:, :3], "rendered rgb", 0.998, 2e-3)
        _compare(gB[:, :3], B[:, :3], "observed rgb", 0.998, 2e-3)
        _compare(gB[:, 3:], B[:, 3:], "observed xyz", 0.998, 2e-4)


@pytest.mark.parametrize("n", [1, 3, 5, 66])
def test_batch_size_does_not_change_a_hypothesis(scene, n):
    """Crops of hypothesis 0 are bit-identical whatever else is in the batch (tile size 16 / 32 / 80 is chosen from the
    batch size; the A/B image boundary is padded to a multiple of four)."""
    e = scene["e"]
    e.set_frame(scene["rgb"], scene["depth"], scene["K"], filter_depth=False)
    base = scene["poses"][[0, 1, 2]]
    poses = np.concatenate([base] * ((n + 2) // 3))[:n].astype(np.float32)
    crops, _, _ = e.make_crops(poses, mode=0)
    ref, _, _ = e.make_crops(poses[:1], mode=0)
    assert torch.equal(crops[0], ref[0]) and torch.equal(crops[n], ref[1])
    if n == 0:
        return
    empty, _, _ = e.make_crops(poses[:0], mode=0)
    assert empty.shape[0] == 0
