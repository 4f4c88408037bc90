"""CPU: the vectorised crop reference (tests/crop_reference.py) against the reviewed oracle, so that the GPU pixel tests
(tests/test_crop_pixels_gpu.py) rest on code that is itself tied to oracle/raster.py and oracle/pipeline.py.

With culling off, the reference's winning face and its fp32 barycentrics must equal oracle/raster.rasterize's tri_id
and bary bit for bit (a closed mesh, an open bowl, a near-plane pose, a vertex-coloured mesh); its windows must equal
geometry.crop_window; its values must equal pipeline.make_crops within the fp32-vs-float64 bars it states.
"""
import numpy as np
import pytest
import torch

import crop_reference as cr


def _poses(rot_seeds, t):
    from foundationpose_b200 import synth

    out = []
    for s in rot_seeds:
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(s)
        p[:3, 3] = t
        out.append(p)
    return np.stack(out).astype(np.float32)


def _case(name):
    from foundationpose_b200 import synth

    if name == "closed":
        mesh = synth.make_mesh(2)
        poses = _poses([0, 7], [0.02, -0.01, 0.6])
        poses[1, :3, 3] = [0.25, 0.18, 0.5]  # window partly outside the frame
    elif name == "bowl":
        mesh = synth.make_mesh(3)
        mesh.faces = mesh.faces[mesh.vertices[mesh.faces].mean(1)[:, 2] < 0.04]
        poses = _poses([5], [0.0, 0.0, 0.55])
        poses[0, :3, :3] = np.diag([1.0, -1.0, -1.0])
    elif name == "near":
        mesh = synth.make_mesh(2)
        poses = _poses([9, 9], [0.004, -0.003, 0.03])  # camera inside the ellipsoid
        poses[1, :3, :3] = np.eye(3)
        poses[1, :3, 3] = [0.0, 0.0, 0.0955]  # the surface 0.5 mm in front of the camera: it crosses the near plane
    else:
        q, f = synth.icosphere(2)
        rng = np.random.default_rng(4)
        mesh = synth.SimpleMesh(q * synth.RADII, f, q, vertex_colors=rng.integers(1, 256, size=(len(q), 4)).astype(np.uint8))
        poses = _poses([3], [0.01, 0.0, 0.6])
    return mesh, poses


@pytest.mark.parametrize("name", ["closed", "bowl", "near", "vcolor"])
def test_reference_matches_the_oracle(name):
    from foundationpose_b200 import synth
    from oracle import geometry, pipeline, raster

    mesh, poses = _case(name)
    mt = pipeline.mesh_tensors(mesh)
    K = synth.DEFAULT_K
    rgb, depth, _ = synth.make_scene(synth.make_texture(0, 256), poses[0].astype(np.float64))
    xyz = geometry.depth2xyzmap(depth, K)
    d = synth.mesh_diameter(mesh.vertices)
    sc = cr.Scene(mt, K, rgb, depth, xyz, d)
    for mode in (0, 1):
        ref = sc.run(poses, mode, cull=False)
        owin, _ = geometry.crop_window(poses, K, d)
        for k in ("left", "top", "sx", "sy"):
            np.testing.assert_array_equal(ref["win"][k], owin[k])
        umin, vmin, umax, vmax = geometry.render_window(owin)
        for n in range(len(poses)):
            tri, bary, _, persp = raster.rasterize(poses[n], mt["pos"], mt["faces"], K, (umin[n], vmin[n], umax[n], vmax[n]))
            np.testing.assert_array_equal(ref["face"][n].numpy(), tri)
            cov = tri >= 0
            assert cov.any()
            np.testing.assert_array_equal(ref["bary"][n].numpy()[cov].view(np.uint32), bary[cov].view(np.uint32))
            if name == "near" and n == 1:
                assert persp.any(), "the near-plane case must reach the homogeneous path"
        A, B, _ = pipeline.make_crops(poses, mt, rgb, depth, xyz, K, d, mode)
        for what, got, want, bar, near in (("A", ref["A"], A, ref["barA"], ref["nearA"]), ("B", ref["B"], B, ref["barB"], ref["nearB"])):
            want = want.permute(0, 2, 3, 1).double()
            # the oracle is fp32 throughout: allow its own roundings on top of the reference's bar.  Its observed rgb
            # samples at coordinates from kornia's op sequence (a 3x3 inverse and matrix products), which differ from
            # the kernel's closed form by up to ~1e-4 px; a colour changes by at most 1 per pixel.
            err = (got - want).abs()
            tol = bar + 4e-6 * want.abs().clamp(min=1.0)
            if what == "B":
                tol[..., :3] += 2e-4
                # nearest samples of coordinates within 1e-3 px of x.5: kornia's chain decides them by its last bits
                # (see geometry.unwarp_nearest), the kernel as exact arithmetic does
                tb = sc.taps(sc._win_t(ref["win"]), tie_tol=1e-3)
                tie = tb["row"]["tie"][:, :, None] | tb["col"]["tie"][:, None, :]
                near = near | tie[..., None]
            bad = (err > tol) & ~near
            assert not bad.any(), f"{name} mode {mode} {what}: {int(bad.sum())} values off, worst {err[bad].max():.3g}"


def test_tie_rule_grid_snaps_to_pixel_centres():
    """The grid built by the GPU test's tie case: every vertex lands exactly on a pixel centre, so the edges of the
    grid pass through pixel centres and the tie rule decides them; the mirrored rule changes the coverage."""
    from foundationpose_b200 import synth
    from oracle import geometry, raster

    mt, poses, d = cr.tie_grid()
    K = synth.DEFAULT_K
    rgb, depth, _ = synth.make_scene(synth.make_texture(0, 256), poses[0].astype(np.float64))
    sc = cr.Scene(mt, K, rgb, depth, geometry.depth2xyzmap(depth, K), d)
    X, Y, Z, iz, xi, yi = sc.project(torch.from_numpy(poses), sc._win_t(cr.windows(poses, K, d)))
    assert ((xi % 256) == 128).all() and ((yi % 256) == 128).all()

    ref = sc.run(poses, 0, cull=False)
    flip = sc.run(poses, 0, cull=False, tie_flip=True)
    assert ((ref["face"] >= 0) != (flip["face"] >= 0)).sum() > 0
    owin, _ = geometry.crop_window(poses, K, d)
    umin, vmin, umax, vmax = geometry.render_window(owin)
    tri, _, _, _ = raster.rasterize(poses[0], mt["pos"], mt["faces"], K, (umin[0], vmin[0], umax[0], vmax[0]))
    np.testing.assert_array_equal(ref["face"][0].numpy(), tri)


def test_meshlet_of_face_partitions_the_mesh():
    """The face-to-meshlet map the GPU test's one-binning-round probe uses: every face in exactly one meshlet, meshlets
    in binning order hold contiguous runs of fp_op_build_meshlets' face list, and subdivision 6 needs two rounds."""
    from foundationpose_b200 import synth

    v, f = synth.icosphere(6)
    m = cr.meshlet_of_face(v * synth.RADII, f)
    counts = np.bincount(m)
    assert len(counts) > 1024 and counts.min() >= 1 and counts.max() <= 64 and counts.sum() == len(f)
