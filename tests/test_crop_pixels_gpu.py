"""Every pixel of the crop producer (csrc/fp_crop.cu, the product instantiation crop_tile_kernel<TILE, false, false,
false>, through Engine.make_crops(..., want_dbg=True)) against the vectorised exact reference tests/crop_reference.py,
run on the GPU at 252 hypotheses (tile 80), 5 (tile 32) and 1 (tile 16).  tests/test_crop_reference_cpu.py ties that
reference to oracle/raster.py and oracle/pipeline.py.

Exact, with no allowance: the crop windows, the rendered coverage (a covered pixel has nonzero rendered rgb: every
test texture and vertex colour is >= 1), the winning face (seen through its rendered camera xyz, below), and the fp16
crop buffer (bit-equal to __float2half_rn of the dbg record, zero border and even / odd column layout included).

Bars, per element, derived from the kernel's fp32 roundings (u = 2^-24; each first-order bound doubled):
  * rendered xyz: the kernel's weights w_i = (b_i iz_i) z are three roundings from the exact ones (none on the
    homogeneous path, which is all _rn intrinsics); the 3-term sum two more, fused or not: |dX| <= (3 + 2) u sum |w_i X_i|;
    then (X - t) and * inv_radius one rounding each;
  * rendered rgb: the interpolated uv as xyz, x = u Wt - 0.5 two roundings, the bilinear fetch moves by at most the
    largest colour step of its four texels per texel of coordinate error, plus its own ~12 roundings; the Lambert term
    ~10 roundings per vertex; the shading line 4;
  * observed rgb: the tap weights and the 4-term sum, ~10 roundings; observed xyz: the normalisation's two.
The winning face is exact when the rendered xyz is within its bar and the same comparison REJECTS the second-nearest
covering face on the pixels where two surfaces overlap (a defect probe).  Elements within their bar of a discontinuity
(the z < tau and |o| >= 2 cuts of normalise_xyz, the 0 / 1 clips) are counted and reported, not compared.

Further defect probes, each of which the comparison must reject: a reference that never rasterises the faces of
meshlets 1024 and up (what a crop producer that ran one binning round would give), bilinear taps with border instead
of zero padding on windows that cross the frame edge, and the top-left tie rule mirrored on a grid whose edges pass
through pixel centres.
"""
import os
import time

import numpy as np
import pytest
import torch

import crop_reference as cr

pytestmark = pytest.mark.gpu

S = 160


@pytest.fixture(autouse=True)
def _release_cached_memory():
    yield
    torch.cuda.empty_cache()


def _engine(mt, d, rgb, depth, K, no_cull=False):
    from foundationpose_b200.engine import Engine

    if no_cull:
        os.environ["FPOSE_NO_CULL"] = "1"
    try:
        e = Engine()
    finally:
        os.environ.pop("FPOSE_NO_CULL", None)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt.get("uv"), tex=mt.get("tex"), vertex_colors=mt.get("vcolor"))
    e.set_frame(rgb, depth, K, filter_depth=False)
    return e


def _sphere(pos):
    """The mesh's bounding sphere as fp_set_mesh derives it (fp_meshlet.cu): bounding-box centre, largest distance."""
    p = np.asarray(pos, dtype=np.float32).astype(np.float64)
    c = (p.min(0) + p.max(0)) / 2
    r = np.sqrt(((p - c) ** 2).sum(1)).max()
    return np.float32(c).tolist() + [float(np.float32(r * 1.0001 + 1e-9))]


def _reference(e, mt, d, rgb, K):
    info = e.mesh_info()
    depth, xyz = e.get_depth()
    return cr.Scene(mt, K, rgb, depth, xyz, d, front_sign=info["front_sign"], sphere=_sphere(mt["pos"]), device="cuda")


def _textured(sub, uv_shift=0.0):
    from foundationpose_b200 import synth
    from oracle import pipeline

    mesh = synth.make_mesh(sub)
    mesh.visual.image = np.maximum(mesh.visual.image, 1)  # no zero texel: coverage is visible in the rendered rgb
    mt = pipeline.mesh_tensors(mesh)
    mt["uv"] = mt["uv"] + np.float32(uv_shift)
    return mesh, mt


def _poses_at(rots, t):
    P = np.repeat(np.eye(4, dtype=np.float32)[None], len(rots), 0)
    P[:, :3, :3] = rots
    P[:, :3, 3] = t
    return P


def _edge_translations(K, H, W, z=0.6):
    """Windows across each frame edge and corner, one entirely outside, one larger than the frame, one a few px wide."""
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    x = lambda u: (u - cx) * z / fx
    y = lambda v: (v - cy) * z / fy
    ts = [[x(u), y(v), z] for u, v in ((0, cy), (W, cy), (cx, 0), (cx, H), (0, 0), (W, 0), (0, H), (W, H))]
    ts += [[x(W + 250), y(cy), z], [0.0, 0.0, 0.12], [0.0, 0.0, 25.0]]
    return np.asarray(ts, dtype=np.float32)


def _product_poses(K, H, W, t=(0.02, -0.01, 0.6)):
    from foundationpose_b200 import hypotheses, synth

    grid = hypotheses.make_rotation_grid().astype(np.float32)
    edges = _edge_translations(K, H, W)
    P = np.concatenate([_poses_at(grid[:, :3, :3], t), _poses_at(np.stack([synth.random_rotation(i) for i in range(len(edges))]), 0)])
    P[len(grid):, :3, 3] = edges
    return P, np.arange(len(grid), len(P))


def _compare(e, sc, poses, mode, cull=True, what=""):
    """Runs the kernel and the reference on the same poses and asserts every exact and barred check of the module
    docstring.  Returns (kernel dbg, reference) for the probes."""
    from foundationpose_b200 import packing

    t0 = time.perf_counter()
    crops, dbg, win = e.make_crops(poses, mode=mode, want_dbg=True)
    ref = sc.run(poses, mode, cull=cull, second=True)
    torch.cuda.synchronize()
    N = len(poses)
    # windows
    w = win.cpu().numpy()
    for k, name in enumerate(("left", "top", "sx", "sy")):
        np.testing.assert_array_equal(w[:, k], ref["win"][name], err_msg=f"{what}: window {name}")
    # coverage
    gA, gB = dbg[:, 0].double(), dbg[:, 1].double()
    cov_k = dbg[:, 0, ..., :3].sum(-1) > 0
    cov_r = ref["face"] >= 0
    diff = cov_k != cov_r
    if diff.any():
        n, r, j = [int(v) for v in torch.nonzero(diff)[0]]
        raise AssertionError(f"{what}: coverage differs on {int(diff.sum())} pixels, first at hypothesis {n} pixel "
                             f"(row {r}, col {j}): kernel {bool(cov_k[n, r, j])}, reference face {int(ref['face'][n, r, j])}")
    # rendered and observed values
    ratios = []
    for side, got, want, bar, near in (("rendered", gA, ref["A"], ref["barA"], ref["nearA"]), ("observed", gB, ref["B"], ref["barB"], ref["nearB"])):
        err = torch.where(near, 0.0, (got - want).abs())
        ratio = (err / bar.clamp(min=1e-300)).max().item()  # bar 0 (uncovered pixels): exact zeros required
        ratios.append(ratio)
        bad = err > bar
        if bad.any():
            n, r, j, c = [int(v) for v in torch.nonzero(bad)[0]]
            raise AssertionError(f"{what}: {side} values off on {int(bad.sum())} elements, first at hypothesis {n} (row {r}, "
                                 f"col {j}, channel {c}): kernel {got[n, r, j, c].item():.9g}, reference {want[n, r, j, c].item():.9g}, "
                                 f"bar {bar[n, r, j, c].item():.3g}, face {int(ref['face'][n, r, j])}")
    # the winning face: the second-nearest covering face must be rejected wherever two surfaces overlap, i.e. where it
    # shares no vertex with the winner (two faces folded along a shared edge agree on the points of that edge)
    f1, f2 = sc.faces[ref["face"].clamp(min=0)], sc.faces[ref["face2"].clamp(min=0)]
    shared = (f1[..., :, None] == f2[..., None, :]).any(-1).any(-1)
    over = (ref["face2"] >= 0) & cov_r & ~shared
    rej = ((gA - ref["A2"]).abs() > ref["barA"]).any(-1)
    n_over, n_rej = int(over.sum()), int((rej & over).sum())
    # fp16 buffer: bit-equal to the dbg record rounded to nearest, zero border, even / odd column layout
    canvas = packing.unpad_image_c8(crops)
    inner = canvas[:, 3:163, 3:163, :6]
    want16 = torch.cat([dbg[:, 0], dbg[:, 1]], 0).half()
    assert torch.equal(inner.view(torch.int16), want16.view(torch.int16)), f"{what}: fp16 crop buffer"
    border = canvas.clone()
    border[:, 3:163, 3:163, :6] = 0
    assert not border.view(torch.int16).any(), f"{what}: nonzero border or padding channel"
    n_near = int(ref["nearA"].any(-1).sum() + ref["nearB"].any(-1).sum())
    dt = time.perf_counter() - t0
    print(f"{what} mode {mode}: N={N}, windows / coverage / faces exact over {N * S * S} pixels ({int(cov_r.sum())} covered); "
          f"worst error/bar rendered {ratios[0]:.3f} observed {ratios[1]:.3f}; second-face probe rejected on {n_rej}/{n_over} "
          f"overlap pixels; {n_near} pixels within a bar of a discontinuity; {dt:.1f} s")
    assert n_rej == n_over, f"{what}: the second-nearest face passes the comparison on {n_over - n_rej} overlap pixels"
    assert n_near <= 1e-3 * N * S * S, f"{what}: {n_near} pixels near a discontinuity"
    return dbg, ref


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sub,min_meshlets", [(6, 1024), (7, 4096)])
def test_large_closed_mesh_252(sub, min_meshlets):
    """Textured closed mesh past one (subdivision 6: 81 920 faces) and four (7: 327 680 faces) binning rounds of 1024
    meshlets: the 252-pose rotation grid plus windows across every frame edge, modes 0 and 1, with the product's
    culling and with FPOSE_NO_CULL (every triangle rasterised)."""
    from foundationpose_b200 import synth

    t0 = time.perf_counter()
    mesh, mt = _textured(sub)
    K = synth.DEFAULT_K
    P, edge = _product_poses(K, 480, 640)
    rgb, depth, _ = synth.make_scene(synth.make_texture(1, 512), _poses_at(P[:1, :3, :3], [0.02, -0.01, 0.6])[0].astype(np.float64))
    d = synth.mesh_diameter(mesh.vertices)
    e = _engine(mt, d, rgb, depth, K)
    info = e.mesh_info()
    print(f"subdivision {sub}: {info['F']} faces, {info['meshlets']} meshlets ({-(-info['meshlets'] // 1024)} binning rounds)")
    assert info["meshlets"] > min_meshlets and info["front_sign"] == -1
    sc = _reference(e, mt, d, rgb, K)
    for mode in (0, 1):
        dbg, ref = _compare(e, sc, P, mode, cull=True, what=f"sub {sub} culled")
    # probe: a crop producer that ran one binning round would miss the faces of meshlets 1024 and up
    drop = cr.meshlet_of_face(mt["pos"], mt["faces"]) >= 1024
    probe = sc.run(P, 1, drop_faces=drop)
    share = (probe["face"] != ref["face"]).double().mean().item()
    print(f"sub {sub}: dropping the {int(drop.sum())} faces of meshlets >= 1024 changes the face of {share * 100:.2f}% of pixels")
    assert share > 0.01
    # probe: border padding must fail on every window that crosses the frame edge
    cross = edge[:10]  # the last edge pose is the few-pixel window inside the frame
    tb = sc.run(P[cross], 1, border=True)
    err = (dbg[cross, 1, ..., :3].double() - tb["B"][..., :3]).abs() > tb["barB"][..., :3]
    per_pose = err.flatten(1).double().mean(1)
    print(f"sub {sub}: border padding rejected on {[f'{v * 100:.1f}%' for v in per_pose.tolist()]} of the pixels of the "
          f"windows that cross the frame edge")
    assert (per_pose > 0).all()
    del e, sc
    e2 = _engine(mt, d, rgb, depth, K, no_cull=True)
    assert e2.mesh_info()["front_sign"] == 0
    sc2 = _reference(e2, mt, d, rgb, K)
    _compare(e2, sc2, P, 0, cull=False, what=f"sub {sub} unculled")
    print(f"sub {sub}: {time.perf_counter() - t0:.1f} s")


def _bowl():
    from foundationpose_b200 import synth
    from oracle import pipeline

    mesh = synth.make_mesh(4)
    mesh.visual.image = np.maximum(mesh.visual.image, 1)
    mesh.faces = mesh.faces[mesh.vertices[mesh.faces].mean(1)[:, 2] < 0.04]
    return mesh, pipeline.mesh_tensors(mesh)


def _vcolour():
    from foundationpose_b200 import synth
    from oracle import pipeline

    q, f = synth.icosphere(4)
    rng = np.random.default_rng(4)
    mesh = synth.SimpleMesh(q * synth.RADII, f, q, vertex_colors=rng.integers(1, 256, size=(len(q), 4)).astype(np.uint8))
    return mesh, pipeline.mesh_tensors(mesh)


@pytest.mark.parametrize("case", ["bowl", "near", "uv+3.25", "uv-2.5", "odd_frame", "vcolour"])
@pytest.mark.parametrize("N", [5, 1])
def test_special_paths(case, N):
    """The paths a closed mesh in front of the camera never takes, at 5 hypotheses (tile 32) and 1 (tile 16): an open
    bowl seen through its opening (back faces win), the camera inside the object and 0.5 mm from its surface (the
    homogeneous near-plane path), uv shifted by +3.25 and -2.5 (the general-modulo texture wrap), a 641 x 479 frame with
    its own intrinsics, and a vertex-coloured mesh."""
    from foundationpose_b200 import synth

    K, H, W = synth.DEFAULT_K, 480, 640
    base = np.eye(4)
    base[:3, :3] = synth.random_rotation(3)
    base[:3, 3] = [0.01, 0.0, 0.6]
    rots = np.stack([synth.random_rotation(20 + i) for i in range(N)])
    P = _poses_at(rots, [0.01, 0.0, 0.6])
    if case == "bowl":
        mesh, mt = _bowl()
        P[0, :3, :3] = np.diag([1.0, -1.0, -1.0])  # looking into the bowl
    elif case == "near":
        mesh, mt = _textured(3)
        P[:, :3, 3] = [0.004, -0.003, 0.03]  # camera inside the ellipsoid
        P[0, :3, :3] = np.eye(3)
        P[0, :3, 3] = [0.0, 0.0, 0.0955]  # the surface 0.5 mm in front of the camera crosses the near plane
    elif case.startswith("uv"):
        mesh, mt = _textured(4, uv_shift=float(case[2:]))
    elif case == "odd_frame":
        mesh, mt = _textured(4)
        K, H, W = np.array([[601.0, 0, 321.3], [0, 598.5, 238.9], [0, 0, 1.0]]), 479, 641
        P[1:, :3, 3] = _edge_translations(K, H, W)[: N - 1]
    else:
        mesh, mt = _vcolour()
    rgb, depth, _ = synth.make_scene(synth.make_texture(1, 512), base, K=K, H=H, W=W)
    d = synth.mesh_diameter(mesh.vertices)
    e = _engine(mt, d, rgb, depth, K)
    if case == "near":
        assert e.crop_stats(P)["near_plane_triangles"] > 0
    sc = _reference(e, mt, d, rgb, K)
    for mode in (0, 1):
        dbg, _ = _compare(e, sc, P, mode, cull=True, what=f"{case} N={N}")
        if case == "near":
            # outside the bounding sphere, but the near plane cuts the front faces away: the inside shows through
            assert (dbg[0, 0, ..., :3].sum(-1) > 0).all()


def test_tie_rule_on_pixel_centres():
    """A grid whose every edge passes through pixel centres: the kernel's coverage equals the reference's exactly, and
    the mirrored top-left rule changes it."""
    from foundationpose_b200 import synth

    mt, P, d = cr.tie_grid()
    K = synth.DEFAULT_K
    rgb, depth, _ = synth.make_scene(synth.make_texture(1, 512), P[0].astype(np.float64))
    e = _engine(mt, d, rgb, depth, K)
    sc = _reference(e, mt, d, rgb, K)
    dbg, ref = _compare(e, sc, P, 0, cull=True, what="tie grid")
    flip = sc.run(P, 0, tie_flip=True)
    cov_k = dbg[:, 0, ..., :3].sum(-1) > 0
    n_diff = int((cov_k != (flip["face"] >= 0)).sum())
    print(f"tie grid: the mirrored tie rule changes the coverage of {n_diff} pixels")
    assert n_diff > 0
