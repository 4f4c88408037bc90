"""Synthetic inputs of the benchmark / tests (SURVEY.md §8d): a textured ellipsoid mesh, a 640x480
RGB-D frame of it in front of a textured plane, and seeded weights (weights.random_state_dict).

Everything is numpy on the host and deterministic for a given seed; no file IO, no network.
The frame is produced analytically (ray / ellipsoid intersection), not by any renderer, so it does
not depend on the code under test.
"""
import numpy as np


class _Visual:
    def __init__(self, uv, image):
        self.uv = uv
        self.image = image  # uint8 (Ht, Wt, 3)
        self.vertex_colors = None


class SimpleMesh:
    """Minimal stand-in for the trimesh.Trimesh attributes the hot path reads
    (Utils.py:104-130: vertices, faces, vertex_normals, visual.uv, visual.material.image)."""

    def __init__(self, vertices, faces, vertex_normals, uv=None, texture=None, vertex_colors=None):
        self.vertices = np.asarray(vertices, dtype=np.float64)
        self.faces = np.asarray(faces, dtype=np.int64)
        self.vertex_normals = np.asarray(vertex_normals, dtype=np.float64)
        self.visual = _Visual(uv, texture)
        self.visual.vertex_colors = vertex_colors

    def copy(self):
        return SimpleMesh(self.vertices.copy(), self.faces.copy(), self.vertex_normals.copy(),
                          None if self.visual.uv is None else self.visual.uv.copy(), self.visual.image,
                          self.visual.vertex_colors)


def icosphere(subdivisions):
    """Unit icosphere: V = 10 * 4^s + 2 vertices, F = 20 * 4^s faces."""
    t = (1.0 + 5.0 ** 0.5) / 2.0
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
                  [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int64)
    verts = [tuple(x) for x in v]
    for _ in range(subdivisions):
        cache = {}
        new_f = []

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = (np.array(verts[a]) + np.array(verts[b])) / 2.0
                m /= np.linalg.norm(m)
                verts.append(tuple(m))
                cache[key] = len(verts) - 1
            return cache[key]

        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            new_f += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = np.array(new_f, dtype=np.int64)
    return np.array(verts, dtype=np.float64), f


RADII = np.array([0.05, 0.03, 0.095])  # 0.10 x 0.06 x 0.19 m, roughly a mustard bottle


def sphere_uv(q):
    """Spherical UV of unit directions q (..., 3) -> (..., 2) in [0, 1]."""
    u = np.arctan2(q[..., 1], q[..., 0]) / (2 * np.pi) + 0.5
    v = np.arccos(np.clip(q[..., 2], -1, 1)) / np.pi
    return np.stack([u, v], -1)


def make_texture(seed=0, size=1024, block=16):
    rng = np.random.default_rng(seed)
    low = rng.integers(0, 256, size=(size // block, size // block, 3), dtype=np.uint8)
    return np.ascontiguousarray(np.repeat(np.repeat(low, block, 0), block, 1))


def make_mesh(subdivisions=5, tex_seed=0, tex_size=1024, scale=1.0):
    """Textured icosphere ellipsoid of radii RADII * scale (the object make_multi_scene draws at that scale)."""
    q, f = icosphere(subdivisions)
    radii = RADII * scale
    verts = q * radii
    nrm = q / radii
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    uv = sphere_uv(q)
    return SimpleMesh(verts, f, nrm, uv=uv, texture=make_texture(tex_seed, tex_size))


def vertex_coloured(mesh):
    """The same object with its texture sampled at the vertices: uint8 vertex colours instead of uv + texture."""
    tex = mesh.visual.image
    Ht, Wt = tex.shape[:2]
    tx = np.clip((mesh.visual.uv[:, 0] * Wt).astype(np.int64), 0, Wt - 1)
    ty = np.clip(((1.0 - mesh.visual.uv[:, 1]) * Ht).astype(np.int64), 0, Ht - 1)
    return SimpleMesh(mesh.vertices, mesh.faces, mesh.vertex_normals, vertex_colors=tex[ty, tx])


def mesh_diameter(vertices):
    """Largest pairwise vertex distance (Utils.py:559-574), exact: see meshprep.mesh_diameter."""
    from .meshprep import mesh_diameter as _exact

    return _exact(vertices)


DEFAULT_K = np.array([[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1.0]])


def random_rotation(seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def make_scene(mesh_texture, pose, K=DEFAULT_K, H=480, W=640, plane_z=1.2, seed=1, depth_noise=0.001):
    """Analytic RGB-D frame: ellipsoid (radii RADII, texture via spherical UV) at `pose` (4x4 ob_in_cam)
    in front of a textured plane at z = plane_z.  Returns rgb uint8 (H,W,3), depth float32 (H,W), mask bool."""
    rgb, depth, owner = make_multi_scene([(mesh_texture, pose, 1.0)], K, H, W, plane_z, seed, depth_noise)
    return rgb, depth, owner == 0


def make_multi_scene(objects, K=DEFAULT_K, H=480, W=640, plane_z=1.2, seed=1, depth_noise=0.001):
    """Analytic RGB-D frame of several ellipsoids in front of the textured plane of make_scene.  objects: sequence of
    (texture, pose, scale): an ellipsoid of radii RADII * scale (make_mesh(scale=scale)) at `pose` (4x4 ob_in_cam),
    coloured from `texture` via spherical UV.  On every pixel ray the nearest positive hit wins, so objects occlude
    each other.  Returns rgb uint8 (H,W,3), depth float32 (H,W) and the index of the object seen at each pixel (-1 =
    the plane)."""
    rng = np.random.default_rng(seed)
    vs, us = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    d = np.stack([(us - K[0, 2]) / K[0, 0], (vs - K[1, 2]) / K[1, 1], np.ones_like(us, dtype=np.float64)], -1)
    depth = np.full((H, W), plane_z, dtype=np.float64)
    bg = make_texture(seed + 100, 512, 32)
    bu = ((d[..., 0] * plane_z * 400).astype(np.int64)) % 512
    bv = ((d[..., 1] * plane_z * 400).astype(np.int64)) % 512
    rgb = bg[bv, bu].copy()
    owner = np.full((H, W), -1, dtype=np.int64)
    nearest = np.full((H, W), np.inf)
    for k, (texture, pose, scale) in enumerate(objects):
        radii = RADII * scale
        R, t = pose[:3, :3], pose[:3, 3]
        o_ob = -R.T @ t
        d_ob = d @ R  # rows: R^T d
        so, sd = o_ob / radii, d_ob / radii
        a = (sd * sd).sum(-1)
        b = 2 * (sd * so).sum(-1)
        c = (so * so).sum() - 1.0
        disc = b * b - 4 * a * c
        hit = disc > 0
        s = np.where(hit, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0)
        hit &= (s > 0) & (s < nearest)
        depth[hit] = s[hit]
        nearest[hit] = s[hit]
        owner[hit] = k
        p_ob = o_ob + d_ob * s[..., None]
        uv = sphere_uv(p_ob / radii / np.maximum(np.linalg.norm(p_ob / radii, axis=-1, keepdims=True), 1e-9))
        Ht, Wt = texture.shape[:2]
        tx = np.clip((uv[..., 0] * Wt).astype(np.int64), 0, Wt - 1)
        ty = np.clip(((1.0 - uv[..., 1]) * Ht).astype(np.int64), 0, Ht - 1)  # trimesh uv: v = 0 is the image bottom
        rgb[hit] = texture[ty, tx][hit]
    depth = depth + rng.normal(0, depth_noise, size=depth.shape)
    return rgb.astype(np.uint8), depth.astype(np.float32), owner


def default_scene(subdivisions=5, seed=0):
    """Mesh, GT pose, K and frame of BASELINE.json configs[1] ("model-based register")."""
    mesh = make_mesh(subdivisions)
    pose = np.eye(4)
    pose[:3, :3] = random_rotation(seed)
    pose[:3, 3] = [0.0, 0.0, 0.6]
    rgb, depth, mask = make_scene(mesh.visual.image, pose)
    return mesh, pose, DEFAULT_K.copy(), rgb, depth, mask


def track_sequence(n_frames, pose0, seed=3, max_trans=0.005, max_rot_deg=2.0):
    """Ground-truth poses of a synthetic tracking sequence (SURVEY.md §8d, C3): the object moves by at most
    `max_trans` metres and `max_rot_deg` degrees per frame (a smooth random walk, rng(seed))."""
    rng = np.random.default_rng(seed)
    poses = [np.asarray(pose0, dtype=np.float64).copy()]
    vel_t = rng.normal(size=3)
    vel_r = rng.normal(size=3)
    for _ in range(1, n_frames):
        vel_t = 0.9 * vel_t + 0.4 * rng.normal(size=3)
        vel_r = 0.9 * vel_r + 0.4 * rng.normal(size=3)
        dt = vel_t / max(np.linalg.norm(vel_t), 1e-9) * max_trans * min(1.0, np.linalg.norm(vel_t) / 2.0)
        ang = np.deg2rad(max_rot_deg) * min(1.0, np.linalg.norm(vel_r) / 2.0)
        ax = vel_r / max(np.linalg.norm(vel_r), 1e-9)
        Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
        dR = np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * (Kx @ Kx)
        p = poses[-1].copy()
        p[:3, :3] = dR @ p[:3, :3]
        p[:3, 3] = p[:3, 3] + dt * np.array([1.0, 1.0, 0.5])
        poses.append(p)
    return np.stack(poses)


def write_obj(mesh, path):
    """Wavefront OBJ + MTL + PNG texture of a SimpleMesh (uv in the trimesh convention: v = 0 at the image bottom)."""
    import os

    import cv2

    stem = os.path.splitext(os.path.basename(path))[0]
    d = os.path.dirname(path)
    os.makedirs(d, exist_ok=True)
    with open(path, "w") as fh:
        fh.write(f"mtllib {stem}.mtl\nusemtl material_0\n")
        for p in mesh.vertices:
            fh.write(f"v {p[0]:.9g} {p[1]:.9g} {p[2]:.9g}\n")
        for n in mesh.vertex_normals:
            fh.write(f"vn {n[0]:.9g} {n[1]:.9g} {n[2]:.9g}\n")
        for t in mesh.visual.uv:
            fh.write(f"vt {t[0]:.9g} {t[1]:.9g}\n")
        for f in mesh.faces + 1:
            fh.write("f " + " ".join(f"{i}/{i}/{i}" for i in f) + "\n")
    with open(os.path.join(d, stem + ".mtl"), "w") as fh:
        fh.write(f"newmtl material_0\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nmap_Kd {stem}.png\n")
    cv2.imwrite(os.path.join(d, stem + ".png"), mesh.visual.image[..., ::-1])


def write_demo_scene(root, n_frames=5, subdivisions=3, seed=0):
    """A scene directory in the layout of the reference's demo data (run_demo.py:18-19, datareader.py:57-152):
    mesh/textured_simple.obj (+ .mtl + .png), cam_K.txt, rgb/*.png, depth/*.png (uint16 millimetres), masks/*.png and
    annotated_poses/*.txt (ground truth).  Returns (mesh, gt_poses)."""
    import os

    import cv2

    mesh = make_mesh(subdivisions)
    pose0 = np.eye(4)
    pose0[:3, :3] = random_rotation(seed)
    pose0[:3, 3] = [0.02, -0.01, 0.6]
    poses = track_sequence(n_frames, pose0)
    write_obj(mesh, os.path.join(root, "mesh", "textured_simple.obj"))
    for sub in ("rgb", "depth", "masks", "annotated_poses"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    np.savetxt(os.path.join(root, "cam_K.txt"), DEFAULT_K)
    for i, p in enumerate(poses):
        rgb, depth, mask = make_scene(mesh.visual.image, p, seed=1 + i)
        name = f"{i:06d}"
        cv2.imwrite(os.path.join(root, "rgb", name + ".png"), rgb[..., ::-1])
        cv2.imwrite(os.path.join(root, "depth", name + ".png"), np.clip(np.rint(depth * 1000.0), 0, 65535).astype(np.uint16))
        if i == 0:
            cv2.imwrite(os.path.join(root, "masks", name + ".png"), mask.astype(np.uint8) * 255)
        np.savetxt(os.path.join(root, "annotated_poses", name + ".txt"), p)
    return mesh, poses


def _write_bop_scene(scene_dir, ob_id, poses, tex, seed):
    """One BOP scene directory with ONE annotated object per frame (datareader.py:155-181 layout)."""
    import json
    import os

    import cv2

    for sub in ("rgb", "depth", "mask_visib", "mask"):
        os.makedirs(os.path.join(scene_dir, sub), exist_ok=True)
    cam, gt = {}, {}
    for i, p in enumerate(poses):
        rgb, depth, mask = make_scene(tex, p, seed=seed + i)
        name = f"{i:06d}"
        cv2.imwrite(os.path.join(scene_dir, "rgb", name + ".png"), rgb[..., ::-1])
        cv2.imwrite(os.path.join(scene_dir, "depth", name + ".png"), np.clip(np.rint(depth * 1000.0), 0, 65535).astype(np.uint16))
        for sub in ("mask_visib", "mask"):
            cv2.imwrite(os.path.join(scene_dir, sub, f"{name}_000000.png"), mask.astype(np.uint8) * 255)
        cam[str(i)] = {"cam_K": DEFAULT_K.reshape(-1).tolist(), "depth_scale": 1.0}
        gt[str(i)] = [{"cam_R_m2c": p[:3, :3].reshape(-1).tolist(), "cam_t_m2c": (p[:3, 3] * 1000.0).tolist(), "obj_id": int(ob_id)}]
    with open(os.path.join(scene_dir, "scene_camera.json"), "w") as fh:
        json.dump(cam, fh)
    with open(os.path.join(scene_dir, "scene_gt.json"), "w") as fh:
        json.dump(gt, fh)


def _write_bop_models(models_dir, ob_ids, subdivisions, symmetric=()):
    """obj_<id>.ply (vertex-coloured ellipsoid, MILLIMETRES) + models_info.json; returns {ob_id: texture image}."""
    import json
    import os
    import sys

    os.makedirs(models_dir, exist_ok=True)
    fb = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin", "_fallback")
    try:
        import trimesh
    except ImportError:
        sys.path.append(fb)
        import trimesh
    info, texs = {}, {}
    for ob_id in ob_ids:
        m = make_mesh(subdivisions, tex_seed=int(ob_id), tex_size=256)
        tex = m.visual.image
        Ht, Wt = tex.shape[:2]
        tx = np.clip((m.visual.uv[:, 0] * Wt).astype(np.int64), 0, Wt - 1)
        ty = np.clip(((1.0 - m.visual.uv[:, 1]) * Ht).astype(np.int64), 0, Ht - 1)
        tm = trimesh.Trimesh(m.vertices * 1000.0, m.faces, vertex_normals=m.vertex_normals)
        tm.visual = trimesh.visual.ColorVisuals(vertex_colors=tex[ty, tx])
        tm.export(os.path.join(models_dir, f"obj_{int(ob_id):06d}.ply"))
        lo, hi = (m.vertices * 1000.0).min(0), (m.vertices * 1000.0).max(0)
        e = {"diameter": float(mesh_diameter(m.vertices) * 1000.0), "min_x": float(lo[0]), "min_y": float(lo[1]), "min_z": float(lo[2]),
             "size_x": float(hi[0] - lo[0]), "size_y": float(hi[1] - lo[1]), "size_z": float(hi[2] - lo[2])}
        if ob_id in symmetric:
            e["symmetries_discrete"] = [np.diag([-1.0, -1.0, 1.0, 1.0]).reshape(-1).tolist()]  # half turn about z
        info[str(int(ob_id))] = e
        texs[ob_id] = tex
    with open(os.path.join(models_dir, "models_info.json"), "w") as fh:
        json.dump(info, fh)
    return texs


def write_bop_dataset(root, kind="lm", n_frames=1, subdivisions=2, seed=0, scene_objects=None, symmetric=(6,)):
    """A synthetic dataset in the directory conventions of the reference's dataset drivers:

    kind = "lm"   (run_linemod.py:90-112, datareader.py:400-430): <root>/lm_test_all/test/<ob_id:06d>/ — one scene per
                  object, for the 13 evaluated LINEMOD ids — and <root>/lm_models/models/;
    kind = "ycbv" (run_ycb_video.py:85-118, datareader.py:433-531): <root>/test/<scene:06d>/ for `scene_objects`
                  ({scene id: object id}), <root>/ycbv_models/models/ for all 21 ids, <root>/models/<21 names>/ and
                  <root>/keyframe.txt.

    Every frame shows ONE textured ellipsoid (all objects share the geometry, not the colours).  Returns
    {(scene id, frame id string, object id): ground-truth 4x4 pose}."""
    import os

    gts = {}
    if kind == "lm":
        ob_ids = [i for i in range(1, 16) if i not in (3, 7)]
        texs = _write_bop_models(os.path.join(root, "lm_models", "models"), ob_ids, subdivisions, symmetric)
        scenes = {ob_id: ob_id for ob_id in ob_ids}
        scene_root = os.path.join(root, "lm_test_all", "test")
    elif kind == "ycbv":
        ob_ids = list(range(1, 22))
        texs = _write_bop_models(os.path.join(root, "ycbv_models", "models"), ob_ids, subdivisions, symmetric)
        scenes = dict(scene_objects or {48: 1, 49: 6, 50: 13})
        scene_root = os.path.join(root, "test")
        for i in ob_ids:
            os.makedirs(os.path.join(root, "models", f"{i:03d}_synthetic_object"), exist_ok=True)
    else:
        raise ValueError(kind)
    key_lines = []
    for scene_id, ob_id in scenes.items():
        pose0 = np.eye(4)
        pose0[:3, :3] = random_rotation(seed + 7 * scene_id)
        pose0[:3, 3] = [0.03 * ((scene_id % 3) - 1), -0.02 * ((scene_id % 2)), 0.55 + 0.01 * (scene_id % 5)]
        poses = track_sequence(n_frames, pose0, seed=seed + scene_id)
        _write_bop_scene(os.path.join(scene_root, f"{scene_id:06d}"), ob_id, poses, texs[ob_id], seed=10 * scene_id + 1)
        for i, p in enumerate(poses):
            gts[(scene_id, f"{i:06d}", ob_id)] = p
            key_lines.append(f"{scene_id:04d}/{i:06d}")
    if kind == "ycbv":
        with open(os.path.join(root, "keyframe.txt"), "w") as fh:
            fh.write("\n".join(key_lines) + "\n")
    return gts
