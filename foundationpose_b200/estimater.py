"""Host-side mirror of the reference's estimator and predictor surfaces, running on libfpose.so.

Same names, argument orders and error behaviour as
  estimater.py:18-268                              FoundationPose {register, track_one, reset_object, ...}
  learning/training/predict_pose_refine.py:92-239  PoseRefinePredictor {predict, last_trans_update, ...}
  learning/training/predict_score.py:117-226       ScorePredictor {predict}
so a driver written against the reference (run_demo.py:38-63) only changes its import.

Differences that are deliberate (DESIGN.md §1): no nvdiffrast context is needed (`glctx` is accepted
and ignored).  Visualisation is what the reference's drivers reach: `predict(get_vis=True)` returns the reference's
canvases (composed on the device by fp_vis, labelled on the host, foundationpose_b200/vis.py), register() at debug >= 2
writes color.png, depth.png, ob_mask.png, vis_refiner.png, vis_score.png (and the .ply clouds when open3d imports)
to debug_dir, and track_one() at debug >= 2 puts the refiner canvas in extra['vis'].  `predict()` honours the
per-call `mesh` / `mesh_tensors` / `mesh_diameter` / `xyz_map` arguments of the reference: a mesh that is not
the one already in the context is uploaded first, a caller-supplied xyz map replaces the derived one.
"""
import logging
import os
import weakref

import numpy as np
import torch

from . import hypotheses, meshprep, synth, weights
from .engine import MAX_CAMERAS, MAX_MESHES, Engine


class _Cfg(dict):
    __getattr__ = dict.__getitem__

    def __setattr__(self, k, v):
        self[k] = v


class _ModelHandle:
    """Stands in for the `.model` attribute the reference estimator moves between devices
    (estimater.py:97-100); the packed weights live inside the fp_ctx."""

    def to(self, *a, **k):
        return self

    def cuda(self):
        return self

    def eval(self):
        return self


_shared_engine = None


def get_engine():
    """One fp_ctx per process/device, shared by the scorer and the refiner (they share mesh + frame)."""
    global _shared_engine
    if _shared_engine is None:
        _shared_engine = Engine()
    return _shared_engine


def _load_cfg_and_weights(run_name, kind, state_dict, cfg):
    """Config + weights the way the reference predictors find them (predict_pose_refine.py:96-131,
    predict_score.py:120-143): weights/<run>/config.yml next to model_best.pth, then the reference's
    backward-compatibility defaults for missing keys.  Without a checkpoint tree (this repository ships none)
    the released-config values of weights.DEFAULT_CFG and the seeded stand-in weights are used."""
    path = weights.find_reference_weights(run_name) if state_dict is None else None
    if path is not None:
        c = _Cfg(weights.load_reference_config(os.path.join(os.path.dirname(path), "config.yml"), kind))
        state_dict = weights.load_checkpoint(path)
        logging.info(f"Using pretrained model from {path}")
    else:
        c = _Cfg(weights.DEFAULT_CFG)
        if state_dict is None:
            logging.info(f"weights/{run_name}/model_best.pth not found: using the seeded synthetic {kind} weights")
            state_dict = weights.random_state_dict(kind, seed=0)
    if cfg:
        unknown = set(cfg) - set(weights.DEFAULT_CFG) - {"ckpt_dir", "enable_amp", "use_mask", "n_view", "normal_uint8"}
        if unknown:
            raise ValueError(f"unsupported config keys for the {kind} predictor: {sorted(unknown)}")
        c.update(cfg)
    if not c["normalize_xyz"] or c["rot_rep"] != "axis_angle" or c["trans_rep"] != "tracknet" or c["use_normal"]:
        raise NotImplementedError("engine supports the released configs: normalize_xyz, tracknet, axis_angle, no normals")
    if list(c["input_resize"]) != [160, 160] or int(c["c_in"]) != 6:
        raise NotImplementedError("engine supports input_resize = [160, 160] and c_in = 6 (the released configs)")
    return c, state_dict


def _mesh_arrays(mesh_tensors):
    """Accepts this package's make_mesh_tensors() dict or the reference's (Utils.py:104-130: torch tensors under
    'pos', 'faces', 'vnormals', 'uv', 'tex' [1,H,W,3 float 0..1] or 'vertex_color')."""
    g = lambda k: mesh_tensors.get(k)
    to_np = lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    out = dict(pos=to_np(g("pos")), faces=to_np(g("faces")), normals=to_np(g("normals") if g("normals") is not None else g("vnormals")))
    if g("uv") is not None and g("tex") is not None:
        tex = to_np(g("tex"))
        if tex.ndim == 4:
            tex = tex[0]
        if tex.dtype != np.uint8:  # the reference keeps the texture as float 0..1
            tex = np.clip(np.rint(tex * 255.0), 0, 255).astype(np.uint8)
        out["uv"], out["tex"] = to_np(g("uv")), tex
    else:
        vc = g("vcolor") if g("vcolor") is not None else g("vertex_color")
        out["vcolor"] = to_np(vc)
    return out


def _sync_mesh(engine, mesh, mesh_tensors, mesh_diameter):
    """predict()'s per-call mesh arguments (predict_pose_refine.py:171-172, predict_score.py:176-177): upload the
    mesh unless it is the one the context already holds."""
    src = mesh_tensors if mesh_tensors is not None else mesh
    if src is None:
        if engine.diameter is None:
            raise ValueError("predict(): no mesh in the context and none passed (mesh / mesh_tensors)")
        return
    d = float(mesh_diameter) if mesh_diameter is not None else engine.diameter
    if getattr(engine, "_mesh_src", None) is src and (d is None or d == engine.diameter):
        return
    mt = _mesh_arrays(mesh_tensors) if mesh_tensors is not None else make_mesh_tensors(mesh)
    if d is None:
        d = synth.mesh_diameter(mt["pos"])
    engine.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt.get("uv"), tex=mt.get("tex"), vertex_colors=mt.get("vcolor"))
    engine._mesh_src = src


class PoseRefinePredictor:
    def __init__(self, engine=None, state_dict=None, cfg=None):
        self.amp = True
        self.run_name = "2023-10-28-18-33-37"
        self.engine = engine or get_engine()
        self.cfg, sd = _load_cfg_and_weights(self.run_name, "refine", state_dict, cfg)
        self.engine.load_network("refine", sd)
        self.engine.set_config("refine", self.cfg["crop_ratio"], self.cfg["rot_normalizer"])
        self.model = _ModelHandle()
        self.dataset = None
        self.last_trans_update = None
        self.last_rot_update = None

    @torch.inference_mode()
    def predict(self, rgb, depth, K, ob_in_cams, xyz_map=None, normal_map=None, get_vis=False, mesh=None, mesh_tensors=None,
                glctx=None, mesh_diameter=None, iteration=5, _frame_ready=False):
        """@rgb: (H,W,3) uint8; @ob_in_cams: (N,4,4).  Returns ((N,4,4) cuda tensor, canvas): canvas is None, or with
        get_vis the reference's (N*166+6, 1314, 3) uint8 image of every hypothesis's crops before and after refinement."""
        e = self.engine
        _sync_mesh(e, mesh, mesh_tensors, mesh_diameter)
        if not _frame_ready:
            e.set_frame(rgb, depth, K, filter_depth=False, zfar=float("inf"))
            if xyz_map is not None:
                e.set_xyz_map(xyz_map)
        poses, lt, lr = e.refine(ob_in_cams, iteration)
        self.last_trans_update = lt
        self.last_rot_update = lr
        if not get_vis:
            return poses, None
        from . import vis  # cv2: only the debug canvases need it

        return poses, vis.refine_canvas(e, ob_in_cams, poses)


class ScorePredictor:
    def __init__(self, amp=True, engine=None, state_dict=None, cfg=None):
        self.amp = amp
        self.run_name = "2024-01-11-20-02-45"
        self.engine = engine or get_engine()
        self.cfg, sd = _load_cfg_and_weights(self.run_name, "score", state_dict, cfg)
        self.engine.load_network("score", sd)
        self.engine.set_config("score", self.cfg["crop_ratio"])
        self.model = _ModelHandle()
        self.dataset = None

    @torch.inference_mode()
    def predict(self, rgb, depth, K, ob_in_cams, normal_map=None, get_vis=False, mesh=None, mesh_tensors=None, glctx=None,
                mesh_diameter=None, _frame_ready=False):
        """Returns ((N,) cuda tensor of scores = logits + 100, canvas): canvas is None, or with get_vis the reference's
        (N*105, 409, 3) uint8 image of every hypothesis's crops, ranked by descending score."""
        e = self.engine
        _sync_mesh(e, mesh, mesh_tensors, mesh_diameter)
        if not _frame_ready:
            e.set_frame(rgb, depth, K, filter_depth=False)
        scores, _ = e.score(ob_in_cams)
        if not get_vis:
            return scores, None
        from . import vis  # cv2: only the debug canvases need it

        return scores, vis.score_canvas(e, ob_in_cams, scores)


def make_mesh_tensors(mesh):
    """Utils.py:104-130 on a trimesh-like object -> host arrays for fp_set_mesh."""
    out = dict(pos=np.asarray(mesh.vertices, dtype=np.float32), faces=np.asarray(mesh.faces, dtype=np.int32),
               normals=np.asarray(mesh.vertex_normals, dtype=np.float32))
    uv = getattr(mesh.visual, "uv", None)
    img = getattr(mesh.visual, "image", None)
    if img is None and getattr(mesh.visual, "material", None) is not None:
        img = np.asarray(mesh.visual.material.image.convert("RGB"))
    if uv is not None and img is not None:
        uv = np.asarray(uv, dtype=np.float32).copy()
        uv[:, 1] = 1 - uv[:, 1]
        out["uv"] = uv
        out["tex"] = np.ascontiguousarray(np.asarray(img)[..., :3], dtype=np.uint8)
    else:
        vc = getattr(mesh.visual, "vertex_colors", None)
        if vc is None:
            vc = np.tile(np.array([128, 128, 128]).reshape(1, 3), (len(mesh.vertices), 1))
        out["vcolor"] = np.asarray(vc, dtype=np.float32)[..., :3] / 255.0
    return out


class FoundationPose:
    def __init__(self, model_pts, model_normals, symmetry_tfs=None, mesh=None, scorer=None, refiner=None, glctx=None, debug=0,
                 debug_dir="/tmp/fpose_b200_debug"):
        self.gt_pose = None
        self.ignore_normal_flip = True
        self.debug = debug
        self.debug_dir = debug_dir
        os.makedirs(debug_dir, exist_ok=True)
        self.engine = (refiner.engine if refiner is not None else (scorer.engine if scorer is not None else get_engine()))
        self.reset_object(model_pts, model_normals, symmetry_tfs=symmetry_tfs, mesh=mesh)
        self.make_rotation_grid(min_n_views=40, inplane_step=60)
        self.glctx = glctx
        self.scorer = scorer if scorer is not None else ScorePredictor(engine=self.engine)
        self.refiner = refiner if refiner is not None else PoseRefinePredictor(engine=self.engine)
        self.pose_last = None  # used for tracking; per the centred mesh
        # True: read (tx, ty, tz, n_valid) back before the 252 x K loop so that an empty / depth-less mask returns
        # without running it (the reference's control flow, one extra sync); False: sync-free, the loop runs and its
        # result is discarded in that case
        self.strict_early_out = bool(debug)

    def reset_object(self, model_pts, model_normals, symmetry_tfs=None, mesh=None):
        max_xyz = mesh.vertices.max(axis=0)
        min_xyz = mesh.vertices.min(axis=0)
        self.model_center = (min_xyz + max_xyz) / 2
        self.mesh_ori = mesh.copy()
        mesh = mesh.copy()
        mesh.vertices = mesh.vertices - self.model_center.reshape(1, 3)
        self.diameter = synth.mesh_diameter(mesh.vertices)
        self.vox_size = max(self.diameter / 20.0, 0.003)
        self.dist_bin = self.vox_size / 2
        self.angle_bin = 20  # deg
        # estimater.py:59-64: voxel-down-sampled model points / normals (used by callers for ADD-style metrics)
        pts, nrm = meshprep.voxel_down_sample(mesh.vertices, self.vox_size, normals=model_normals)
        self.max_xyz = pts.max(axis=0)
        self.min_xyz = pts.min(axis=0)
        self.pts = torch.tensor(pts, dtype=torch.float32, device="cuda")
        self.normals = torch.nn.functional.normalize(torch.tensor(nrm, dtype=torch.float32, device="cuda"), dim=-1)
        self.mesh_path = None  # the reference exports a temporary .obj for its debug tooling; not needed here
        self.mesh = mesh
        self.mesh_tensors = make_mesh_tensors(mesh)
        mt = self.mesh_tensors
        self.engine.set_mesh(mt["pos"], mt["normals"], mt["faces"], self.diameter, uv=mt.get("uv"), tex=mt.get("tex"),
                             vertex_colors=mt.get("vcolor"))
        self.engine._mesh_src = self.mesh_tensors
        if symmetry_tfs is None:
            self.symmetry_tfs = np.eye(4, dtype=np.float32)[None]
        else:
            self.symmetry_tfs = np.asarray(symmetry_tfs, dtype=np.float32)

    def get_tf_to_centered_mesh(self):
        tf = torch.eye(4, dtype=torch.float32, device="cuda")
        tf[:3, 3] = -torch.as_tensor(self.model_center, device="cuda", dtype=torch.float32)
        return tf

    def to_device(self, s="cuda:0"):
        """estimater.py:88-102 moves tensors / modules / the raster context to `s`.  Here the packed weights, the
        mesh and the frame live in the fp_ctx, which is bound to ONE device for its lifetime: moving to the
        context's own device is a no-op, anything else must be a new Engine on that device (see
        foundationpose_b200.replicas for one estimator per GPU)."""
        dev = torch.device(s)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        if dev.type != "cuda" or idx != self.engine.device_index:
            raise RuntimeError(f"to_device({s!r}): this estimator's fp_ctx lives on cuda:{self.engine.device_index}; "
                               "create the Engine / FoundationPose under torch.cuda.device(...) of the target GPU instead")
        for k, v in list(self.__dict__.items()):
            if torch.is_tensor(v):
                self.__dict__[k] = v.to(s)
        return self

    def make_rotation_grid(self, min_n_views=40, inplane_step=60):
        rot_grid = hypotheses.make_rotation_grid(min_n_views, inplane_step, self.symmetry_tfs)
        self.rot_grid = torch.as_tensor(rot_grid, device="cuda", dtype=torch.float32)
        self._rot_grid_host = torch.from_numpy(rot_grid.copy()).pin_memory()

    def generate_random_pose_hypo(self, K, rgb, depth, mask, scene_pts=None):
        ob_in_cams = self.rot_grid.clone()
        center = self.guess_translation(depth=depth, mask=mask, K=K)
        ob_in_cams[:, :3, 3] = torch.tensor(center, device="cuda", dtype=torch.float32).reshape(1, 3)
        return ob_in_cams

    def guess_translation(self, depth, mask, K):
        return hypotheses.guess_translation(depth, mask, K)

    def register(self, K, rgb, depth, ob_mask, ob_id=None, glctx=None, iteration=5):
        """Compute the object pose in the frame (estimater.py:159-240). Returns (4,4) numpy."""
        e = self.engine
        # erode_depth + bilateral_filter_depth + depth2xyzmap on the device (estimater.py:173-174, :214), then the
        # translation guess and the start poses, also on the device: nothing synchronises until the result is read
        e.set_frame(rgb, depth, K, filter_depth=True, zfar=float("inf"))
        poses, info = e.start_poses(ob_mask, self.rot_grid)
        dump = self.debug >= 2
        if dump:
            import cv2  # only the debug dumps need it

            # estimater.py:176-180: the filtered frame's cloud and the mask, before the early exit.  The frame may be
            # device-resident: the dumps take host copies
            depth_f, xyz = (t.cpu().numpy() for t in e.get_depth())
            rgb_h = rgb.cpu().numpy() if torch.is_tensor(rgb) else np.asarray(rgb)
            self._write_cloud("scene_raw.ply", xyz, rgb_h)
            m = ob_mask.cpu().numpy() if torch.is_tensor(ob_mask) else np.asarray(ob_mask)
            cv2.imwrite(f"{self.debug_dir}/ob_mask.png", (m * 255.0).clip(0, 255))
        if self.strict_early_out:
            # estimater.py:181-189 returns BEFORE the hypothesis loop when fewer than 4 valid masked pixels remain;
            # knowing that on the host costs one 16-byte read-back (a synchronisation the sync-free path avoids)
            head = info.cpu().numpy()
            if head[3] < 4:
                logging.info("valid too small, return")
                pose = np.eye(4)
                pose[:3, 3] = head[:3]
                return pose
        if dump:
            # estimater.py:191-195
            cv2.imwrite(f"{self.debug_dir}/color.png", np.ascontiguousarray(rgb_h[..., ::-1]))
            cv2.imwrite(f"{self.debug_dir}/depth.png", (depth_f * 1000).astype(np.uint16))
            self._write_cloud("scene_complete.ply", xyz, rgb_h)
        self.H, self.W = depth.shape[:2]
        self.K = K
        self.ob_id = ob_id
        self.ob_mask = ob_mask
        poses, canvas = self.refiner.predict(mesh=self.mesh, mesh_tensors=self.mesh_tensors, rgb=rgb, depth=depth, K=K,
                                             ob_in_cams=poses, normal_map=None, xyz_map=None, glctx=self.glctx,
                                             mesh_diameter=self.diameter, iteration=iteration, get_vis=dump, _frame_ready=True)
        if canvas is not None:
            cv2.imwrite(f"{self.debug_dir}/vis_refiner.png", canvas[..., ::-1])
        scores, canvas = self.scorer.predict(mesh=self.mesh, rgb=rgb, depth=depth, K=K, ob_in_cams=poses, normal_map=None,
                                             mesh_tensors=self.mesh_tensors, glctx=self.glctx, mesh_diameter=self.diameter,
                                             get_vis=dump, _frame_ready=True)
        if canvas is not None:
            cv2.imwrite(f"{self.debug_dir}/vis_score.png", canvas[..., ::-1])
        ids = torch.as_tensor(scores).argsort(descending=True)
        scores = scores[ids]
        poses = poses[ids]
        best_pose = poses[0] @ self.get_tf_to_centered_mesh()
        prev = (self.pose_last, getattr(self, "best_id", None), getattr(self, "poses", None), getattr(self, "scores", None))
        self.pose_last = poses[0]
        self.best_id = ids[0]
        self.poses = poses
        self.scores = scores
        # the only host synchronisation of register(): (tx, ty, tz, n_valid) and the best pose in one read-back
        out = torch.cat([info, best_pose.reshape(-1)]).cpu().numpy()
        if out[3] < 4:
            # estimater.py:183-189: too few valid pixels -> identity rotation, guessed translation
            logging.info("valid too small, return")
            pose = np.eye(4)
            pose[:3, 3] = out[:3]
            self.pose_last, self.best_id, self.poses, self.scores = prev  # the reference returns before touching them
            return pose
        return out[4:].reshape(4, 4).copy()

    def _write_cloud(self, name, xyz, rgb):
        """The debug point clouds (estimater.py:178-179, :194-195): valid pixels of the xyz map (host), coloured by the
        host rgb; only with open3d."""
        try:
            import open3d as o3d
        except ImportError:
            logging.info(f"open3d is not installed: {name} not written")
            return
        valid = xyz[..., 2] >= 0.001
        pcd = o3d.geometry.PointCloud()
        pcd.points = o3d.utility.Vector3dVector(xyz[valid].astype(np.float64))
        pcd.colors = o3d.utility.Vector3dVector(rgb[valid].astype(np.float64) / 255.0)
        o3d.io.write_point_cloud(f"{self.debug_dir}/{name}", pcd)

    def track_one(self, rgb, depth, K, iteration, extra={}):
        if self.pose_last is None:
            logging.info("Please init pose by register first")
            raise RuntimeError
        e = self.engine
        _sync_mesh(e, self.mesh, self.mesh_tensors, self.diameter)
        if torch.is_tensor(rgb) or torch.is_tensor(depth):
            # device-resident frame: enqueue the stages one by one (estimater.py:255-264)
            e.set_frame(rgb, depth, K, filter_depth=True, zfar=float("inf"))
            pose, canvas = self.refiner.predict(mesh=self.mesh, mesh_tensors=self.mesh_tensors, rgb=rgb, depth=depth, K=K,
                                                ob_in_cams=self.pose_last.reshape(1, 4, 4), normal_map=None, xyz_map=None,
                                                mesh_diameter=self.diameter, glctx=self.glctx, iteration=iteration,
                                                get_vis=self.debug >= 2, _frame_ready=True)
            if self.debug >= 2:
                extra["vis"] = canvas
            self.pose_last = pose
            return (pose @ self.get_tf_to_centered_mesh()).data.cpu().numpy().reshape(4, 4)
        # host frame (what the drivers pass): the whole frame is one CUDA-graph launch (fp_track)
        pose_in = self.pose_last.reshape(4, 4)
        pose_dev, pose_host = e.track(rgb, depth, K, pose_in, iteration)
        if self.debug >= 2:
            # fp_track leaves this frame in the context — its filtered depth and its xyz map with zfar = inf, what the
            # refiner cropped from — so the canvas pass (estimater.py:263-266) crops the same frame, after the pose is out
            from . import vis  # cv2: only the debug canvases need it

            extra["vis"] = vis.refine_canvas(e, pose_in, pose_dev)
        self.pose_last = pose_dev.reshape(1, 4, 4)
        self.refiner.last_trans_update = self.refiner.last_rot_update = None
        return _uncentre(pose_host, self.model_center)


def _uncentre(pose_host, model_center):
    """pose @ T(-model_center) on the host (estimater.py:268): the pose of the original, un-centred mesh."""
    out = pose_host.astype(np.float64)
    out[:3, 3] -= out[:3, :3] @ np.asarray(model_center, dtype=np.float64)
    return out.astype(np.float32)


def _object_slot(est, caller="track_objects"):
    """The slot of `est`'s mesh in its engine (1..MAX_MESHES-1; slot 0 stays with the single-object calls): assigned at
    first use, reloaded when reset_object() replaced the estimator's mesh_tensors.  Shared by track_objects and
    register_objects, so registering and then tracking the same estimators uploads no mesh."""
    e = est.engine
    owners = e.__dict__.setdefault("_object_slots", {})  # slot -> weakref to the estimator that owns it
    slot = getattr(est, "_object_slot", None)
    if slot is None or slot not in owners or owners[slot]() is not est:
        for s in [s for s, r in owners.items() if r() is None]:
            del owners[s]  # the estimator was garbage-collected
        free = [s for s in range(1, MAX_MESHES) if s not in owners]
        if not free:
            raise ValueError(f"{caller}: an engine holds at most {MAX_MESHES - 1} object meshes")
        slot = free[0]
        owners[slot] = weakref.ref(est)
        est._object_slot, est._object_slot_src = slot, None
    if est._object_slot_src is not est.mesh_tensors:
        mt = est.mesh_tensors
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], est.diameter, uv=mt.get("uv"), tex=mt.get("tex"),
                   vertex_colors=mt.get("vcolor"), slot=slot)
        est._object_slot_src = mt
    return slot


def _shared_engine_of(estimators, caller):
    """The one engine all `estimators` share; refuses mixed engines, repeated estimators and more objects than slots."""
    e = estimators[0].engine
    if any(est.engine is not e for est in estimators):
        raise ValueError(f"{caller}: the estimators must share one engine")
    if len({id(est) for est in estimators}) != len(estimators):
        raise ValueError(f"{caller}: an estimator appears more than once")
    if len(estimators) > MAX_MESHES - 1:
        raise ValueError(f"{caller}: at most {MAX_MESHES - 1} objects per engine, got {len(estimators)}")
    return e


def track_objects(estimators, rgb, depth, K, iteration=2):
    """`[est.track_one(rgb, depth, K, iteration) for est in estimators]` for several objects of one camera stream, as ONE
    CUDA-graph launch per frame (fp_track_objects): the frame is uploaded and filtered once and the objects' poses are
    refined as one batch, each rendering its own mesh.  Same poses as the per-object calls; updates every pose_last.

    The estimators must share one engine (the default: get_engine()).  Each one keeps its mesh in a slot of that engine,
    so alternating objects re-uploads nothing.  Host frames only (uint8 (H,W,3) rgb, float32 (H,W) depth).
    Returns a list of (4,4) float32 poses of the original meshes."""
    estimators = list(estimators)
    if not estimators:
        return []
    if torch.is_tensor(rgb) or torch.is_tensor(depth):
        raise TypeError("track_objects takes host frames (numpy); for device-resident frames call track_one per object")
    e = _shared_engine_of(estimators, "track_objects")
    if any(est.pose_last is None for est in estimators):
        logging.info("Please init pose by register first")
        raise RuntimeError
    slots = [_object_slot(est) for est in estimators]
    poses_in = torch.stack([est.pose_last.reshape(4, 4) for est in estimators])
    poses_dev, poses_host = e.track_objects(rgb, depth, K, poses_in, slots, iteration)
    out = []
    for i, est in enumerate(estimators):
        est.pose_last = poses_dev[i].reshape(1, 4, 4)
        est.refiner.last_trans_update = est.refiner.last_rot_update = None
        out.append(_uncentre(poses_host[i], est.model_center))
    return out


def track_cameras(views, iteration=2):
    """`[[est.track_one(rgb, depth, K, iteration) for est in ests] for ests, rgb, depth, K in views]` for objects seen by
    several camera streams (a multi-camera rig, or several recordings on one GPU), as ONE CUDA-graph launch per call
    (fp_track_cameras): every camera's frame is uploaded and filtered, and every (object, camera) pair is refined in one
    batch, each pair tracked independently in its own camera's frame.  Same poses as the per-object calls; updates every
    pose_last.

    views: one (estimators, rgb, depth, K) per camera, each camera with its own frame size and intrinsics.  All
    estimators share one engine and none appears twice, across cameras or within one; at most MAX_MESHES - 1 objects and
    MAX_CAMERAS cameras with objects.  A camera without estimators gives [] and its frame is not uploaded.  Each
    estimator keeps its mesh in the slot track_objects / register_objects use.  Host frames only (uint8 (H,W,3) rgb,
    float32 (H,W) depth).  Returns one list of (4,4) float32 poses of the original meshes per camera."""
    views = [(list(ests), rgb, depth, K) for ests, rgb, depth, K in views]
    if any(torch.is_tensor(rgb) or torch.is_tensor(depth) for _, rgb, depth, _ in views):
        raise TypeError("track_cameras takes host frames (numpy); for device-resident frames call track_one per object")
    used = [v for v in views if v[0]]
    if not used:
        return [[] for _ in views]
    estimators = [est for ests, _, _, _ in used for est in ests]
    e = _shared_engine_of(estimators, "track_cameras")
    if len(used) > MAX_CAMERAS:
        raise ValueError(f"track_cameras: at most {MAX_CAMERAS} cameras with objects, got {len(used)}")
    if any(est.pose_last is None for est in estimators):
        logging.info("Please init pose by register first")
        raise RuntimeError
    slots = [_object_slot(est, "track_cameras") for est in estimators]
    camera_of = [c for c, (ests, _, _, _) in enumerate(used) for _ in ests]
    poses_in = torch.stack([est.pose_last.reshape(4, 4) for est in estimators])
    poses_dev, poses_host = e.track_cameras([(rgb, depth, K) for _, rgb, depth, K in used], poses_in, camera_of, slots, iteration)
    for i, est in enumerate(estimators):
        est.pose_last = poses_dev[i].reshape(1, 4, 4)
        est.refiner.last_trans_update = est.refiner.last_rot_update = None
    flat = iter(_uncentre(poses_host[i], est.model_center) for i, est in enumerate(estimators))
    return [[next(flat) for _ in ests] for ests, _, _, _ in views]


def register_objects(estimators, K, rgb, depth, ob_masks, ob_ids=None, iteration=5):
    """`[est.register(K=K, rgb=rgb, depth=depth, ob_mask=m, ob_id=i, iteration=iteration) for ...]` bit for bit, for
    several objects of one frame in one fp_register_objects call: the frame is uploaded and filtered once, every object's
    start poses come from one launch, the objects' hypotheses are refined and featurised together in passes of up to 512
    (each rendering its own mesh), and one scorer tail keeps every object's hypotheses to themselves.  Each estimator
    uses its own rotation grid (symmetric objects bring fewer hypotheses) and ends in the state its register() call
    would leave (pose_last, best_id, poses and scores ranked by descending score, H, W, K, ob_id, ob_mask); an object
    with fewer than 4 valid masked depth pixels returns the identity rotation with the guessed translation and keeps
    its previous state.  Everything comes back to the host in one read-back.

    The estimators must share one engine; each keeps its mesh in the same slot track_objects uses, so tracking them
    afterwards uploads no mesh.  Host frames and masks only (uint8 (H,W,3) rgb, float32 (H,W) depth, (H,W) masks).
    Returns a list of (4,4) poses of the original meshes."""
    estimators = list(estimators)
    if not estimators:
        return []
    if torch.is_tensor(rgb) or torch.is_tensor(depth) or any(torch.is_tensor(m) and m.is_cuda for m in ob_masks):
        raise TypeError("register_objects takes host frames and masks (numpy); for device-resident frames call register per object")
    e = _shared_engine_of(estimators, "register_objects")
    ob_masks = list(ob_masks)
    masks = [m.numpy() if torch.is_tensor(m) else np.asarray(m) for m in ob_masks]
    M = len(estimators)
    if len(masks) != M:
        raise ValueError(f"register_objects: {M} estimators but {len(masks)} masks")
    H, W = np.shape(depth)[:2]
    for i, m in enumerate(masks):
        if m.shape != (H, W):
            raise ValueError(f"register_objects: mask {i} has shape {m.shape}, the frame is {(H, W)}")
    ob_ids = [None] * M if ob_ids is None else list(ob_ids)
    if len(ob_ids) != M:
        raise ValueError(f"register_objects: {M} estimators but {len(ob_ids)} ob_ids")
    slots = [_object_slot(est, "register_objects") for est in estimators]
    poses, scores, _, info = e.register_objects(rgb, depth, K, np.stack(masks), [est.rot_grid for est in estimators], slots,
                                                iteration)
    return _finish_register(estimators, poses, scores, info, [(K, H, W)] * M, ob_ids, ob_masks)


def register_cameras(views, ob_ids=None, iteration=5):
    """`[register_objects(ests, K, rgb, depth, ob_masks, ob_ids, iteration) for ests, rgb, depth, K, ob_masks in views]`
    bit for bit, in the returned poses and in every estimator's state, for objects seen by several camera streams (a
    multi-camera rig re-acquiring its objects) in one fp_register_cameras call: every camera's frame is uploaded and
    filtered, every object's start poses come from one launch pair over its own camera's depth and intrinsics, the
    hypotheses of all objects are refined and featurised together in passes of up to 512 (a pass may mix cameras), and
    one scorer tail keeps every object's hypotheses to themselves.  Each estimator uses its own rotation grid and keeps
    its mesh in the slot track_objects / track_cameras use, so tracking them afterwards uploads no mesh.  Everything
    comes back to the host in one read-back.

    views: one (estimators, rgb, depth, K, ob_masks) per camera, each camera with its own frame size and intrinsics and
    one (H,W) mask of its frame per estimator.  ob_ids: None, or one list (or None) per view.  All estimators share one
    engine and none appears twice, across cameras or within one; at most MAX_MESHES - 1 objects and MAX_CAMERAS cameras
    with objects.  A camera without estimators gives [] and its frame is not uploaded.  Host frames and masks only
    (uint8 (H,W,3) rgb, float32 (H,W) depth).  Returns one list of (4,4) poses of the original meshes per camera."""
    views = [(list(ests), rgb, depth, K, list(ob_masks)) for ests, rgb, depth, K, ob_masks in views]
    ob_ids = [None] * len(views) if ob_ids is None else list(ob_ids)
    if len(ob_ids) != len(views):
        raise ValueError(f"register_cameras: {len(views)} views but {len(ob_ids)} ob_ids lists")
    if any(torch.is_tensor(rgb) or torch.is_tensor(depth) or any(torch.is_tensor(m) and m.is_cuda for m in ms)
           for _, rgb, depth, _, ms in views):
        raise TypeError("register_cameras takes host frames and masks (numpy); for device-resident frames call register per object")
    used = [c for c, v in enumerate(views) if v[0]]
    if not used:
        return [[] for _ in views]
    estimators = [est for c in used for est in views[c][0]]
    e = _shared_engine_of(estimators, "register_cameras")
    if len(used) > MAX_CAMERAS:
        raise ValueError(f"register_cameras: at most {MAX_CAMERAS} cameras with objects, got {len(used)}")
    masks, ob_masks, ids, frames, camera_of = [], [], [], [], []
    for j, c in enumerate(used):
        ests, rgb, depth, K, ms = views[c]
        H, W = np.shape(depth)[:2]
        if len(ms) != len(ests):
            raise ValueError(f"register_cameras: camera {c}: {len(ests)} estimators but {len(ms)} masks")
        for i, m in enumerate(ms):
            a = m.numpy() if torch.is_tensor(m) else np.asarray(m)
            if a.shape != (H, W):
                raise ValueError(f"register_cameras: camera {c}: mask {i} has shape {a.shape}, the frame is {(H, W)}")
            masks.append(a)
        v_ids = [None] * len(ests) if ob_ids[c] is None else list(ob_ids[c])
        if len(v_ids) != len(ests):
            raise ValueError(f"register_cameras: camera {c}: {len(ests)} estimators but {len(v_ids)} ob_ids")
        ob_masks += ms
        ids += v_ids
        frames += [(K, H, W)] * len(ests)
        camera_of += [j] * len(ests)
    slots = [_object_slot(est, "register_cameras") for est in estimators]
    poses, scores, _, info = e.register_cameras([views[c][1:4] for c in used], masks, [est.rot_grid for est in estimators],
                                                camera_of, slots, iteration)
    flat = iter(_finish_register(estimators, poses, scores, info, frames, ids, ob_masks))
    return [[next(flat) for _ in ests] for ests, _, _, _, _ in views]


def _finish_register(estimators, poses, scores, info, frames, ob_ids, ob_masks):
    """register()'s ranking, early exit and state updates (estimater.py:181-240) for every estimator, from the object-major
    outputs of Engine.register_objects / register_cameras.  frames[i] = (K, H, W) of estimator i's camera.  Returns the
    list of (4,4) poses of the original meshes."""
    # per object, the ranking and best pose of register(): estimater.py:224-234 on that object's rows
    ranked, rows, o = [], [], 0
    for i, est in enumerate(estimators):
        n = len(est.rot_grid)
        ids = scores[o:o + n].argsort(descending=True)
        p, s = poses[o:o + n][ids], scores[o:o + n][ids]
        best_pose = p[0] @ est.get_tf_to_centered_mesh()
        ranked.append((ids, p, s))
        rows.append(torch.cat([info[i], best_pose.reshape(-1)]))
        o += n
    out = torch.stack(rows).cpu().numpy()  # the one host synchronisation: (tx, ty, tz, n_valid) and the best pose per object
    result = []
    for i, est in enumerate(estimators):
        early = out[i, 3] < 4
        est.refiner.last_trans_update = est.refiner.last_rot_update = None
        if not (early and getattr(est, "strict_early_out", False)):  # register()'s strict path returns before recording the frame
            est.K, est.H, est.W = frames[i]
            est.ob_id = ob_ids[i]
            est.ob_mask = ob_masks[i]
        if early:
            # estimater.py:183-189: too few valid pixels -> identity rotation, guessed translation, state untouched
            logging.info("valid too small, return")
            pose = np.eye(4)
            pose[:3, 3] = out[i, :3]
            result.append(pose)
            continue
        ids, p, s = ranked[i]
        est.pose_last = p[0]
        est.best_id = ids[0]
        est.poses = p
        est.scores = s
        result.append(out[i, 4:].reshape(4, 4).copy())
    return result
