"""Host-side owner of one `fp_ctx`: packs reference checkpoints for the CUDA kernels and exposes the
hot-path entry points of libfpose.so on torch CUDA tensors.

torch is used for device memory, streams and (in parallel.py) torch.distributed only; every
computation on the hot path happens inside the C-ABI library.
"""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib, packing
from ._lib import lib

CROP_SHAPE = (166, 2, 84, 8)  # padded fp16 crop image consumed by the stem convolution: rows x {even, odd cols} x pairs x ch


class _FpTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("dtype", C.c_int), ("numel", C.c_longlong)]


def _proto():
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    lib.fp_create.argtypes = [C.POINTER(vp)]
    lib.fp_destroy.argtypes = [vp]
    lib.fp_set_config.argtypes = [vp, i, f, f]
    lib.fp_mesh_info.argtypes = [vp, C.POINTER(i)]
    lib.fp_set_crop_tile.argtypes = [vp, i]
    lib.fp_crop_stats.argtypes = [vp, vp, i, i, C.POINTER(i), vp]
    lib.fp_track.argtypes = [vp, vp, vp, C.POINTER(f), i, i, vp, i, vp, vp, vp]
    lib.fp_track_objects.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, C.POINTER(i), vp, i, vp, vp, vp]
    lib.fp_track_cameras.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(f), C.POINTER(i), C.POINTER(i), i, C.POINTER(i),
                                     C.POINTER(i), vp, i, vp, vp, vp]
    lib.fp_register_objects.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, C.POINTER(i), C.POINTER(i), vp, vp, i, vp, vp, vp,
                                        vp, vp]
    lib.fp_register_cameras.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(f), C.POINTER(i), C.POINTER(i), i,
                                        C.POINTER(i), C.POINTER(i), C.POINTER(i), C.POINTER(vp), vp, i, vp, vp, vp, vp, vp]
    lib.fp_graph_captures.argtypes = [vp]
    lib.fp_graph_captures.restype = C.c_ulonglong
    lib.fp_load_network.argtypes = [vp, i, C.POINTER(_FpTensor), i]
    lib.fp_set_mesh.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp, i, i, f]
    lib.fp_set_mesh_slot.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp, i, i, f]
    lib.fp_set_frame.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, f, vp]
    lib.fp_get_depth.argtypes = [vp, vp, vp, vp]
    lib.fp_set_xyz_map.argtypes = [vp, vp, vp]
    lib.fp_make_crops.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    lib.fp_start_poses.argtypes = [vp, vp, i, vp, i, vp, vp, vp]
    lib.fp_refine.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    lib.fp_score.argtypes = [vp, vp, i, vp, vp, vp]
    lib.fp_score_features.argtypes = [vp, vp, i, vp, vp]
    lib.fp_score_tail.argtypes = [vp, vp, i, vp, vp, vp]
    lib.fp_register.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    lib.fp_op_refine_net.argtypes = [vp, vp, i, vp, vp, vp]
    lib.fp_op_score_feats.argtypes = [vp, vp, i, vp, vp]
    lib.fp_op_tokens.argtypes = [vp, i, vp, i, vp, vp]
    lib.fp_op_depth_filter.argtypes = [vp, vp, i, i, i, vp]
    lib.fp_op_pose_update.argtypes = [vp, vp, vp, vp, i, f, f, vp]
    lib.fp_vis.argtypes = [vp, i, vp, vp, i, vp, vp, C.POINTER(i), vp]
    lib.fp_vis_size.argtypes = [i, i, C.POINTER(i)]
    lib.fp_vis_colormap.argtypes = [vp]
    lib.fp_vis_crops.argtypes = [vp, vp, i, i, vp, vp]
    lib.fp_vis_workspace_bytes.argtypes = [vp]
    lib.fp_vis_workspace_bytes.restype = C.c_ulonglong
    for name in ("fp_create", "fp_destroy", "fp_set_config", "fp_mesh_info", "fp_set_crop_tile", "fp_crop_stats", "fp_track", "fp_track_objects", "fp_track_cameras", "fp_register_objects", "fp_register_cameras", "fp_set_xyz_map", "fp_load_network", "fp_set_mesh",
                 "fp_set_mesh_slot", "fp_set_frame",
                 "fp_get_depth", "fp_make_crops", "fp_start_poses", "fp_refine", "fp_score", "fp_score_features", "fp_score_tail",
                 "fp_register", "fp_op_refine_net", "fp_op_score_feats", "fp_op_tokens", "fp_op_depth_filter",
                 "fp_op_pose_update", "fp_vis", "fp_vis_size", "fp_vis_colormap", "fp_vis_crops"):
        getattr(lib, name).restype = C.c_int


_proto()

FRAME_ON_DEVICE = 1
MAX_MESHES = 64  # FP_MAX_MESHES: mesh slots per context
MAX_CAMERAS = 16  # FP_MAX_CAMERAS: camera streams per fp_track_cameras / fp_register_cameras call
_NO_PIN = os.environ.get("FPOSE_NO_PIN") == "1"  # A/B: skip the pinned staging of host frames
FRAME_FILTER_DEPTH = 2


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# ---------------------------------------------------------------------------------------------
# checkpoint -> packed tensors
# ---------------------------------------------------------------------------------------------
def _bn_of(sd, prefix):
    if f"{prefix}.weight" not in sd:
        return None
    return {"weight": sd[f"{prefix}.weight"], "bias": sd[f"{prefix}.bias"], "running_mean": sd[f"{prefix}.running_mean"],
            "running_var": sd[f"{prefix}.running_var"], "eps": 1e-5}


def pack_network(sd, kind):
    """Reference state_dict (learning/models/{refine,score}_network.py layout) -> {name: np.ndarray}."""
    A, AB = ("encodeA", "encodeAB") if kind == "refine" else ("encoderA", "encoderAB")
    convs = [(f"{A}.0.net.0", f"{A}.0.net.1"), (f"{A}.1.net.0", f"{A}.1.net.1"),
             (f"{A}.2.conv1", f"{A}.2.bn1"), (f"{A}.2.conv2", f"{A}.2.bn2"),
             (f"{A}.3.conv1", f"{A}.3.bn1"), (f"{A}.3.conv2", f"{A}.3.bn2"),
             (f"{AB}.0.conv1", f"{AB}.0.bn1"), (f"{AB}.0.conv2", f"{AB}.0.bn2"),
             (f"{AB}.1.conv1", f"{AB}.1.bn1"), (f"{AB}.1.conv2", f"{AB}.1.bn2"),
             (f"{AB}.2.net.0", f"{AB}.2.net.1"),
             (f"{AB}.3.conv1", f"{AB}.3.bn1"), (f"{AB}.3.conv2", f"{AB}.3.bn2"),
             (f"{AB}.4.conv1", f"{AB}.4.bn1"), (f"{AB}.4.conv2", f"{AB}.4.bn2")]
    out = {}
    for i, (cname, bname) in enumerate(convs):
        w = sd[f"{cname}.weight"]
        if i == 0 and w.shape[1] > 8:
            raise ValueError("stem convolution supports c_in <= 8 (reference configs use 6)")
        wf, bf = packing.fold_bn(w, sd.get(f"{cname}.bias"), _bn_of(sd, bname))
        out[f"enc.{i}.w"] = (packing.pack_conv7(wf) if i == 0 else packing.pack_conv3(wf)).numpy()
        out[f"enc.{i}.b"] = bf.float().contiguous().numpy()
    out["pe"] = sd["pos_embed.pe"].float().reshape(-1, 512)[:400].contiguous().numpy()
    h16 = lambda t: t.detach().float().contiguous().half().numpy()
    f32 = lambda t: t.detach().float().contiguous().numpy()
    if kind == "refine":
        heads = ("trans_head", "rot_head")
        out["heads.in_w"] = h16(torch.cat([sd[f"{h}.0.self_attn.in_proj_weight"] for h in heads], 0))
        out["heads.in_b"] = f32(torch.cat([sd[f"{h}.0.self_attn.in_proj_bias"] for h in heads], 0))
        for g, h in enumerate(heads):
            if sd[f"{h}.1.weight"].shape[0] != 3:
                raise ValueError("only rot_rep='axis_angle' (3 outputs) is supported")
            out[f"head{g}.out_w"] = h16(sd[f"{h}.0.self_attn.out_proj.weight"])
            out[f"head{g}.out_b"] = f32(sd[f"{h}.0.self_attn.out_proj.bias"])
            out[f"head{g}.ln1_g"] = f32(sd[f"{h}.0.norm1.weight"])
            out[f"head{g}.ln1_b"] = f32(sd[f"{h}.0.norm1.bias"])
            out[f"head{g}.ff1_w"] = h16(sd[f"{h}.0.linear1.weight"])
            out[f"head{g}.ff1_b"] = f32(sd[f"{h}.0.linear1.bias"])
            out[f"head{g}.ff2_w"] = h16(sd[f"{h}.0.linear2.weight"])
            out[f"head{g}.ff2_b"] = f32(sd[f"{h}.0.linear2.bias"])
            out[f"head{g}.ln2_g"] = f32(sd[f"{h}.0.norm2.weight"])
            out[f"head{g}.ln2_b"] = f32(sd[f"{h}.0.norm2.bias"])
            out[f"head{g}.fin_w"] = f32(sd[f"{h}.1.weight"])
            out[f"head{g}.fin_b"] = f32(sd[f"{h}.1.bias"])
    else:
        # `att` runs on the fp16 tensor-core path; the cross-hypothesis tail stays fp32 end to end
        # (0.3 GFLOP in total, and it decides the arg-max)
        for src, dst, cvt in (("att", "att", h16), ("att_cross", "cross", f32)):
            out[f"{dst}.in_w"] = cvt(sd[f"{src}.in_proj_weight"])
            out[f"{dst}.in_b"] = f32(sd[f"{src}.in_proj_bias"])
            out[f"{dst}.out_w"] = cvt(sd[f"{src}.out_proj.weight"])
            out[f"{dst}.out_b"] = f32(sd[f"{src}.out_proj.bias"])
        # `att`'s out_proj acts on the token MEAN (one 512-vector per hypothesis): a [N,512] x [512,512] product in fp32
        out["att.out_w32"] = f32(sd["att.out_proj.weight"])
        del out["att.out_w"]
        out["lin.w"] = f32(sd["linear.weight"].reshape(-1))
        out["lin.b"] = f32(sd["linear.bias"].reshape(-1))
    return out


class Engine:
    """One fp_ctx on the current CUDA device."""

    def __init__(self):
        if not torch.cuda.is_available():
            raise _lib.FposeError("foundationpose_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        h = C.c_void_p()
        _lib.check(lib.fp_create(C.byref(h)), "fp_create")
        self._h = h
        self.device_index = torch.cuda.current_device()
        self.diameter = None
        self.frame_hw = None

    def close(self):
        if getattr(self, "_h", None):
            lib.fp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- setup
    def set_config(self, kind, crop_ratio=1.2, rot_normalizer=0.3490658503988659):
        """Per-predictor config (each reference predictor reads its own config.yml): kind 'refine' | 'score'."""
        which = 0 if kind == "refine" else 1
        _lib.check(lib.fp_set_config(self._h, which, float(crop_ratio), float(rot_normalizer)), "fp_set_config")

    def load_network(self, kind, state_dict):
        packed = pack_network(state_dict, kind)
        arr = (_FpTensor * len(packed))()
        keep = []
        for i, (name, a) in enumerate(packed.items()):
            a = np.ascontiguousarray(a)
            keep.append(a)
            arr[i] = _FpTensor(name.encode(), a.ctypes.data, 1 if a.dtype == np.float16 else 0, a.size)
        _lib.check(lib.fp_load_network(self._h, 0 if kind == "refine" else 1, arr, len(packed)), "fp_load_network")

    def set_mesh(self, vertices, normals, faces, diameter, uv=None, tex=None, vertex_colors=None, slot=0):
        """uv: (V,2) with v already flipped (Utils.py:117); tex: uint8 (Ht,Wt,3); vertex_colors: float 0..1.
        slot: 0..MAX_MESHES-1; slot 0 is the mesh of every single-object call, the others are for track_objects."""
        pos = np.ascontiguousarray(vertices, dtype=np.float32)
        nrm = np.ascontiguousarray(normals, dtype=np.float32)
        fc = np.ascontiguousarray(faces, dtype=np.int32)
        uvp = texp = colp = None
        Ht = Wt = 0
        if uv is not None and tex is not None:
            uvp = np.ascontiguousarray(uv, dtype=np.float32)
            texp = np.ascontiguousarray(tex[..., :3], dtype=np.uint8)
            Ht, Wt = texp.shape[:2]
        else:
            colp = np.ascontiguousarray(vertex_colors, dtype=np.float32)
        cp = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
        _lib.check(lib.fp_set_mesh_slot(self._h, int(slot), len(pos), len(fc), cp(pos), cp(nrm), cp(uvp), cp(colp), cp(fc), cp(texp),
                                        Ht, Wt, float(diameter)), "fp_set_mesh")
        if slot == 0:
            self.diameter = float(diameter)
            self.mesh_key = (len(pos), len(fc), float(diameter))

    def graph_captures(self):
        """Number of CUDA graphs this context has captured (a replay captures none)."""
        return int(lib.fp_graph_captures(self._h))

    def mesh_info(self):
        """dict(meshlets, closed, front_sign, V, F) of the mesh in the context (fp_mesh_info)."""
        info = (C.c_int * 5)()
        _lib.check(lib.fp_mesh_info(self._h, info), "fp_mesh_info")
        return dict(meshlets=info[0], closed=bool(info[1]), front_sign=info[2], V=info[3], F=info[4])

    def set_crop_tile(self, tile=0):
        """Force the crop producer's tile edge (16 / 32 / 80; 0 = automatic from the batch size)."""
        _lib.check(lib.fp_set_crop_tile(self._h, int(tile)), "fp_set_crop_tile")

    def crop_stats(self, poses, mode=0):
        """Work counters of one crop pass: dict(meshlet_visits, triangles, fragments, near_plane_triangles)."""
        poses = self._poses(poses)
        st = (C.c_int * 4)()
        _lib.check(lib.fp_crop_stats(self._h, _p(poses), len(poses), mode, st, _stream()), "fp_crop_stats")
        return dict(meshlet_visits=st[0], triangles=st[1], fragments=st[2], near_plane_triangles=st[3])

    def track(self, rgb, depth, K, pose_in, iterations, pose_out=None):
        """fp_track: one CUDA-graph launch per frame (upload + depth filters + xyz map + refiner passes + read-back).
        rgb uint8 (H,W,3) / depth float32 (H,W) HOST arrays; pose_in (4,4) CUDA tensor or None (continue).
        Returns (pose_out CUDA (4,4), pose host (4,4) float32 numpy)."""
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        H, W = depth.shape
        Kf = (C.c_float * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        if pose_in is not None:
            pose_in = pose_in.reshape(4, 4).contiguous().float()
        if pose_out is None:
            pose_out = torch.empty(4, 4, dtype=torch.float32, device="cuda")
        host = np.empty((4, 4), dtype=np.float32)
        _lib.check(lib.fp_track(self._h, C.c_void_p(rgb.ctypes.data), C.c_void_p(depth.ctypes.data), Kf, H, W, _p(pose_in),
                                int(iterations), _p(pose_out), C.c_void_p(host.ctypes.data), _stream()), "fp_track")
        self.frame_hw = (H, W)
        return pose_out, host

    def track_objects(self, rgb, depth, K, poses_in, slots, iterations):
        """fp_track_objects: `track` for M objects of one frame in ONE CUDA-graph launch, object i rendering the mesh in
        slot slots[i] (loaded by set_mesh(..., slot=)).  rgb uint8 (H,W,3) / depth float32 (H,W) HOST arrays; poses_in
        (M,4,4) CUDA tensor.  Returns (poses CUDA (M,4,4), poses host (M,4,4) float32 numpy)."""
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        H, W = depth.shape
        Kf = (C.c_float * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        poses_in = poses_in.reshape(-1, 4, 4).contiguous().float()
        M = len(poses_in)
        slots = [int(s) for s in slots]
        if len(slots) != M:
            raise ValueError(f"track_objects: {M} poses but {len(slots)} slots")
        out = torch.empty(M, 4, 4, dtype=torch.float32, device="cuda")
        host = np.empty((M, 4, 4), dtype=np.float32)
        _lib.check(lib.fp_track_objects(self._h, C.c_void_p(rgb.ctypes.data), C.c_void_p(depth.ctypes.data), Kf, H, W, M,
                                        (C.c_int * M)(*slots), _p(poses_in), int(iterations), _p(out),
                                        C.c_void_p(host.ctypes.data), _stream()), "fp_track_objects")
        self.frame_hw = (H, W)
        return out, host

    def track_cameras(self, frames, poses_in, camera_of, slots, iterations):
        """fp_track_cameras: `track_objects` for M objects spread over C camera streams in ONE CUDA-graph launch.  frames: C
        tuples (rgb uint8 (H,W,3), depth float32 (H,W), K (3,3)) of HOST arrays, one per camera, each with its own size and
        intrinsics; object i is seen by camera camera_of[i] and renders the mesh in slot slots[i]; poses_in (M,4,4) CUDA
        tensor.  Returns (poses CUDA (M,4,4), poses host (M,4,4) float32 numpy)."""
        frames = [(np.ascontiguousarray(rgb, dtype=np.uint8), np.ascontiguousarray(depth, dtype=np.float32), K) for rgb, depth, K in frames]
        n_cam = len(frames)
        poses_in = poses_in.reshape(-1, 4, 4).contiguous().float()
        M = len(poses_in)
        camera_of, slots = [int(c) for c in camera_of], [int(s) for s in slots]
        if len(camera_of) != M or len(slots) != M:
            raise ValueError(f"track_cameras: {M} poses, {len(camera_of)} camera ids and {len(slots)} slots")
        rgbs = (C.c_void_p * n_cam)(*[rgb.ctypes.data for rgb, _, _ in frames])
        depths = (C.c_void_p * n_cam)(*[depth.ctypes.data for _, depth, _ in frames])
        Ks = (C.c_float * (9 * n_cam))(*[float(x) for _, _, K in frames for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        Hs = (C.c_int * n_cam)(*[depth.shape[0] for _, depth, _ in frames])
        Ws = (C.c_int * n_cam)(*[depth.shape[1] for _, depth, _ in frames])
        out = torch.empty(M, 4, 4, dtype=torch.float32, device="cuda")
        host = np.empty((M, 4, 4), dtype=np.float32)
        _lib.check(lib.fp_track_cameras(self._h, n_cam, rgbs, depths, Ks, Hs, Ws, M, (C.c_int * M)(*camera_of), (C.c_int * M)(*slots),
                                        _p(poses_in), int(iterations), _p(out), C.c_void_p(host.ctypes.data), _stream()),
                   "fp_track_cameras")
        self.frame_hw = frames[0][1].shape  # camera 0's frame is the context's frame
        return out, host

    def register_objects(self, rgb, depth, K, masks, rot_grids, slots, iterations):
        """fp_register_objects: the register() hot path for M objects of one frame in one call, object i rendering the mesh
        in slot slots[i].  rgb uint8 (H,W,3) / depth float32 (H,W) / masks (M,H,W) (nonzero = object) HOST arrays;
        rot_grids: M CUDA float32 (N_i,4,4) rotation grids.  Returns CUDA tensors: poses (sum N_i,4,4) refined, object-major
        and unranked; scores (sum N_i,); best (M,) int32, each object's first arg-max relative to its own rows; info (M,4)
        = (tx, ty, tz, n_valid) per object."""
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        H, W = depth.shape
        masks = np.ascontiguousarray(masks)
        M = len(masks)
        if masks.shape != (M, H, W):
            raise ValueError(f"register_objects: masks must be (M, {H}, {W}), got {masks.shape}")
        masks = np.ascontiguousarray(masks > 0, dtype=np.uint8)  # the reference tests `mask > 0` (estimater.py:138, :183)
        slots = [int(s) for s in slots]
        rot_grids = [g.reshape(-1, 4, 4) for g in rot_grids]
        if len(slots) != M or len(rot_grids) != M:
            raise ValueError(f"register_objects: {M} masks, {len(slots)} slots and {len(rot_grids)} rotation grids")
        n_hyp = [len(g) for g in rot_grids]
        grids = torch.cat(rot_grids).to(device="cuda", dtype=torch.float32).contiguous()
        total = len(grids)
        Kf = (C.c_float * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        poses = torch.empty(total, 4, 4, dtype=torch.float32, device="cuda")
        scores = torch.empty(total, dtype=torch.float32, device="cuda")
        best = torch.empty(M, dtype=torch.int32, device="cuda")
        info = torch.empty(M, 4, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_register_objects(self._h, C.c_void_p(rgb.ctypes.data), C.c_void_p(depth.ctypes.data), Kf, H, W, M,
                                           (C.c_int * M)(*slots), (C.c_int * M)(*n_hyp), C.c_void_p(masks.ctypes.data), _p(grids),
                                           int(iterations), _p(poses), _p(scores), _p(best), _p(info), _stream()),
                   "fp_register_objects")
        self.frame_hw = (H, W)
        return poses, scores, best, info

    def register_cameras(self, frames, masks, rot_grids, camera_of, slots, iterations):
        """fp_register_cameras: `register_objects` for M objects spread over C camera streams in one call.  frames: C tuples
        (rgb uint8 (H,W,3), depth float32 (H,W), K (3,3)) of HOST arrays, one per camera, each with its own size and
        intrinsics; object i is seen by camera camera_of[i], renders the mesh in slot slots[i] and has the HOST mask
        masks[i] (nonzero = object) of its camera's frame size; rot_grids: M CUDA float32 (N_i,4,4) rotation grids.
        Returns the CUDA tensors of register_objects: poses (sum N_i,4,4), scores (sum N_i,), best (M,), info (M,4)."""
        frames = [(np.ascontiguousarray(rgb, dtype=np.uint8), np.ascontiguousarray(depth, dtype=np.float32), K) for rgb, depth, K in frames]
        n_cam = len(frames)
        M = len(masks)
        camera_of, slots = [int(c) for c in camera_of], [int(s) for s in slots]
        rot_grids = [g.reshape(-1, 4, 4) for g in rot_grids]
        if len(camera_of) != M or len(slots) != M or len(rot_grids) != M:
            raise ValueError(f"register_cameras: {M} masks, {len(camera_of)} camera ids, {len(slots)} slots and "
                             f"{len(rot_grids)} rotation grids")
        masks = [np.asarray(m) for m in masks]
        for i, (m, c) in enumerate(zip(masks, camera_of)):
            if 0 <= c < n_cam and m.shape != frames[c][1].shape:
                raise ValueError(f"register_cameras: mask {i} has shape {m.shape}, camera {c}'s frame is {frames[c][1].shape}")
        masks = [np.ascontiguousarray(m > 0, dtype=np.uint8) for m in masks]  # the reference tests `mask > 0` (estimater.py:138, :183)
        n_hyp = [len(g) for g in rot_grids]
        grids = torch.cat(rot_grids).to(device="cuda", dtype=torch.float32).contiguous()
        total = len(grids)
        rgbs = (C.c_void_p * n_cam)(*[rgb.ctypes.data for rgb, _, _ in frames])
        depths = (C.c_void_p * n_cam)(*[depth.ctypes.data for _, depth, _ in frames])
        Ks = (C.c_float * (9 * n_cam))(*[float(x) for _, _, K in frames for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        Hs = (C.c_int * n_cam)(*[depth.shape[0] for _, depth, _ in frames])
        Ws = (C.c_int * n_cam)(*[depth.shape[1] for _, depth, _ in frames])
        poses = torch.empty(total, 4, 4, dtype=torch.float32, device="cuda")
        scores = torch.empty(total, dtype=torch.float32, device="cuda")
        best = torch.empty(M, dtype=torch.int32, device="cuda")
        info = torch.empty(M, 4, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_register_cameras(self._h, n_cam, rgbs, depths, Ks, Hs, Ws, M, (C.c_int * M)(*camera_of),
                                           (C.c_int * M)(*slots), (C.c_int * M)(*n_hyp), (C.c_void_p * M)(*[m.ctypes.data for m in masks]),
                                           _p(grids), int(iterations), _p(poses), _p(scores), _p(best), _p(info), _stream()),
                   "fp_register_cameras")
        self.frame_hw = frames[0][1].shape  # camera 0's frame is the context's frame
        return poses, scores, best, info

    def set_frame(self, rgb, depth, K, filter_depth=True, zfar=float("inf")):
        """rgb uint8 (H,W,3), depth float32 (H,W): numpy / CPU tensors (pinned for async H2D) or CUDA tensors."""
        Kf = (C.c_float * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        flags = FRAME_FILTER_DEPTH if filter_depth else 0
        if torch.is_tensor(rgb) and rgb.is_cuda:
            assert torch.is_tensor(depth) and depth.is_cuda
            rgb = rgb.contiguous()
            depth = depth.contiguous().float()
            assert rgb.dtype == torch.uint8
            flags |= FRAME_ON_DEVICE
            H, W = depth.shape
            rp, dp = _p(rgb), _p(depth)
        else:
            rgb = rgb if torch.is_tensor(rgb) else torch.from_numpy(np.ascontiguousarray(rgb, dtype=np.uint8))
            depth = depth if torch.is_tensor(depth) else torch.from_numpy(np.ascontiguousarray(depth, dtype=np.float32))
            rgb = rgb.contiguous()
            depth = depth.contiguous()
            assert rgb.dtype == torch.uint8 and depth.dtype == torch.float32
            H, W = depth.shape
            if not rgb.is_pinned() and not _NO_PIN:
                # pageable host memory makes cudaMemcpyAsync synchronous and staged by the driver: stage through a
                # pinned buffer owned by the engine (the previous frame's copy has been consumed: same stream)
                pin = getattr(self, "_pin", None)
                if pin is None or pin[0].shape != rgb.shape or pin[1].shape != depth.shape:
                    torch.cuda.current_stream().synchronize()
                    pin = self._pin = (torch.empty(rgb.shape, dtype=torch.uint8).pin_memory(), torch.empty(depth.shape, dtype=torch.float32).pin_memory(),
                                       torch.cuda.Event())
                else:
                    pin[2].synchronize()
                pin[0].copy_(rgb)
                pin[1].copy_(depth)
                rgb, depth = pin[0], pin[1]
            rp, dp = _p(rgb), _p(depth)
        self._frame_keep = (rgb, depth)
        _lib.check(lib.fp_set_frame(self._h, rp, dp, Kf, H, W, flags, float(zfar), _stream()), "fp_set_frame")
        if getattr(self, "_pin", None) is not None and rgb is self._pin[0]:
            self._pin[2].record()  # the staging buffers may be overwritten once this point of the stream has passed
        self.frame_hw = (H, W)

    def set_xyz_map(self, xyz_map):
        """Caller-supplied xyz map (H,W,3) float32 — numpy / CPU tensor / CUDA tensor — instead of the derived one."""
        x = xyz_map if torch.is_tensor(xyz_map) else torch.from_numpy(np.ascontiguousarray(xyz_map, dtype=np.float32))
        x = x.float().contiguous()
        assert tuple(x.shape) == (*self.frame_hw, 3), "xyz_map must be (H, W, 3)"
        self._xyz_keep = x
        _lib.check(lib.fp_set_xyz_map(self._h, _p(x), _stream()), "fp_set_xyz_map")

    def get_depth(self):
        H, W = self.frame_hw
        d = torch.empty(H, W, dtype=torch.float32, device="cuda")
        x = torch.empty(H, W, 3, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_get_depth(self._h, _p(d), _p(x), _stream()), "fp_get_depth")
        return d, x

    def start_poses(self, mask, rot_grid):
        """guess_translation + start poses on the device (no host synchronisation).
        mask: bool/uint8 (H,W) numpy / CPU tensor / CUDA tensor; rot_grid: (N,4,4) CUDA float32.
        Returns poses (N,4,4) and info (4,) = (tx, ty, tz, n_valid), both CUDA tensors."""
        rot_grid = rot_grid.contiguous()
        N = len(rot_grid)
        # the reference tests `mask > 0` (estimater.py:138, :183): binarise before the uint8 cast so that fractional
        # float masks and values >= 256 behave the same
        if not torch.is_tensor(mask):
            mask = torch.as_tensor(np.ascontiguousarray(mask))
        m = (mask if mask.dtype == torch.bool else (mask > 0)).to(torch.uint8).contiguous()
        on_dev = 1 if m.is_cuda else 0
        self._mask_keep = m
        poses = torch.empty(N, 4, 4, dtype=torch.float32, device="cuda")
        info = torch.empty(4, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_start_poses(self._h, _p(m), on_dev, _p(rot_grid), N, _p(poses), _p(info), _stream()), "fp_start_poses")
        return poses, info

    # ---- hot path
    @staticmethod
    def _poses(poses):
        poses = torch.as_tensor(poses, dtype=torch.float32)
        if not poses.is_cuda:
            poses = poses.cuda()
        return poses.reshape(-1, 4, 4).contiguous()

    def make_crops(self, poses, mode=0, want_crops=True, want_dbg=False):
        poses = self._poses(poses)
        N = len(poses)
        crops = torch.empty(2 * N, *CROP_SHAPE, dtype=torch.float16, device="cuda") if want_crops else None
        dbg = torch.empty(N, 2, 160, 160, 6, dtype=torch.float32, device="cuda") if want_dbg else None
        win = torch.empty(N, 4, dtype=torch.float32, device="cuda")
        if N == 0:
            return crops, dbg, win
        _lib.check(lib.fp_make_crops(self._h, _p(poses), N, mode, _p(crops), _p(dbg), _p(win), _stream()), "fp_make_crops")
        return crops, dbg, win

    def refine(self, poses, iterations):
        poses = self._poses(poses)
        N = len(poses)
        out = torch.empty_like(poses)
        lt = torch.empty(N, 3, dtype=torch.float32, device="cuda")
        lr = torch.empty(N, 3, 3, dtype=torch.float32, device="cuda")
        if N == 0:
            return out, lt, lr
        _lib.check(lib.fp_refine(self._h, _p(poses), N, int(iterations), _p(out), _p(lt), _p(lr), _stream()), "fp_refine")
        return out, lt, lr

    def score(self, poses):
        poses = self._poses(poses)
        N = len(poses)
        scores = torch.empty(N, dtype=torch.float32, device="cuda")
        best = torch.empty(1, dtype=torch.int32, device="cuda")
        _lib.check(lib.fp_score(self._h, _p(poses), N, _p(scores), _p(best), _stream()), "fp_score")
        return scores, best

    def score_features(self, poses):
        poses = self._poses(poses)
        N = len(poses)
        feats = torch.empty(N, 512, dtype=torch.float32, device="cuda")
        if N == 0:
            return feats
        _lib.check(lib.fp_score_features(self._h, _p(poses), N, _p(feats), _stream()), "fp_score_features")
        return feats

    def score_tail(self, feats):
        feats = feats.contiguous().float()
        L = feats.shape[0]
        scores = torch.empty(L, dtype=torch.float32, device="cuda")
        best = torch.empty(1, dtype=torch.int32, device="cuda")
        _lib.check(lib.fp_score_tail(self._h, _p(feats), L, _p(scores), _p(best), _stream()), "fp_score_tail")
        return scores, best

    def register_host(self, poses_host, iterations, out_poses=None, out_scores=None):
        """fp_register: pinned host buffers in, host buffers out (synchronous)."""
        poses_host = poses_host if torch.is_tensor(poses_host) else torch.from_numpy(np.ascontiguousarray(poses_host, dtype=np.float32))
        poses_host = poses_host.reshape(-1, 4, 4).contiguous()
        N = len(poses_host)
        out_poses = torch.empty(N, 4, 4, dtype=torch.float32).pin_memory() if out_poses is None else out_poses
        out_scores = torch.empty(N, dtype=torch.float32).pin_memory() if out_scores is None else out_scores
        best = torch.zeros(1, dtype=torch.int32)
        _lib.check(lib.fp_register(self._h, _p(poses_host), N, int(iterations), _p(out_poses), _p(out_scores), _p(best),
                                   _stream()), "fp_register")
        return out_poses, out_scores, int(best.item())

    # ---- debug canvases
    def vis(self, kind, poses_a, poses_b=None, order=None):
        """fp_vis: the get_vis canvas of the context's current frame and mesh, without its text labels, as a CUDA uint8
        (H, W, 3) tensor.  kind 'refine': the crops at poses_a (the poses predict() received) beside those at poses_b
        (the refined poses); kind 'score': the scorer's rows of poses_a, row s showing hypothesis order[s]."""
        k = 0 if kind == "refine" else 1
        poses_a = self._poses(poses_a)
        N = len(poses_a)
        if k == 0:
            poses_b = self._poses(poses_b)
            if len(poses_b) != N:
                raise ValueError(f"vis: {N} start poses but {len(poses_b)} refined poses")
        else:
            order = torch.as_tensor(order, device="cuda").to(torch.int32).contiguous()
            if order.numel() != N:
                raise ValueError(f"vis: {N} poses but {order.numel()} row indices")
        H, W = vis_size(kind, N)
        canvas = torch.empty(H, W, 3, dtype=torch.uint8, device="cuda")
        _lib.check(lib.fp_vis(self._h, k, _p(poses_a), _p(poses_b) if k == 0 else None, N, _p(order) if k == 1 else None,
                              _p(canvas), None, _stream()), "fp_vis")
        return canvas

    def vis_crops(self, poses, mode=0):
        """The crop pass of vis alone (test hook): (N, 2, 160, 160, 4) CUDA float32 = (r, g, b, depth) of the rendered
        and the observed crop; depth is the normalised z (mode 0, refiner) or raw metres (mode 1, scorer)."""
        poses = self._poses(poses)
        rec = torch.empty(len(poses), 2, 160, 160, 4, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_vis_crops(self._h, _p(poses), len(poses), int(mode), _p(rec), _stream()), "fp_vis_crops")
        return rec

    def vis_workspace_bytes(self):
        """Device memory the debug canvases hold in this context (0 until the first vis call)."""
        return int(lib.fp_vis_workspace_bytes(self._h))

    # ---- single-operator hooks (tests)
    def op_refine_net(self, crops, N):
        trans = torch.empty(N, 3, dtype=torch.float32, device="cuda")
        rot = torch.empty(N, 3, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_op_refine_net(self._h, _p(crops), N, _p(trans), _p(rot), _stream()), "fp_op_refine_net")
        return trans, rot

    def op_score_feats(self, crops, N):
        feats = torch.empty(N, 512, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_op_score_feats(self._h, _p(crops), N, _p(feats), _stream()), "fp_op_score_feats")
        return feats

    def op_tokens(self, kind, crops, N):
        tok = torch.empty(N, 400, 512, dtype=torch.float16, device="cuda")
        _lib.check(lib.fp_op_tokens(self._h, 0 if kind == "refine" else 1, _p(crops), N, _p(tok), _stream()), "fp_op_tokens")
        return tok


def vis_size(kind, N):
    """(H, W) of Engine.vis's canvas for N hypotheses (no GPU needed)."""
    hw = (C.c_int * 2)()
    _lib.check(lib.fp_vis_size(0 if kind == "refine" else 1, int(N), hw), "fp_vis_size")
    return hw[0], hw[1]


def vis_colormap():
    """The canvases' colour map: (256, 3) uint8 RGB (no GPU needed)."""
    out = np.empty((256, 3), dtype=np.uint8)
    _lib.check(lib.fp_vis_colormap(C.c_void_p(out.ctypes.data)), "fp_vis_colormap")
    return out


def crops_from_planar(A, B):
    """(N,6,160,160) float A, B -> the fp16 padded crop buffer layout [2N][166][2][84][8] (packing.pad_image_c8)."""
    return packing.pad_image_c8(torch.cat([A, B], 0))


def op_depth_filter(depth, which):
    depth = depth.contiguous().float()
    out = torch.empty_like(depth)
    H, W = depth.shape
    _lib.check(lib.fp_op_depth_filter(_p(depth), _p(out), H, W, which, _stream()), "fp_op_depth_filter")
    return out


def op_pose_update(poses, trans, rot, mesh_diameter, rot_normalizer):
    poses = poses.contiguous().float()
    out = torch.empty_like(poses)
    _lib.check(lib.fp_op_pose_update(_p(poses), _p(trans.contiguous().float()), _p(rot.contiguous().float()), _p(out),
                                     len(poses), float(mesh_diameter), float(rot_normalizer), _stream()), "fp_op_pose_update")
    return out
