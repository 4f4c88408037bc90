"""Host-side owner of one `fp_ctx`: packs reference checkpoints for the CUDA kernels and exposes the
hot-path entry points of libfpose.so on torch CUDA tensors.

torch is used for device memory, streams and (in parallel.py) torch.distributed only; every
computation on the hot path happens inside the C-ABI library.
"""
import ctypes as C
import weakref

import numpy as np
import torch

from . import _lib, packing
from ._lib import lib
from .frames import DEFAULT_FORMAT, Color, Depth, depth_sensor, frame_format

CROP_SHAPE = (166, 2, 84, 8)  # padded fp16 crop image consumed by the stem convolution: rows x {even, odd cols} x pairs x ch


class _FpTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("dtype", C.c_int), ("numel", C.c_longlong)]


class _FpFrameFormat(C.Structure):
    _fields_ = [("color", C.c_int), ("depth", C.c_int), ("depth_scale", C.c_float), ("rgb_pitch", C.c_int),
                ("depth_pitch", C.c_int)]


def _proto():
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    lib.fp_create.argtypes = [C.POINTER(vp)]
    lib.fp_destroy.argtypes = [vp]
    lib.fp_set_config.argtypes = [vp, i, f, f]
    lib.fp_mesh_info.argtypes = [vp, C.POINTER(i)]
    lib.fp_set_crop_tile.argtypes = [vp, i]
    lib.fp_set_camera_format.argtypes = [vp, i, C.POINTER(_FpFrameFormat)]
    lib.fp_set_camera_depth_sensor.argtypes = [vp, i, C.POINTER(_lib.DepthSensor)]
    lib.fp_crop_stats.argtypes = [vp, vp, i, i, C.POINTER(i), vp]
    lib.fp_track.argtypes = [vp, vp, vp, C.POINTER(f), i, i, vp, i, vp, vp, vp]
    lib.fp_track_objects.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, C.POINTER(i), vp, i, vp, vp, vp]
    lib.fp_track_cameras.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(f), C.POINTER(i), C.POINTER(i), i, C.POINTER(i),
                                     C.POINTER(i), vp, i, vp, vp, vp]
    lib.fp_register_objects.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, C.POINTER(i), C.POINTER(i), vp, vp, i, vp, vp, vp,
                                        vp, vp]
    lib.fp_register_cameras.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(f), C.POINTER(i), C.POINTER(i), i,
                                        C.POINTER(i), C.POINTER(i), C.POINTER(i), C.POINTER(vp), vp, i, vp, vp, vp, vp, vp]
    lib.fp_track_submit.argtypes = [vp, vp, vp, C.POINTER(f), i, i, vp, i, vp, vp, C.POINTER(C.c_ulonglong)]
    lib.fp_track_objects_submit.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, C.POINTER(i), vp, i, vp, vp,
                                            C.POINTER(C.c_ulonglong)]
    lib.fp_track_cameras_submit.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(f), C.POINTER(i), C.POINTER(i), i,
                                            C.POINTER(i), C.POINTER(i), vp, i, vp, vp, C.POINTER(C.c_ulonglong)]
    lib.fp_track_wait.argtypes = [vp, C.c_ulonglong, vp]
    lib.fp_track_cameras_fit_submit.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(f), C.POINTER(i), C.POINTER(i), i,
                                                C.POINTER(i), C.POINTER(i), vp, i, f, vp, vp, vp, C.POINTER(C.c_ulonglong)]
    lib.fp_track_fit_wait.argtypes = [vp, C.c_ulonglong, vp, vp]
    lib.fp_graph_captures.argtypes = [vp]
    lib.fp_graph_captures.restype = C.c_ulonglong
    lib.fp_load_network.argtypes = [vp, i, C.POINTER(_FpTensor), i]
    lib.fp_set_mesh.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp, i, i, f]
    lib.fp_set_mesh_slot.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp, i, i, f]
    lib.fp_set_frame.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, f, vp]
    lib.fp_get_depth.argtypes = [vp, i, vp, vp, C.POINTER(i), vp]
    lib.fp_set_xyz_map.argtypes = [vp, vp, vp]
    lib.fp_make_crops.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    lib.fp_start_poses.argtypes = [vp, vp, i, vp, i, vp, vp, vp]
    lib.fp_refine.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    lib.fp_score.argtypes = [vp, vp, i, vp, vp, vp]
    lib.fp_score_features.argtypes = [vp, vp, i, vp, vp]
    lib.fp_score_tail.argtypes = [vp, vp, i, vp, vp, vp]
    lib.fp_op_score_tail_segments.argtypes = [vp, vp, i, C.POINTER(i), i, vp, vp, vp]
    lib.fp_register.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    lib.fp_op_refine_net.argtypes = [vp, vp, i, vp, vp, vp]
    lib.fp_op_score_feats.argtypes = [vp, vp, i, vp, vp]
    lib.fp_op_encoder.argtypes = [vp, i, vp, i, i, vp, vp]
    lib.fp_op_encoder.restype = C.c_longlong
    lib.fp_op_heads.argtypes = [vp, i, vp, i, i, vp, vp]
    lib.fp_op_heads.restype = C.c_longlong
    lib.fp_op_encoder_layer.argtypes = [i, i, C.POINTER(i)]
    lib.fp_op_depth_filter.argtypes = [vp, vp, i, i, i, vp]
    lib.fp_op_pose_update.argtypes = [vp, vp, vp, vp, C.POINTER(i), i, vp, vp, vp, vp]
    lib.fp_vis.argtypes = [vp, i, vp, vp, i, vp, vp, C.POINTER(i), vp]
    lib.fp_vis_size.argtypes = [i, i, C.POINTER(i)]
    lib.fp_vis_colormap.argtypes = [vp]
    lib.fp_vis_crops.argtypes = [vp, vp, i, i, vp, vp]
    lib.fp_vis_workspace_bytes.argtypes = [vp]
    lib.fp_vis_workspace_bytes.restype = C.c_ulonglong
    for name in ("fp_create", "fp_destroy", "fp_set_config", "fp_mesh_info", "fp_set_crop_tile", "fp_set_camera_format", "fp_set_camera_depth_sensor", "fp_crop_stats", "fp_track", "fp_track_objects", "fp_track_cameras", "fp_track_submit", "fp_track_objects_submit",
                 "fp_track_cameras_submit", "fp_track_wait", "fp_track_cameras_fit_submit", "fp_track_fit_wait", "fp_register_objects", "fp_register_cameras", "fp_set_xyz_map", "fp_load_network", "fp_set_mesh",
                 "fp_set_mesh_slot", "fp_set_frame",
                 "fp_get_depth", "fp_make_crops", "fp_start_poses", "fp_refine", "fp_score", "fp_score_features", "fp_score_tail",
                 "fp_op_score_tail_segments", "fp_register", "fp_op_refine_net", "fp_op_score_feats", "fp_op_encoder_layer", "fp_op_depth_filter",
                 "fp_op_pose_update", "fp_vis", "fp_vis_size", "fp_vis_colormap", "fp_vis_crops"):
        getattr(lib, name).restype = C.c_int


_proto()

FRAME_ON_DEVICE = 1
MAX_MESHES = 64  # FP_MAX_MESHES: mesh slots per context
MAX_CAMERAS = 16  # FP_MAX_CAMERAS: camera streams per fp_track_cameras / fp_register_cameras call
MAX_IN_FLIGHT = 2  # FP_TRACK_MAX_IN_FLIGHT: tracking calls in flight per context (its staging sets)
FIT_COUNTS = 5  # FP_FIT_COUNTS: covered, valid, inlier, occluded, behind
FRAME_FILTER_DEPTH = 2


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _on_device(x):
    return torch.is_tensor(x) and x.is_cuda


def _ptr(x):
    """Address of a host array or a CUDA tensor."""
    return C.c_void_p(x.data_ptr() if torch.is_tensor(x) else x.ctypes.data)


def _check_wrapped_device(x, what, device):
    if _on_device(x.img) and device is not None and x.img.device.index != device:
        raise ValueError(f"{what}: {type(x).__name__} is a CUDA tensor on device {x.img.device.index}, the engine's is {device}")


def _frame(rgb, depth, what, device=None):
    """One camera's frame as the tracking and register calls take it: (rgb, depth, (H, W), format, sensor).  Each buffer
    is a host array (made a contiguous uint8 / float32 numpy array, staged by the library) or a CUDA tensor on the
    engine's device, read in place in stream order: rgb uint8 (H,W,3), depth (H,W) converted to float32, both made
    contiguous.  A Color / Depth (frames.py) is taken as it is, in its own layout, wherever it lives; format is the camera
    format of the pair (frames.frame_format), sensor its depth sensor (frames.depth_sensor).  (H, W) is the colour
    frame's: with a depth sensor the depth image has the sensor's own size."""
    fmt, sensor = frame_format(rgb, depth), depth_sensor(depth)
    if isinstance(depth, Depth):
        _check_wrapped_device(depth, what, device)
        H, W = depth.H, depth.W
        depth = depth.img
        if sensor is not None:  # the frame is the colour camera's
            H, W = (rgb.H, rgb.W) if isinstance(rgb, Color) else tuple(rgb.shape if torch.is_tensor(rgb) else np.shape(rgb))[:2]
    elif _on_device(depth):
        if depth.dim() != 2:
            raise ValueError(f"{what}: depth must be (H, W), got {tuple(depth.shape)}")
        depth = depth.contiguous().float()
        H, W = depth.shape
    else:
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        H, W = depth.shape
    if isinstance(rgb, Color):
        _check_wrapped_device(rgb, what, device)
        if (rgb.H, rgb.W) != (H, W):  # with a sensor (H, W) is the colour frame's already
            raise ValueError(f"{what}: the colour frame is {rgb.H} x {rgb.W}, the depth frame {H} x {W}")
        rgb = rgb.img
    elif _on_device(rgb):
        if rgb.dtype != torch.uint8:
            raise ValueError(f"{what}: a CUDA rgb frame must be uint8, got {rgb.dtype}")
        if tuple(rgb.shape) != (H, W, 3):
            raise ValueError(f"{what}: rgb must be ({H}, {W}, 3) to match depth, got {tuple(rgb.shape)}")
        rgb = rgb.contiguous()
    else:
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    return rgb, depth, (int(H), int(W)), fmt, sensor


def _device_mask(m):
    """A CUDA mask (bool, uint8 or float) as the library reads it: contiguous uint8, 1 where `m > 0` (the reference's
    test, estimater.py:138, :183), binarised on the device."""
    return (m > 0).to(torch.uint8).contiguous()


def _hold(bufs):
    """The CUDA tensors among `bufs`, each recorded on the current stream: the library reads them in that stream's order,
    so the caching allocator must not hand their memory to another stream before it has passed the call."""
    held = [b for b in bufs if _on_device(b)]
    st = torch.cuda.current_stream()
    for b in held:
        b.record_stream(st)
    return held


def _camera_args(frames, hw=None):
    """The (rgb pointers, depth pointers, K [C][9], H, W) arguments of the multi-camera calls for (rgb, depth, K) frames
    whose buffers _frame made.  hw: each camera's colour frame size (H, W) as _frame gives it; None: the depth's shape
    (no camera has a depth sensor)."""
    n_cam = len(frames)
    hw = [tuple(depth.shape[:2]) for _, depth, _ in frames] if hw is None else hw
    rgbs = (C.c_void_p * n_cam)(*[_ptr(rgb).value for rgb, _, _ in frames])
    depths = (C.c_void_p * n_cam)(*[_ptr(depth).value for _, depth, _ in frames])
    Ks = (C.c_float * (9 * n_cam))(*[float(x) for _, _, K in frames for x in np.asarray(K, dtype=np.float64).reshape(-1)])
    Hs = (C.c_int * n_cam)(*[int(h) for h, _ in hw])
    Ws = (C.c_int * n_cam)(*[int(w) for _, w in hw])
    return rgbs, depths, Ks, Hs, Ws


# ---------------------------------------------------------------------------------------------
# checkpoint -> packed tensors
# ---------------------------------------------------------------------------------------------
def _bn_of(sd, prefix):
    if f"{prefix}.weight" not in sd:
        return None
    return {"weight": sd[f"{prefix}.weight"], "bias": sd[f"{prefix}.bias"], "running_mean": sd[f"{prefix}.running_mean"],
            "running_var": sd[f"{prefix}.running_var"], "eps": 1e-5}


def encoder_convs(kind):
    """State-dict prefixes (convolution, batch norm) of encoder layers 0..14, packed as "enc.<layer>.w" / ".b"."""
    A, AB = ("encodeA", "encodeAB") if kind == "refine" else ("encoderA", "encoderAB")
    return [(f"{A}.0.net.0", f"{A}.0.net.1"), (f"{A}.1.net.0", f"{A}.1.net.1"),
            (f"{A}.2.conv1", f"{A}.2.bn1"), (f"{A}.2.conv2", f"{A}.2.bn2"),
            (f"{A}.3.conv1", f"{A}.3.bn1"), (f"{A}.3.conv2", f"{A}.3.bn2"),
            (f"{AB}.0.conv1", f"{AB}.0.bn1"), (f"{AB}.0.conv2", f"{AB}.0.bn2"),
            (f"{AB}.1.conv1", f"{AB}.1.bn1"), (f"{AB}.1.conv2", f"{AB}.1.bn2"),
            (f"{AB}.2.net.0", f"{AB}.2.net.1"),
            (f"{AB}.3.conv1", f"{AB}.3.bn1"), (f"{AB}.3.conv2", f"{AB}.3.bn2"),
            (f"{AB}.4.conv1", f"{AB}.4.bn1"), (f"{AB}.4.conv2", f"{AB}.4.bn2")]


def pack_network(sd, kind):
    """Reference state_dict (learning/models/{refine,score}_network.py layout) -> {name: np.ndarray}."""
    out = {}
    for i, (cname, bname) in enumerate(encoder_convs(kind)):
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


def _tensor_array(packed):
    """{name: np.ndarray} -> (fp_tensor_t array, the arrays it points into: keep them alive until the call returns)."""
    arr = (_FpTensor * len(packed))()
    keep = []
    for i, (name, a) in enumerate(packed.items()):
        a = np.ascontiguousarray(a)
        keep.append(a)
        arr[i] = _FpTensor(name.encode(), a.ctypes.data, 1 if a.dtype == np.float16 else 0, a.size)
    return arr, keep


def _mesh_args(vertices, normals, faces, uv=None, tex=None, vertex_colors=None):
    """The (V, F, pos, nrm, uv, vcol, faces, tex_rgb, Ht, Wt) arguments of fp_set_mesh*, and the arrays the pointers point
    into: keep them alive until the call returns."""
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
    keep = (pos, nrm, uvp, colp, fc, texp)
    return (len(pos), len(fc), cp(pos), cp(nrm), cp(uvp), cp(colp), cp(fc), cp(texp), Ht, Wt), keep


class PendingPoses:
    """The host poses of one tracking call submitted with wait=False.  result() waits for the call's read-back (once; later
    calls return the same result) and returns what the blocking call returns as its host poses: the poses array, or for a
    call with a fit (track_cameras(..., fit_delta=)) the tuple (poses, fit counts (M, FIT_COUNTS) int32).  A handle
    dropped without result() is collected by its engine at a later submit or at close, so its ticket never leaks.  It
    holds the call's device frames until result() has collected the call."""

    def __init__(self, engine, ticket, shape, held=(), fit=False):
        self._engine, self.ticket, self._shape, self._host, self._held = engine, ticket, shape, None, list(held)
        self._fit = fit
        self._dropped = weakref.finalize(self, engine._dropped.append, ticket)

    def result(self):
        if self._host is None:
            self._dropped.detach()
            host = np.empty(self._shape, dtype=np.float32)
            if self._fit:
                self._host = (host, self._engine._wait_fit(self.ticket, host))
            else:
                self._engine._wait(self.ticket, host)
                self._host = host
            self._held = []
        return self._host


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
        self._dropped = []  # tickets of PendingPoses dropped without result()
        self._last_ticket = 0
        self._formats = [DEFAULT_FORMAT] * MAX_CAMERAS  # the frame format the context holds for each camera
        self._sensors = [None] * MAX_CAMERAS  # the depth sensor the context holds for each camera (frames.depth_sensor)

    def close(self):
        if getattr(self, "_h", None):
            self._collect_dropped(0)
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
        arr, keep = _tensor_array(pack_network(state_dict, kind))
        _lib.check(lib.fp_load_network(self._h, 0 if kind == "refine" else 1, arr, len(arr)), "fp_load_network")

    def set_mesh(self, vertices, normals, faces, diameter, uv=None, tex=None, vertex_colors=None, slot=0):
        """uv: (V,2) with v already flipped (Utils.py:117); tex: uint8 (Ht,Wt,3); vertex_colors: float 0..1.
        slot: 0..MAX_MESHES-1; slot 0 is the mesh of every single-object call, the others are for track_objects."""
        args, keep = _mesh_args(vertices, normals, faces, uv, tex, vertex_colors)
        _lib.check(lib.fp_set_mesh_slot(self._h, int(slot), *args, float(diameter)), "fp_set_mesh")
        if slot == 0:
            self.diameter = float(diameter)
            self.mesh_key = (args[0], args[1], float(diameter))

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

    def _set_formats(self, fmts, sensors=None):
        """fp_set_camera_format for camera i = 0, 1, ... wherever fmts[i] differs from the format the context holds, and
        fp_set_camera_depth_sensor wherever sensors[i] (frames.depth_sensor; None: every camera without) differs from
        the sensor it holds."""
        for i, f in enumerate(fmts):
            if self._formats[i] != f:
                ff = _FpFrameFormat(*f)
                _lib.check(lib.fp_set_camera_format(self._h, i, C.byref(ff)), "fp_set_camera_format")
                self._formats[i] = f
        for i, sn in enumerate(sensors if sensors is not None else [None] * len(fmts)):
            if self._sensors[i] != sn:
                rec = None if sn is None else C.byref(_lib.DepthSensor.of(*sn))
                _lib.check(lib.fp_set_camera_depth_sensor(self._h, i, rec), "fp_set_camera_depth_sensor")
                self._sensors[i] = sn

    # ---- tracking: every call is a submit and, with wait=True, its fp_track_wait
    def _collect_dropped(self, keep):
        """Collects the dropped handles' tickets except those of the last `keep` submits (still running, most likely)."""
        for t in [t for t in self._dropped if t <= self._last_ticket - keep]:
            self._dropped.remove(t)
            _lib.check(lib.fp_track_wait(self._h, t, None), "fp_track_wait")

    def _submit(self, fn, args, what, out, shape, wait, bufs=(), fit=False):
        """Submits one tracking call (`fn(ctx, *args, stream, &ticket)`) on the frame buffers `bufs`.  Returns (out, host
        poses) with wait, else (out, PendingPoses), which holds the device buffers among `bufs` until it is collected.
        fit: a call with a fit, whose host result is (poses, counts)."""
        if not getattr(self, "_h", None):
            raise _lib.FposeError(f"{what}: the engine is closed")
        self._collect_dropped(MAX_IN_FLIGHT)
        ticket = C.c_ulonglong()
        _lib.check(fn(self._h, *args, _stream(), C.byref(ticket)), what)
        self._last_ticket = ticket.value
        if not wait:
            return out, PendingPoses(self, ticket.value, shape, _hold(bufs), fit)
        host = np.empty(shape, dtype=np.float32)
        if fit:
            return out, (host, self._wait_fit(ticket.value, host))
        self._wait(ticket.value, host)
        return out, host

    def _wait(self, ticket, host):
        if not getattr(self, "_h", None):
            raise _lib.FposeError("fp_track_wait: the engine is closed")
        _lib.check(lib.fp_track_wait(self._h, ticket, C.c_void_p(host.ctypes.data)), "fp_track_wait")

    def _wait_fit(self, ticket, host):
        """fp_track_fit_wait: the poses into `host` (M,4,4); returns the counts (M, FIT_COUNTS) int32."""
        if not getattr(self, "_h", None):
            raise _lib.FposeError("fp_track_fit_wait: the engine is closed")
        counts = np.empty((host.shape[0], FIT_COUNTS), dtype=np.int32)
        _lib.check(lib.fp_track_fit_wait(self._h, ticket, C.c_void_p(host.ctypes.data), C.c_void_p(counts.ctypes.data)),
                   "fp_track_fit_wait")
        return counts

    def track(self, rgb, depth, K, pose_in, iterations, pose_out=None, wait=True):
        """fp_track: one CUDA-graph launch per frame (upload + depth filters + xyz map + refiner passes + read-back).
        rgb uint8 (H,W,3) / depth float32 (H,W): host arrays, or CUDA tensors on the engine's device, read in place in the
        current stream's order (see _frame), or a Color / Depth (frames.py) in a sensor's own layout, host or device;
        pose_in (4,4) CUDA tensor or None (continue).
        Returns (pose_out CUDA (4,4), pose host (4,4) float32 numpy).  wait=False returns as soon as the call is
        submitted (the host arrays may then be reused): (pose_out, PendingPoses), pose_out complete in stream order."""
        rgb, depth, (H, W), fmt, sensor = _frame(rgb, depth, "track", self.device_index)
        Kf = (C.c_float * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        self._set_formats([fmt], [sensor])
        if pose_in is not None:
            pose_in = pose_in.reshape(4, 4).contiguous().float()
        if pose_out is None:
            pose_out = torch.empty(4, 4, dtype=torch.float32, device="cuda")
        out = self._submit(lib.fp_track_submit, (_ptr(rgb), _ptr(depth), Kf, H, W, _p(pose_in), int(iterations), _p(pose_out)),
                           "fp_track", pose_out, (4, 4), wait, (rgb, depth))
        self.frame_hw = (H, W)
        return out

    def track_objects(self, rgb, depth, K, poses_in, slots, iterations, wait=True):
        """fp_track_objects: `track` for M objects of one frame in ONE CUDA-graph launch, object i rendering the mesh in
        slot slots[i] (loaded by set_mesh(..., slot=)).  rgb uint8 (H,W,3) / depth float32 (H,W): host arrays or CUDA
        tensors, as `track`; poses_in (M,4,4) CUDA tensor.  Returns (poses CUDA (M,4,4), poses host (M,4,4) float32
        numpy); wait=False as `track`."""
        rgb, depth, (H, W), fmt, sensor = _frame(rgb, depth, "track_objects", self.device_index)
        Kf = (C.c_float * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        poses_in = poses_in.reshape(-1, 4, 4).contiguous().float()
        M = len(poses_in)
        slots = [int(s) for s in slots]
        if len(slots) != M:
            raise ValueError(f"track_objects: {M} poses but {len(slots)} slots")
        self._set_formats([fmt], [sensor])
        out = torch.empty(M, 4, 4, dtype=torch.float32, device="cuda")
        res = self._submit(lib.fp_track_objects_submit, (_ptr(rgb), _ptr(depth), Kf, H, W, M, (C.c_int * M)(*slots), _p(poses_in),
                                                         int(iterations), _p(out)),
                           "fp_track_objects", out, (M, 4, 4), wait, (rgb, depth))
        self.frame_hw = (H, W)
        return res

    def track_cameras(self, frames, poses_in, camera_of, slots, iterations, wait=True, fit_delta=None):
        """fp_track_cameras: `track_objects` for M objects spread over C camera streams in ONE CUDA-graph launch.  frames: C
        tuples (rgb uint8 (H,W,3), depth float32 (H,W), K (3,3)), one per camera, each with its own size and intrinsics and
        each buffer a host array, a CUDA tensor or a Color / Depth, as `track` (one call may mix them, and each camera has
        its own format); object i is seen by camera
        camera_of[i] and renders the mesh in slot slots[i]; poses_in (M,4,4) CUDA tensor.  Returns (poses CUDA (M,4,4),
        poses host (M,4,4) float32 numpy); wait=False as `track`.

        fit_delta (metres): also count, in the same launch, how well each returned pose's rendered depth agrees with the
        observed depth (fp_track_cameras_fit_submit, include/fpose.h): returns (poses CUDA, poses host, fit) with fit an
        int32 (M, FIT_COUNTS) numpy array of (covered, valid, inlier, occluded, behind) pixels; wait=False returns
        (poses CUDA, PendingPoses) whose result() gives (poses host, fit).  The poses are those of the call without it."""
        made = [(_frame(rgb, depth, f"track_cameras: camera {c}", self.device_index), K) for c, (rgb, depth, K) in enumerate(frames)]
        frames = [(f[0], f[1], K) for f, K in made]
        hw = [f[2] for f, _ in made]  # each camera's colour frame size
        n_cam = len(frames)
        poses_in = poses_in.reshape(-1, 4, 4).contiguous().float()
        M = len(poses_in)
        camera_of, slots = [int(c) for c in camera_of], [int(s) for s in slots]
        if len(camera_of) != M or len(slots) != M:
            raise ValueError(f"track_cameras: {M} poses, {len(camera_of)} camera ids and {len(slots)} slots")
        if n_cam <= MAX_CAMERAS:  # more cameras: fp_track_cameras refuses the call
            self._set_formats([f[3] for f, _ in made], [f[4] for f, _ in made])
        rgbs, depths, Ks, Hs, Ws = _camera_args(frames, hw)
        out = torch.empty(M, 4, 4, dtype=torch.float32, device="cuda")
        ids = (n_cam, rgbs, depths, Ks, Hs, Ws, M, (C.c_int * M)(*camera_of), (C.c_int * M)(*slots), _p(poses_in), int(iterations))
        bufs = [b for rgb, depth, _ in frames for b in (rgb, depth)]
        if fit_delta is None:
            res = self._submit(lib.fp_track_cameras_submit, (*ids, _p(out)), "fp_track_cameras", out, (M, 4, 4), wait, bufs)
        else:
            res = self._submit(lib.fp_track_cameras_fit_submit, (*ids, float(fit_delta), _p(out), None), "fp_track_cameras_fit",
                               out, (M, 4, 4), wait, bufs, fit=True)
            if wait:
                res = (res[0], *res[1])
        self.frame_hw = hw[0]  # camera 0's frame is the context's frame
        return res

    def register_objects(self, rgb, depth, K, masks, rot_grids, slots, iterations):
        """fp_register_objects: the register() hot path for M objects of one frame in one call, object i rendering the mesh
        in slot slots[i].  rgb uint8 (H,W,3) / depth float32 (H,W): host arrays, CUDA tensors or a Color / Depth, as
        `track`; masks
        (M,H,W) (nonzero = object): a host array, or a CUDA bool / uint8 / float tensor (or a sequence of M CUDA (H,W)
        masks) binarised on the device; rot_grids: M CUDA float32 (N_i,4,4) rotation grids.  Returns CUDA tensors: poses
        (sum N_i,4,4) refined, object-major and unranked; scores (sum N_i,); best (M,) int32, each object's first arg-max
        relative to its own rows; info (M,4) = (tx, ty, tz, n_valid) per object."""
        rgb, depth, (H, W), fmt, sensor = _frame(rgb, depth, "register_objects", self.device_index)
        if not _on_device(masks) and len(masks) and all(_on_device(m) for m in masks):
            masks = torch.stack(list(masks))
        masks = masks if _on_device(masks) else np.ascontiguousarray(masks)
        M = len(masks)
        if tuple(masks.shape) != (M, H, W):
            raise ValueError(f"register_objects: masks must be (M, {H}, {W}), got {tuple(masks.shape)}")
        if _on_device(masks):
            masks = _device_mask(masks)
        else:
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
        self._set_formats([fmt], [sensor])
        _lib.check(lib.fp_register_objects(self._h, _ptr(rgb), _ptr(depth), Kf, H, W, M, (C.c_int * M)(*slots), (C.c_int * M)(*n_hyp),
                                           _ptr(masks), _p(grids), int(iterations), _p(poses), _p(scores), _p(best), _p(info),
                                           _stream()),
                   "fp_register_objects")  # synchronises its stream: the device inputs are free again on return
        self.frame_hw = (H, W)
        return poses, scores, best, info

    def register_cameras(self, frames, masks, rot_grids, camera_of, slots, iterations):
        """fp_register_cameras: `register_objects` for M objects spread over C camera streams in one call.  frames: C tuples
        (rgb uint8 (H,W,3), depth float32 (H,W), K (3,3)), one per camera, each with its own size and intrinsics and each
        buffer a host array, a CUDA tensor or a Color / Depth, as `track_cameras`; object i is seen by camera camera_of[i], renders the mesh in slot
        slots[i] and has the mask masks[i] (nonzero = object) of its camera's frame size, a host array or a CUDA bool /
        uint8 / float tensor binarised on the device; rot_grids: M CUDA float32 (N_i,4,4) rotation grids.
        Returns the CUDA tensors of register_objects: poses (sum N_i,4,4), scores (sum N_i,), best (M,), info (M,4)."""
        made = [(_frame(rgb, depth, f"register_cameras: camera {c}", self.device_index), K) for c, (rgb, depth, K) in enumerate(frames)]
        frames = [(f[0], f[1], K) for f, K in made]
        hw = [f[2] for f, _ in made]  # each camera's colour frame size
        n_cam = len(frames)
        M = len(masks)
        camera_of, slots = [int(c) for c in camera_of], [int(s) for s in slots]
        rot_grids = [g.reshape(-1, 4, 4) for g in rot_grids]
        if len(camera_of) != M or len(slots) != M or len(rot_grids) != M:
            raise ValueError(f"register_cameras: {M} masks, {len(camera_of)} camera ids, {len(slots)} slots and "
                             f"{len(rot_grids)} rotation grids")
        masks = [m if _on_device(m) else np.asarray(m) for m in masks]
        for i, (m, c) in enumerate(zip(masks, camera_of)):
            if 0 <= c < n_cam and tuple(m.shape) != hw[c]:
                raise ValueError(f"register_cameras: mask {i} has shape {tuple(m.shape)}, camera {c}'s frame is "
                                 f"{hw[c]}")
        # the reference tests `mask > 0` (estimater.py:138, :183)
        masks = [_device_mask(m) if _on_device(m) else np.ascontiguousarray(m > 0, dtype=np.uint8) for m in masks]
        n_hyp = [len(g) for g in rot_grids]
        grids = torch.cat(rot_grids).to(device="cuda", dtype=torch.float32).contiguous()
        total = len(grids)
        rgbs, depths, Ks, Hs, Ws = _camera_args(frames, hw)
        poses = torch.empty(total, 4, 4, dtype=torch.float32, device="cuda")
        scores = torch.empty(total, dtype=torch.float32, device="cuda")
        best = torch.empty(M, dtype=torch.int32, device="cuda")
        info = torch.empty(M, 4, dtype=torch.float32, device="cuda")
        if n_cam <= MAX_CAMERAS:  # more cameras: fp_register_cameras refuses the call
            self._set_formats([f[3] for f, _ in made], [f[4] for f, _ in made])
        _lib.check(lib.fp_register_cameras(self._h, n_cam, rgbs, depths, Ks, Hs, Ws, M, (C.c_int * M)(*camera_of),
                                           (C.c_int * M)(*slots), (C.c_int * M)(*n_hyp), (C.c_void_p * M)(*[_ptr(m).value for m in masks]),
                                           _p(grids), int(iterations), _p(poses), _p(scores), _p(best), _p(info), _stream()),
                   "fp_register_cameras")  # synchronises its stream: the device inputs are free again on return
        self.frame_hw = hw[0]  # camera 0's frame is the context's frame
        return poses, scores, best, info

    def set_frame(self, rgb, depth, K, filter_depth=True, zfar=float("inf")):
        """rgb uint8 (H,W,3), depth float32 (H,W): numpy / CPU tensors or CUDA tensors, or a Color / Depth (frames.py) in
        a sensor's own layout, both on the host or both on the device.  Pageable host frames are staged by the library and
        may be reused once this returns."""
        Kf = (C.c_float * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        flags = FRAME_FILTER_DEPTH if filter_depth else 0
        fmt, sensor = DEFAULT_FORMAT, None
        if isinstance(rgb, Color) or isinstance(depth, Depth):
            rgb, depth, (H, W), fmt, sensor = _frame(rgb, depth, "set_frame", self.device_index)
            if _on_device(rgb) != _on_device(depth):
                raise ValueError("set_frame: rgb and depth must both be CUDA tensors or both be on the host")
            if _on_device(rgb):
                flags |= FRAME_ON_DEVICE
            else:
                rgb, depth = (x if torch.is_tensor(x) else torch.from_numpy(x) for x in (rgb, depth))
        elif torch.is_tensor(rgb) and rgb.is_cuda:
            assert torch.is_tensor(depth) and depth.is_cuda
            rgb = rgb.contiguous()
            depth = depth.contiguous().float()
            assert rgb.dtype == torch.uint8
            flags |= FRAME_ON_DEVICE
        else:
            rgb = rgb if torch.is_tensor(rgb) else torch.from_numpy(np.ascontiguousarray(rgb, dtype=np.uint8))
            depth = depth if torch.is_tensor(depth) else torch.from_numpy(np.ascontiguousarray(depth, dtype=np.float32))
            rgb = rgb.contiguous()
            depth = depth.contiguous()
            assert rgb.dtype == torch.uint8 and depth.dtype == torch.float32
        if sensor is None:
            H, W = depth.shape
        # device and page-locked frames are read in place after the call returns, in stream order: keep them until then
        in_place = rgb.is_cuda or (rgb.is_pinned() and depth.is_pinned())
        self._frame_keep = (rgb, depth) if in_place else None
        self._set_formats([fmt], [sensor])
        _lib.check(lib.fp_set_frame(self._h, _p(rgb), _p(depth), Kf, H, W, flags, float(zfar), _stream()), "fp_set_frame")
        self.frame_hw = (H, W)

    def set_xyz_map(self, xyz_map):
        """Caller-supplied xyz map (H,W,3) float32 — numpy / CPU tensor / CUDA tensor — instead of the derived one."""
        x = xyz_map if torch.is_tensor(xyz_map) else torch.from_numpy(np.ascontiguousarray(xyz_map, dtype=np.float32))
        x = x.float().contiguous()
        assert tuple(x.shape) == (*self.frame_hw, 3), "xyz_map must be (H, W, 3)"
        self._xyz_keep = x
        _lib.check(lib.fp_set_xyz_map(self._h, _p(x), _stream()), "fp_set_xyz_map")

    def get_depth(self, camera=0):
        """Camera `camera`'s filtered depth (H,W) and xyz map (H,W,3) as the last frame-taking call prepared them, at that
        camera's size (test hook).  Cameras 1.. exist after track_cameras / register_cameras only."""
        hw = (C.c_int * 2)()
        _lib.check(lib.fp_get_depth(self._h, int(camera), None, None, hw, _stream()), "fp_get_depth")
        H, W = hw[0], hw[1]
        d = torch.empty(H, W, dtype=torch.float32, device="cuda")
        x = torch.empty(H, W, 3, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_get_depth(self._h, int(camera), _p(d), _p(x), None, _stream()), "fp_get_depth")
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
        # a device mask is read after the call returns, in stream order; the library stages a host mask (a new,
        # pageable tensor) before it returns
        self._mask_keep = m if on_dev else None
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

    def score_tail_segments(self, feats, seg, scores=None, best=None):
        """fp_op_score_tail_segments: the register calls' segmented tail on given features (test hook).  feats (L,512)
        CUDA; seg: the n_seg + 1 row offsets (0, ..., L).  Returns scores (L,) = logits + 100 and best (n_seg,) int32,
        each segment's first arg-max relative to its first row, written into `scores` / `best` when given."""
        feats = feats.contiguous().float()
        L = feats.shape[0]
        seg = [int(s) for s in seg]
        n_seg = len(seg) - 1
        scores = torch.empty(L, dtype=torch.float32, device="cuda") if scores is None else scores
        best = torch.empty(max(n_seg, 1), dtype=torch.int32, device="cuda") if best is None else best
        _lib.check(lib.fp_op_score_tail_segments(self._h, _p(feats), L, (C.c_int * len(seg))(*seg), n_seg, _p(scores), _p(best),
                                                 _stream()), "fp_op_score_tail_segments")
        return scores, best

    def register_host(self, poses_host, iterations, out_poses=None, out_scores=None):
        """fp_register: host buffers in and out (synchronous)."""
        poses_host = poses_host if torch.is_tensor(poses_host) else torch.from_numpy(np.ascontiguousarray(poses_host, dtype=np.float32))
        poses_host = poses_host.reshape(-1, 4, 4).contiguous()
        N = len(poses_host)
        out_poses = torch.empty(N, 4, 4, dtype=torch.float32) if out_poses is None else out_poses
        out_scores = torch.empty(N, dtype=torch.float32) if out_scores is None else out_scores
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

    def op_pose_update(self, poses, trans, rot, mesh_of=None):
        """fp_op_pose_update: one refine-loop pose update, hypothesis n scaled by the half-diameter of the mesh in slot
        mesh_of[n] (None = slot 0) and rotated with the context's rot_normalizer.  Returns the new poses (N,4,4), the
        translation deltas (N,3) and the rotation deltas (N,3,3), CUDA float32."""
        poses = self._poses(poses)
        N = len(poses)
        out = torch.empty_like(poses)
        td = torch.empty(N, 3, dtype=torch.float32, device="cuda")
        rd = torch.empty(N, 3, 3, dtype=torch.float32, device="cuda")
        ids = None if mesh_of is None else (C.c_int * N)(*[int(m) for m in mesh_of])
        _lib.check(lib.fp_op_pose_update(self._h, _p(poses), _p(trans.contiguous().float()), _p(rot.contiguous().float()), ids, N,
                                         _p(out), _p(td), _p(rd), _stream()), "fp_op_pose_update")
        return out, td, rd

    def op_score_feats(self, crops, N):
        feats = torch.empty(N, 512, dtype=torch.float32, device="cuda")
        _lib.check(lib.fp_op_score_feats(self._h, _p(crops), N, _p(feats), _stream()), "fp_op_score_feats")
        return feats

    def op_encoder(self, kind, crops, N, last=14):
        """fp_op_encoder: encoder layers 0..last of network `kind` on the crops ((2N, *CROP_SHAPE) fp16 CUDA) -> layer
        last's whole output buffer, fp16 NHWC (images, H, W, C) as encoder_layer(last, N)["out_shape"]: all Np + N
        images for layers 0-4, (N, 40, 40, 256) for layer 5, the tokens (N, 20, 20, 512) for layer 14."""
        out = torch.empty(*encoder_layer(last, N)["out_shape"], dtype=torch.float16, device="cuda")
        if N == 0:
            return out
        rc = lib.fp_op_encoder(self._h, 0 if kind == "refine" else 1, _p(crops), int(N), int(last), _p(out), _stream())
        _lib.check(rc if rc < 0 else 0, "fp_op_encoder")
        assert rc == out.numel() * out.element_size(), f"fp_op_encoder copied {rc} bytes into a {tuple(out.shape)} buffer"
        return out

    # fp_op_heads: the buffer each stage leaves, as (dtype, shape at N hypotheses of 400 tokens)
    HEAD_STAGES = {
        "refine": [(torch.float16, lambda N: (N * 400, 3072))]
        + [(torch.float16, lambda N: (2, N * 400, 512))] * 5 + [(torch.float32, lambda N: (2, N, 3))],
        "score": [(torch.float16, lambda N: (N * 400, 1536)), (torch.float16, lambda N: (N * 400, 512)),
                  (torch.float32, lambda N: (N, 512)), (torch.float32, lambda N: (N, 512))],
    }

    def op_heads(self, kind, tok, N, stage):
        """fp_op_heads: the heads of network `kind` (run_refine_heads / run_score_feats) on the tokens (fp16 CUDA, N x 400
        x 512 contiguous) -> the buffer of stage `stage`.  Refiner: 0 qkv (M, 3072), 1 att, 2 x1pre, 3 x1, 4 ff, 5 x2pre
        (each (2, M, 512) fp16, one block per head), 6 head_out (2, N, 3) fp32; scorer: 0 qkv (M, 1536), 1 att (M, 512),
        2 the token mean of att (N, 512) fp32, 3 the features (N, 512) fp32.  M = 400 N."""
        stages = self.HEAD_STAGES[kind]
        if not 0 <= stage < len(stages):
            raise ValueError(f"op_heads: {kind} has stages 0..{len(stages) - 1}, not {stage}")
        assert tok.dtype == torch.float16 and tok.is_contiguous() and tok.numel() == N * 400 * 512
        dtype, shape = stages[stage]
        out = torch.empty(*shape(N), dtype=dtype, device="cuda")
        rc = lib.fp_op_heads(self._h, 0 if kind == "refine" else 1, _p(tok), int(N), int(stage), _p(out), _stream())
        _lib.check(rc if rc < 0 else 0, "fp_op_heads")
        assert rc == out.numel() * out.element_size(), f"fp_op_heads copied {rc} bytes into a {tuple(out.shape)} buffer"
        return out

    def op_tokens(self, kind, crops, N):
        """The encoder's tokens, fp16 (N, 400, 512): op_encoder(kind, crops, N) with the 20 x 20 token grid flattened."""
        return self.op_encoder(kind, crops, N).reshape(N, 400, 512)


def vis_size(kind, N):
    """(H, W) of Engine.vis's canvas for N hypotheses (no GPU needed)."""
    hw = (C.c_int * 2)()
    _lib.check(lib.fp_vis_size(0 if kind == "refine" else 1, int(N), hw), "fp_vis_size")
    return hw[0], hw[1]


def encoder_layer(k, N):
    """Encoder layer k (0..14) at N hypotheses, from the layer table run_encoder runs (no GPU needed): dict(kind,
    n_img (images the layer launches on), H (input height = width), Cin, Cout, src (the layer whose output is its
    input, -1 = the crops), res (the layer whose output it adds, -1 = none), out_split, pe (adds the positional
    embedding), out_shape (images, H, W, C) of its output buffer)."""
    info = (C.c_int * 13)()
    _lib.check(lib.fp_op_encoder_layer(int(k), int(N), info), "fp_op_encoder_layer")
    return dict(kind=info[0], n_img=info[1], H=info[2], Cin=info[3], Cout=info[4], src=info[5], res=info[6],
                out_split=info[7], pe=bool(info[8]), out_shape=tuple(info[9:13]))


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

