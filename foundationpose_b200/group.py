"""One process driving several GPUs (`fp_group`, include/fpose.h): the sharded register of BASELINE.json configs[3]
without torch.distributed — the reference's process model is a single script (run_demo.py), so this is what lets an
unmodified driver use all the GPUs of a box.  The only exchange is each device writing its per-hypothesis feature rows
and refined poses straight into device 0's buffers over NVLink peer memory.

    grp = EngineGroup(range(torch.cuda.device_count()))
    grp.load_network("refine", sd_r); grp.load_network("score", sd_s); grp.set_mesh(...)
    poses, scores, best, info = grp.register(rgb, depth, K, mask, rot_grid, iterations=5)
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import lib
from .engine import _FpTensor, _mesh_args, _tensor_array, pack_network

vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
lib.fp_group_create.argtypes = [i32, C.POINTER(i32), C.POINTER(vp)]
lib.fp_group_destroy.argtypes = [vp]
lib.fp_group_size.argtypes = [vp]
lib.fp_group_ctx.argtypes = [vp, i32]
lib.fp_group_ctx.restype = vp
lib.fp_group_load_network.argtypes = [vp, i32, C.POINTER(_FpTensor), i32]
lib.fp_group_set_config.argtypes = [vp, i32, f32, f32]
lib.fp_group_set_mesh.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, i32, i32, f32]
lib.fp_group_register.argtypes = [vp, vp, vp, C.POINTER(f32), i32, i32, vp, vp, i32, i32, vp, vp, vp, vp]
for _n in ("fp_group_create", "fp_group_destroy", "fp_group_size", "fp_group_load_network", "fp_group_set_config", "fp_group_set_mesh",
           "fp_group_register"):
    getattr(lib, _n).restype = C.c_int


class EngineGroup:
    def __init__(self, device_ids):
        ids = [int(d) for d in device_ids]
        arr = (i32 * len(ids))(*ids)
        h = vp()
        _lib.check(lib.fp_group_create(len(ids), arr, C.byref(h)), "fp_group_create")
        self._h = h
        self.device_ids = ids

    def close(self):
        if getattr(self, "_h", None):
            lib.fp_group_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return len(self.device_ids)

    def load_network(self, kind, state_dict):
        arr, keep = _tensor_array(pack_network(state_dict, kind))
        _lib.check(lib.fp_group_load_network(self._h, 0 if kind == "refine" else 1, arr, len(arr)), "fp_group_load_network")

    def set_config(self, kind, crop_ratio=1.2, rot_normalizer=0.3490658503988659):
        _lib.check(lib.fp_group_set_config(self._h, 0 if kind == "refine" else 1, float(crop_ratio), float(rot_normalizer)), "fp_group_set_config")

    def set_mesh(self, vertices, normals, faces, diameter, uv=None, tex=None, vertex_colors=None):
        args, keep = _mesh_args(vertices, normals, faces, uv, tex, vertex_colors)
        _lib.check(lib.fp_group_set_mesh(self._h, *args, float(diameter)), "fp_group_set_mesh")

    def register(self, rgb, depth, K, mask, rot_grid, iterations=5):
        """HOST numpy in, HOST numpy out: refined poses (N,4,4), scores (N,), best index, info (tx, ty, tz, n_valid)."""
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        m = np.ascontiguousarray(np.asarray(mask) > 0, dtype=np.uint8)
        grid = np.ascontiguousarray(rot_grid, dtype=np.float32).reshape(-1, 16)
        H, W = depth.shape
        N = len(grid)
        Kf = (f32 * 9)(*[float(x) for x in np.asarray(K, dtype=np.float64).reshape(-1)])
        poses = np.empty((N, 4, 4), dtype=np.float32)
        scores = np.empty(N, dtype=np.float32)
        best = np.zeros(1, dtype=np.int32)
        info = np.zeros(4, dtype=np.float32)
        c = lambda a: vp(a.ctypes.data)
        _lib.check(lib.fp_group_register(self._h, c(rgb), c(depth), Kf, H, W, c(m), c(grid), N, int(iterations), c(poses), c(scores), c(best),
                                         c(info)), "fp_group_register")
        return poses, scores, int(best[0]), info
