"""ctypes binding of libfpose.so (the C ABI declared in include/fpose.h).

There is deliberately no fallback: if the CUDA library is missing, importing this module raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# FPOSE_LIB_PATH: load another in-tree build of the same sources (A/B experiments with compile-time variants)
LIB_PATH = os.environ.get("FPOSE_LIB_PATH") or os.path.join(_HERE, "lib", "libfpose.so")


class FposeError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        # try to build in-tree (needs nvcc); never fall back to a CPU path
        from . import build as _build

        _build.build()
    if not os.path.exists(LIB_PATH):
        raise FposeError(f"{LIB_PATH} is missing: build it with `python -m foundationpose_b200.build`")
    return C.CDLL(LIB_PATH)


lib = _load()


class DepthSensor(C.Structure):
    """struct fp_depth_sensor (include/fpose.h)."""

    _fields_ = [("H", C.c_int), ("W", C.c_int), ("K", C.c_float * 9), ("T_color_from_depth", C.c_float * 16)]

    @classmethod
    def of(cls, H, W, K, T):
        """The record of a depth image of H x W with intrinsics K (9 floats) and T_color_from_depth (16 floats), row-major."""
        return cls(int(H), int(W), (C.c_float * 9)(*[float(x) for x in K]), (C.c_float * 16)(*[float(x) for x in T]))


class GemmLayer(C.Structure):
    """struct fp_gemm_layer (include/fpose.h)."""

    _fields_ = [
        ("kind", C.c_int),
        ("n_img", C.c_int),
        ("Hin", C.c_int),
        ("Win", C.c_int),
        ("Cin", C.c_int),
        ("Cout", C.c_int),
        ("in_", C.c_void_p),
        ("w", C.c_void_p),
        ("bias", C.c_void_p),
        ("res", C.c_void_p),
        ("res_ld", C.c_int),
        ("out", C.c_void_p),
        ("out_ld", C.c_int),
        ("out_split", C.c_int),
        ("post_add", C.c_void_p),
        ("relu", C.c_int),
    ]


LAYER_LINEAR, LAYER_CONV3_S1, LAYER_CONV3_S2, LAYER_CONV7_S2 = 0, 1, 2, 3

lib.fp_last_error.restype = C.c_char_p
lib.fp_launch_count.restype = C.c_ulonglong
lib.fp_op_gemm_layer.argtypes = [C.POINTER(GemmLayer), C.c_void_p]
lib.fp_op_gemm_layer.restype = C.c_int
lib.fp_pose_errors.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_void_p]
lib.fp_pose_errors.restype = C.c_int
lib.fp_sym_pose_errors.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                   C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
lib.fp_sym_pose_errors.restype = C.c_int
lib.fp_vsd_errors.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                              C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_int,
                              C.c_void_p, C.c_void_p, C.c_void_p]
lib.fp_vsd_errors.restype = C.c_int


def check(rc, what=""):
    if rc != 0:
        msg = lib.fp_last_error()
        raise FposeError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")


def launch_count():
    return int(lib.fp_launch_count())


lib.fp_prof_enable.argtypes = [C.c_int]
lib.fp_prof_enable.restype = C.c_int
lib.fp_prof_collect.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int)]
lib.fp_prof_collect.restype = C.c_int


def prof_enable(on):
    check(lib.fp_prof_enable(1 if on else 0), "fp_prof_enable")


def prof_collect(kind):
    """-> (total_ms, total_work, launches) of kernel `kind` (0 = implicit GEMM [FLOPs], 1 = crop [bytes])."""
    ms, work, n = C.c_double(), C.c_double(), C.c_int()
    check(lib.fp_prof_collect(kind, C.byref(ms), C.byref(work), C.byref(n)), "fp_prof_collect")
    return ms.value, work.value, n.value
