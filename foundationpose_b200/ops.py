"""Thin torch-tensor front end over the single-operator C-ABI hooks (`fp_op_*`).

Used by the parity tests to check each CUDA kernel against the oracle in isolation.  torch is only
the owner of device memory and streams here; all compute happens inside libfpose.so.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import lib


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.FposeError("libfpose operators need CUDA tensors (there is no CPU path)")


def gemm_layer(kind, x, w_packed, bias, *, n_img, Hin, Win, Cin, Cout, out=None, out_ld=None, out_split=0,
               res=None, res_ld=0, post_add=None, relu=False):
    """Run one implicit-GEMM layer.  `x`: fp16 activation tensor in the layout the kind expects."""
    _require_cuda(x, w_packed, bias, res, post_add, out)
    assert x.dtype == torch.float16 and w_packed.dtype == torch.float16 and bias.dtype == torch.float32
    if kind == _lib.LAYER_LINEAR:
        Ho, Wo = 1, Win
    elif kind == _lib.LAYER_CONV3_S1:
        Ho, Wo = Hin, Win
    else:
        Ho, Wo = Hin // 2, Win // 2
    if out is None:
        out_ld = Cout
        out = torch.empty(n_img, Ho, Wo, Cout, dtype=torch.float16, device=x.device)
    L = _lib.GemmLayer(kind, n_img, Hin, Win, Cin, Cout, _ptr(x), _ptr(w_packed), _ptr(bias), _ptr(res),
                       res_ld, _ptr(out), out_ld, out_split, _ptr(post_add), 1 if relu else 0)
    _lib.check(lib.fp_op_gemm_layer(C.byref(L), _stream()), "fp_op_gemm_layer")
    return out


def gemm_tile_n(kind, *, n_img, Hin, Win, Cin, Cout, out_split=0):
    """Output channels per tile (64, 128 or 256) that `gemm_layer` picks for this shape on the current device."""
    lib.fp_op_gemm_tile_n.argtypes = [C.POINTER(_lib.GemmLayer), C.POINTER(C.c_int)]
    lib.fp_op_gemm_tile_n.restype = C.c_int
    L = _lib.GemmLayer(kind, n_img, Hin, Win, Cin, Cout, None, None, None, None, 0, None, Cout, out_split, None, 0)
    tile_n = C.c_int(0)
    _lib.check(lib.fp_op_gemm_tile_n(C.byref(L), C.byref(tile_n)), "fp_op_gemm_tile_n")
    return tile_n.value


def gemm_tile_m(kind, *, n_img, Hin, Win, Cin, Cout, out_split=0):
    """Output pixels (linear rows) per tile that `gemm_layer` picks for this shape: 128, 256 for the swapped
    128-channel tile, 64 for the weight-stationary K = 512 linear kernel."""
    lib.fp_op_gemm_tile_m.argtypes = [C.POINTER(_lib.GemmLayer), C.POINTER(C.c_int)]
    lib.fp_op_gemm_tile_m.restype = C.c_int
    L = _lib.GemmLayer(kind, n_img, Hin, Win, Cin, Cout, None, None, None, None, 0, None, Cout, out_split, None, 0)
    tile_m = C.c_int(0)
    _lib.check(lib.fp_op_gemm_tile_m(C.byref(L), C.byref(tile_m)), "fp_op_gemm_tile_m")
    return tile_m.value


lib.fp_op_attention.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
lib.fp_op_attention.restype = C.c_int


def attention(qkv, impl=1):
    """qkv fp16 [B*400, 1536] -> fp16 [B*400, 512]; `impl` is ignored: one implementation, the wgmma kernel."""
    _require_cuda(qkv)
    assert qkv.dtype == torch.float16 and qkv.shape[1] == 1536 and qkv.shape[0] % 400 == 0
    B = qkv.shape[0] // 400
    out = torch.empty(qkv.shape[0], 512, dtype=torch.float16, device=qkv.device)
    _lib.check(lib.fp_op_attention(_ptr(qkv), _ptr(out), B, impl, _stream()), "fp_op_attention")
    return out


lib.fp_op_attention_groups.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
lib.fp_op_attention_groups.restype = C.c_int
lib.fp_op_layernorm.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
lib.fp_op_layernorm.restype = C.c_int
lib.fp_op_head_final.argtypes = [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_void_p]
lib.fp_op_head_final.restype = C.c_int
lib.fp_op_token_mean_proj.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
lib.fp_op_token_mean_proj.restype = C.c_int


def attention_groups(qkv, B, n_groups, *, ld=None):
    """Attention of the heads' launch: `qkv` fp16 rows of `ld` elements (default: the tensor's row stride), B * 400 of
    them from qkv's first element, group g's q | k | v at columns [1536 g, 1536 g + 1536) -> fp16 [n_groups, B*400, 512].
    `qkv` may be a column slice of a wider tensor (pass ld)."""
    _require_cuda(qkv)
    assert qkv.dtype == torch.float16 and qkv.stride(-1) == 1
    ld = qkv.stride(0) if ld is None else ld
    out = torch.empty(n_groups, B * 400, 512, dtype=torch.float16, device=qkv.device)
    _lib.check(lib.fp_op_attention_groups(_ptr(qkv), ld, n_groups, _ptr(out), B, _stream()), "fp_op_attention_groups")
    return out


def layernorm(x, gamma, beta):
    """fp16 [rows, 512] -> fp16 [rows, 512]: LayerNorm with fp32 gamma / beta, eps 1e-5."""
    _require_cuda(x, gamma, beta)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.shape[-1] == 512
    assert gamma.dtype == torch.float32 and beta.dtype == torch.float32
    y = torch.empty_like(x)
    rows = x.numel() // 512
    _lib.check(lib.fp_op_layernorm(_ptr(x), _ptr(y), _ptr(gamma), _ptr(beta), rows, _stream()), "fp_op_layernorm")
    return y


def head_final(x, gamma, beta, w, bias):
    """Refiner read-out: fp16 [B, 400, 512] -> fp32 [B, out_dim] = w . mean over tokens of LayerNorm(x) + bias."""
    _require_cuda(x, gamma, beta, w, bias)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.shape[1:] == (400, 512)
    B, out_dim = x.shape[0], w.shape[0]
    out = torch.empty(B, out_dim, dtype=torch.float32, device=x.device)
    _lib.check(lib.fp_op_head_final(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(w.contiguous()), _ptr(bias), _ptr(out), B, out_dim,
                                    _stream()), "fp_op_head_final")
    return out


def token_mean_proj(x, w, bias):
    """Scorer features: fp16 [B, 400, 512] -> fp32 [B, 512] = w (mean over tokens of x) + bias, w fp32 [512, 512]."""
    _require_cuda(x, w, bias)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.shape[1:] == (400, 512)
    assert w.dtype == torch.float32 and w.is_contiguous() and w.shape == (512, 512)
    B = x.shape[0]
    mean_ws = torch.empty(B, 512, dtype=torch.float32, device=x.device)
    out = torch.empty(B, 512, dtype=torch.float32, device=x.device)
    _lib.check(lib.fp_op_token_mean_proj(_ptr(x), _ptr(w), _ptr(bias), _ptr(mean_ws), _ptr(out), B, _stream()),
               "fp_op_token_mean_proj")
    return out


lib.fp_align_depth.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_longlong, C.POINTER(_lib.DepthSensor), C.POINTER(C.c_float),
                               C.c_int, C.c_int, C.c_void_p, C.c_void_p]
lib.fp_align_depth.restype = C.c_int


def align_depth(depth, sensor, K_color, H, W):
    """Depth from its own sensor aligned to a colour frame of H x W with intrinsics K_color (3,3), by the rule of
    fp_set_camera_depth_sensor (include/fpose.h, librealsense's rs2::align to colour): a CUDA float32 (H, W) tensor of
    metres, 0 where no depth lands.  depth: a frames.Depth around a CUDA tensor (float32 metres or uint16 with a scale,
    any row pitch) of the sensor's own size, or a plain CUDA float32 (Hd, Wd) tensor with `sensor` a frames.DepthSensor.
    Runs on the current stream."""
    from .frames import Depth, DepthSensor

    if not isinstance(depth, Depth):
        if not isinstance(sensor, DepthSensor):
            raise TypeError("align_depth: a plain depth tensor needs a DepthSensor")
        depth = Depth(depth, sensor=sensor)
    elif sensor is not None and depth.sensor is not None and sensor is not depth.sensor:
        raise ValueError("align_depth: the Depth has a sensor of its own; pass sensor=None")
    sensor = depth.sensor if depth.sensor is not None else sensor
    if not isinstance(sensor, DepthSensor):
        raise TypeError("align_depth: needs a DepthSensor")
    img = depth.img
    if not (torch.is_tensor(img) and img.is_cuda):
        raise _lib.FposeError("align_depth: the depth must be a CUDA tensor (there is no CPU path)")
    rec = _lib.DepthSensor.of(depth.H, depth.W, sensor.K.reshape(-1), sensor.T.reshape(-1))
    Kc = (C.c_float * 9)(*[float(x) for x in torch.as_tensor(K_color, dtype=torch.float64).reshape(-1)])
    out = torch.empty(int(H), int(W), dtype=torch.float32, device=img.device)
    _lib.check(lib.fp_align_depth(_ptr(img), depth.code, float(depth.scale), depth.pitch, C.byref(rec), Kc, int(H), int(W),
                                  _ptr(out), _stream()), "fp_align_depth")
    return out
