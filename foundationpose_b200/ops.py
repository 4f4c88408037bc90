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
    """Output pixels per tile (128, or 256 for the swapped 128-channel tile) that `gemm_layer` picks for this shape."""
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
