"""Parity of the 256-wide tile of the implicit-GEMM kernel (csrc/fp_gemm.cu) against torch fp32 convolutions /
matmuls on the same fp16-rounded operands, at the batch sizes that select it (it needs enough tiles to fill several
waves of SMs, so the small shapes of test_gemm_gpu.py run the 128-wide tile).  Each case also asserts which tile
width ran, through the read-only tile query; the refiner's linear layers at full height are checked too and stay at
128 wide.  Tolerance as in test_gemm_gpu.py: fp16 output rounding.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _mods():
    from foundationpose_b200 import _lib, ops, packing

    return _lib, ops, packing


@pytest.fixture(autouse=True)
def _fp32_reference():
    # the references are fp32 convolutions / matmuls: no TF32 inside them
    conv, mm = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = conv, mm


def _cmp(got, ref, what, rtol=2e-3, atol=3e-3):
    got = got.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale


@pytest.mark.parametrize("n,use_res", [(252, False), (249, True)])  # 249: an odd number of M tiles, a ragged last one
def test_conv3_256_at_40(n, use_res):
    _lib, ops, packing = _mods()
    H, C = 40, 256
    assert ops.gemm_tile_n(_lib.LAYER_CONV3_S1, n_img=n, Hin=H, Win=H, Cin=C, Cout=C) == 256
    x = _rand(n, H, H, C, seed=1).half()
    w = _rand(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=2)
    b = _rand(C, seed=3)
    res = _rand(n, H, H, C, seed=4).half() if use_res else None
    out = ops.gemm_layer(_lib.LAYER_CONV3_S1, x, packing.pack_conv3(w.cpu()).cuda(), b, n_img=n, Hin=H, Win=H, Cin=C,
                         Cout=C, res=res, res_ld=C, relu=True)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1)
    if use_res:
        ref = ref + res.float()
    _cmp(out, ref.relu(), "conv3 256 @40")


def test_conv3_s2_256_to_512():
    _lib, ops, packing = _mods()
    n, H, Ci, Co = 252, 40, 256, 512
    assert ops.gemm_tile_n(_lib.LAYER_CONV3_S2, n_img=n, Hin=H, Win=H, Cin=Ci, Cout=Co) == 256
    x = _rand(n, H, H, Ci, seed=5).half()
    w = _rand(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=6)
    b = _rand(Co, seed=7)
    out = ops.gemm_layer(_lib.LAYER_CONV3_S2, x, packing.pack_conv3(w.cpu()).cuda(), b, n_img=n, Hin=H, Win=H, Cin=Ci,
                         Cout=Co, relu=True)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.half().float(), b, stride=2, padding=1).relu().permute(0, 2, 3, 1)
    _cmp(out, ref, "conv3 s2 256->512")


def test_conv3_512_at_20_residual_and_pe():
    _lib, ops, packing = _mods()
    n, H, C = 252, 20, 512
    assert ops.gemm_tile_n(_lib.LAYER_CONV3_S1, n_img=n, Hin=H, Win=H, Cin=C, Cout=C) == 256
    x = _rand(n, H, H, C, seed=8).half()
    w = _rand(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=9)
    b = _rand(C, seed=10)
    res = _rand(n, H, H, C, seed=11).half()
    pe = _rand(H * H, C, seed=12)
    out = ops.gemm_layer(_lib.LAYER_CONV3_S1, x, packing.pack_conv3(w.cpu()).cuda(), b, n_img=n, Hin=H, Win=H, Cin=C,
                         Cout=C, res=res, res_ld=C, post_add=pe, relu=True)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1)
    ref = (ref + res.float()).relu() + pe.reshape(1, H, H, C)
    _cmp(out, ref, "conv3 512 @20 +res +pe")


@pytest.mark.parametrize("Co,use_res", [(3072, False), (512, True)])
def test_linear_ragged_last_tile(Co, use_res):
    """The refiner's qkv and head projections (K = 512: too short a k-loop for the wide tile, so 128 wide)."""
    _lib, ops, packing = _mods()
    M, K = 100800, 512  # 787.5 tiles of 128 rows
    assert ops.gemm_tile_n(_lib.LAYER_LINEAR, n_img=1, Hin=1, Win=M, Cin=K, Cout=Co) == 128
    x = _rand(M, K, seed=13).half()
    w = _rand(Co, K, scale=K ** -0.5, seed=14)
    b = _rand(Co, seed=15)
    res = _rand(M, Co, seed=16).half() if use_res else None
    out = ops.gemm_layer(_lib.LAYER_LINEAR, x, packing.pack_linear(w.cpu()).cuda(), b, n_img=1, Hin=1, Win=M, Cin=K,
                         Cout=Co, res=res, res_ld=Co, relu=use_res)
    ref = x.float() @ w.half().float().t() + b
    if use_res:
        ref = (ref + res.float()).relu()
    _cmp(out.reshape(M, Co), ref, f"linear 512->{Co}")


@pytest.mark.parametrize("kind,n,H,C", [(1, 1, 40, 256), (1, 32, 40, 256), (1, 32, 20, 512), (2, 32, 40, 256)])
def test_short_grids_keep_the_128_wide_tile(kind, n, H, C):
    """track_one's single image and a 32-hypothesis shard fill too few waves for the wide tile."""
    _lib, ops, _ = _mods()
    Co = 2 * C if kind == _lib.LAYER_CONV3_S2 else C
    assert ops.gemm_tile_n(kind, n_img=n, Hin=H, Win=H, Cin=C, Cout=Co) == 128
