"""The implicit-GEMM epilogue (csrc/fp_gemm.cu): bias, residual, ReLU and positional embedding at the shapes whose
barrier phases and slab reuse are hardest to get right.

The 256-wide tile stores its four 64-channel batches through two alternating slabs, each with its own residual
barrier, so a CTA's barrier phases depend on how many tiles it has run.  The cases below run grids whose tile count
is not a multiple of the SM count, so some persistent CTAs run an odd number of tiles and the others an even one,
and a 249-image batch whose last image group is ragged.  Each case is checked against an fp32 torch reference
(tolerance as in test_gemm_wide_gpu.py) and for bit-equal outputs across two launches.
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


def _conv3_tiles(n, H, C, tile_n):
    b = 8 if H % 8 == 0 else 4  # pixels per tile side; 128 / b^2 images per tile
    return (H // b) ** 2 * -(-n // (128 // (b * b))) * (C // tile_n)


@pytest.mark.parametrize(
    "n,H,C,use_res,use_pe,tile_n",
    [
        (249, 20, 512, True, True, 256),    # ragged last image group (249 = 31 x 8 + 1)
        (250, 20, 512, True, False, 256),
        (252, 20, 512, False, True, 256),
        (249, 40, 256, True, False, 256),
        (32, 20, 512, True, True, 128),     # a 32-hypothesis shard: the 128-wide tile, both slabs in one pass
    ],
)
def test_conv3_epilogue(n, H, C, use_res, use_pe, tile_n):
    _lib, ops, packing = _mods()
    assert ops.gemm_tile_n(_lib.LAYER_CONV3_S1, n_img=n, Hin=H, Win=H, Cin=C, Cout=C) == tile_n
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = _conv3_tiles(n, H, C, tile_n)
    if tile_n == 256:
        # persistent CTAs run tiles // sms or tiles // sms + 1 tiles: both parities occur
        assert tiles > sms and tiles % sms != 0, (tiles, sms)
    x = _rand(n, H, H, C, seed=21).half()
    w = _rand(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=22)
    b = _rand(C, seed=23)
    res = _rand(n, H, H, C, seed=24).half() if use_res else None
    pe = _rand(H * H, C, seed=25) if use_pe else None
    wp = packing.pack_conv3(w.cpu()).cuda()

    def run():
        return ops.gemm_layer(_lib.LAYER_CONV3_S1, x, wp, b, n_img=n, Hin=H, Win=H, Cin=C, Cout=C, res=res, res_ld=C,
                              post_add=pe, relu=True)

    out = run()
    again = run()
    torch.cuda.synchronize()
    assert torch.equal(out, again), "two launches of the same layer differ"
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1)
    if use_res:
        ref = ref + res.float()
    ref = ref.relu()
    if use_pe:
        ref = ref + pe.reshape(1, H, H, C)
    _cmp(out, ref, f"conv3 {C} @{H} ({n}) res={use_res} pe={use_pe}")
