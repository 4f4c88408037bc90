"""The swapped tile of the implicit-GEMM kernel (csrc/fp_gemm.cu, `gemm_tile_kernel<128, true>`): the encoders'
128-channel 3x3 convolutions with the weights as the wgmma M operand over 256 pixels.  Each case runs one of the
encodeA layers that take it at 252 hypotheses (504 images) and at 249 (A images 0..248, B from 252:
501 images, a ragged last tile), asserts through the tile query which tile ran, and checks the output against torch fp32 on the same
fp16-rounded operands (tolerance as in test_gemm_wide_gpu.py) and bit for bit against the 128 x 128 tile
(FPOSE_SWAP_TILE=0): both tiles sum the same products in the same k order and share the epilogue arithmetic.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (kind, Hin, Cin, residual, out_split): the 128 -> 128 convolutions of encodeA.2 / .3 without and with the residual,
# and the last one, which writes into the 256-channel concat buffer.  encodeA.1 (stride 2, 64 -> 128, 9 k-blocks) keeps
# the 128 x 128 tile.
LAYERS = {
    "conv3_128": (1, 40, 128, False, False),
    "conv3_128_res": (1, 40, 128, True, False),
    "conv3_128_res_split": (1, 40, 128, True, True),
}


def _mods():
    from foundationpose_b200 import _lib, ops, packing

    return _lib, ops, packing


@pytest.fixture(autouse=True)
def _fp32_reference():
    # the references are fp32 convolutions: no TF32 inside them
    conv = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = conv


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale


def _run(layer, n_real, monkeypatch, swap):
    """One encodeA layer over A images 0..n_real-1 and B images from Np = n_real rounded up to 4: (output, reference,
    tile_m).  Without the split the layer sees all Np + n_real images as one batch."""
    _lib, ops, packing = _mods()
    kind, H, Ci, use_res, split = LAYERS[layer]
    Co = 128
    Np = (n_real + 3) & ~3
    n = Np + n_real
    Ho = H
    monkeypatch.setenv("FPOSE_SWAP_TILE", "1" if swap else "0")
    q = dict(n_img=n, Hin=H, Win=H, Cin=Ci, Cout=Co, out_split=Np if split else 0)
    tile_m = ops.gemm_tile_m(kind, **q)
    assert ops.gemm_tile_n(kind, **q) == 128
    x = _rand(n, H, H, Ci, seed=1).half()
    w = _rand(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=2)
    b = _rand(Co, seed=3)
    res = _rand(n, Ho, Ho, Co, seed=4).half() if use_res else None
    kw = dict(n_img=n, Hin=H, Win=H, Cin=Ci, Cout=Co, res=res, res_ld=Co, relu=True)
    if split:
        out = torch.full((n - Np, Ho, Ho, 2 * Co), float("nan"), dtype=torch.float16, device="cuda")
        kw.update(out=out, out_ld=2 * Co, out_split=Np)
    out = ops.gemm_layer(kind, x, packing.pack_conv3(w.cpu()).cuda(), b, **kw)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1)
    if use_res:
        ref = ref + res.float()
    ref = ref.relu()
    if split:  # image i of the output: A image i in channels [0, 128), B image Np + i in [128, 256)
        ref = torch.cat([ref[:n - Np], ref[Np:]], dim=3)
    return out, ref, tile_m


def _cmp(got, ref, what, rtol=2e-3, atol=3e-3):
    got = got.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


@pytest.mark.parametrize("n_real", [252, 249])
@pytest.mark.parametrize("layer", list(LAYERS))
def test_swapped_tile_matches_fp32(layer, n_real, monkeypatch):
    out, ref, tile_m = _run(layer, n_real, monkeypatch, swap=True)
    assert tile_m == 256
    _cmp(out, ref, f"{layer} at {n_real} hypotheses")


@pytest.mark.parametrize("n_real", [252, 249])
@pytest.mark.parametrize("layer", list(LAYERS))
def test_swapped_tile_is_bitwise_the_128_tile(layer, n_real, monkeypatch):
    out_s, _, tile_s = _run(layer, n_real, monkeypatch, swap=True)
    out_n, _, tile_n = _run(layer, n_real, monkeypatch, swap=False)
    assert (tile_s, tile_n) == (256, 128)
    diff = (out_s.float() - out_n.float()).abs().max().item()
    assert torch.equal(out_s, out_n), f"{layer} at {n_real}: largest difference {diff}"


def test_persistent_ctas_run_odd_and_even_tile_counts(monkeypatch):
    """The residual barrier completes once per tile and is waited on with the parity of the CTA's tile count, so a grid
    on which some CTAs run an odd and others an even number of tiles exercises both phases in one launch."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = 25 * ((252 + 252) // 4)  # 5 x 5 blocks of 8 x 8 pixels per 40 x 40 image, four images per tile
    assert tiles > sms and tiles % sms != 0, "every CTA would run the same number of tiles"
    out_s, ref, tile_s = _run("conv3_128_res", 252, monkeypatch, swap=True)
    out_n, _, _ = _run("conv3_128_res", 252, monkeypatch, swap=False)
    assert tile_s == 256
    assert torch.equal(out_s, out_n)
    _cmp(out_s, ref, "conv3 128 +res")


@pytest.mark.parametrize("n_img,H,Ci,kind", [(2, 40, 128, 1), (64, 40, 128, 1), (504, 80, 64, 2), (504, 40, 128, 1)])
def test_short_grids_and_the_switch_keep_the_128_tile(n_img, H, Ci, kind, monkeypatch):
    """track_one's two images and a 32-hypothesis shard fill too few waves, the stride-2 layer's k-loop is too short,
    and FPOSE_SWAP_TILE=0 turns the tile off."""
    _lib, ops, _ = _mods()
    q = dict(n_img=n_img, Hin=H, Win=H, Cin=Ci, Cout=128)
    monkeypatch.setenv("FPOSE_SWAP_TILE", "1")
    if n_img == 504 and kind == _lib.LAYER_CONV3_S1:
        assert ops.gemm_tile_m(kind, **q) == 256
        monkeypatch.setenv("FPOSE_SWAP_TILE", "0")
    assert ops.gemm_tile_m(kind, **q) == 128
    assert ops.gemm_tile_n(kind, **q) == 128
