"""The weight-stationary K = 512 linear kernel (csrc/fp_linear.cu) against the 128 x 128 tile of gemm_tile_kernel, which
FPOSE_LINEAR_WS=0 selects: bit-identical outputs on every head shape (both in-projections, the out-projection / FF2
with their residual, FF1 with its ReLU), at 252 hypotheses' 100 800 rows, a ragged 99 600 (249 hypotheses: the last
64-row tile is partial) and the smallest row count that takes the new kernel; and against a float64 reference with the
tolerance of test_gemm_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

K = 512
SHAPES = [(3072, False, False), (1536, False, False), (512, True, False), (512, False, True)]  # Cout, residual, ReLU


def _mods():
    from foundationpose_b200 import _lib, ops, packing

    return _lib, ops, packing


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _tile_m(M, Co):
    _lib, ops, _ = _mods()
    return ops.gemm_tile_m(_lib.LAYER_LINEAR, n_img=1, Hin=1, Win=M, Cin=K, Cout=Co)


def _smallest_ws_rows(Co):
    """the smallest row count the plan gives the weight-stationary kernel (64-row tiles)"""
    lo, hi = 1, 100800
    assert _tile_m(hi, Co) == 64
    while lo < hi:
        mid = (lo + hi) // 2
        if _tile_m(mid, Co) == 64:
            hi = mid
        else:
            lo = mid + 1
    return lo


@pytest.mark.parametrize("rows", ["100800", "99600", "smallest"])
@pytest.mark.parametrize("Co,use_res,relu", SHAPES)
def test_linear_ws_is_bitwise_the_128_tile(Co, use_res, relu, rows, monkeypatch):
    _lib, ops, packing = _mods()
    monkeypatch.delenv("FPOSE_LINEAR_WS", raising=False)
    M = _smallest_ws_rows(Co) if rows == "smallest" else int(rows)
    x = _rand(M, K, seed=21).half()
    w = _rand(Co, K, scale=K ** -0.5, seed=22)
    b = _rand(Co, seed=23)
    res = _rand(M, Co, seed=24).half() if use_res else None
    wp = packing.pack_linear(w.cpu()).cuda()
    outs = {}
    for flag, tile in (("0", 128), ("1", 64)):
        monkeypatch.setenv("FPOSE_LINEAR_WS", flag)
        assert _tile_m(M, Co) == tile
        outs[flag] = ops.gemm_layer(_lib.LAYER_LINEAR, x, wp, b, n_img=1, Hin=1, Win=M, Cin=K, Cout=Co, res=res,
                                    res_ld=Co, relu=relu).reshape(M, Co)
    torch.cuda.synchronize()
    assert torch.equal(outs["0"], outs["1"]), (
        f"{(outs['0'] != outs['1']).sum().item()} of {M * Co} outputs differ (M {M}, Cout {Co})")
    ref = x.double() @ w.half().double().t() + b.double()
    if use_res:
        ref = ref + res.double()
    if relu:
        ref = ref.relu()
    err = (outs["1"].double() - ref).abs()
    bad = (err > 3e-3 + 2e-3 * ref.abs()).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} outside the fp16 tolerance, max err {err.max().item():.4g}"


def test_short_layers_keep_the_128_tile(monkeypatch):
    """track_one's 400 rows stay on the 128 x 128 tile: a CTA would load a whole weight panel for one or two tiles"""
    monkeypatch.delenv("FPOSE_LINEAR_WS", raising=False)
    for Co, _, _ in SHAPES:
        assert _tile_m(400, Co) == 128
