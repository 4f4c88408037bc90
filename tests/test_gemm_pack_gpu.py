"""Packed last image groups in the implicit-GEMM kernel (csrc/fp_gemm.cu).

A 3x3 convolution's tile is a bw x bh block of bn images (4 x 4 x 8 on 20 x 20 outputs, 8 x 8 x 2 on 40 x 40).  When
n_img % bn = r leaves a partial last group and bn / r >= 2, that group's spatial blocks share tiles, bn / r to a
tile, each as a box of r images.  Packing changes only which pixels share a tile, never an element's k-order or
epilogue arithmetic, so images 0 .. n_img - 1 must be bit-equal to the same inputs run at the next multiple of bn,
whose last group is full.  Only grids of more than one round of persistent CTAs pack (one round takes one tile's
time whatever the packing), so the cases run product-sized batches and two-round grids of a few images.  They cover
every r at both block shapes, stride 1 and 2, the 64-, 128- and 256-wide tiles, the residual, the positional
embedding and the A / B output split.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mods():
    from foundationpose_b200 import _lib, ops, packing

    return _lib, ops, packing


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale


def _same(a, b, what):
    assert a.shape == b.shape, f"{what}: shapes {tuple(a.shape)} and {tuple(b.shape)}"
    eq = a.view(torch.int16) == b.view(torch.int16)
    assert bool(eq.all()), f"{what}: {int((~eq).sum())}/{eq.numel()} fp16 values differ"


# (name, stride-2, input size, Cin, Cout, residual, positional embedding); output size 20: bn = 8, 40: bn = 2
_LAYERS = {
    "s1_512@20": (False, 20, 512, 512, False, False),
    "s1_512@20_res": (False, 20, 512, 512, True, False),
    "s1_512@20_res_pe": (False, 20, 512, 512, True, True),
    "s2_256->512@20": (True, 40, 256, 512, False, False),
    "s1_256@40_res": (False, 40, 256, 256, True, False),
    "s1_128@40_res": (False, 40, 128, 128, True, False),
    "s2_64->128@40": (True, 80, 64, 128, False, False),
    "s1_64@40_res": (False, 40, 64, 64, True, False),
}

_CASES = (
    # 252 hypotheses and every r below them, on the 256-wide tile (249: r = 1, 252: r = 4)
    [(name, 248 + r) for name in ("s1_512@20", "s1_512@20_res", "s1_512@20_res_pe", "s2_256->512@20") for r in range(1, 8)]
    # the 128-wide tile: 3 (17, 19 images) or 2 (9) image groups x 25 blocks x 4 channel tiles, over one round unpacked
    + [("s1_512@20_res_pe", 17), ("s2_256->512@20", 19), ("s1_512@20_res", 9)]
    # 8 x 8 blocks of one image, two to a tile
    + [("s1_256@40_res", 249), ("s2_64->128@40", 249), ("s1_64@40_res", 249)]
)


def _run(name, n, x, w, b, res, pe, out_split=0, out=None, out_ld=None):
    _lib, ops, _ = _mods()
    s2, H, Ci, Co, _, _ = _LAYERS[name]
    kind = _lib.LAYER_CONV3_S2 if s2 else _lib.LAYER_CONV3_S1
    return ops.gemm_layer(kind, x[:n], w, b, n_img=n, Hin=H, Win=H, Cin=Ci, Cout=Co,
                          res=None if res is None else res[:n], res_ld=Co, post_add=pe, relu=True, out=out,
                          out_ld=out_ld, out_split=out_split)


def _tiles(name, n, out_split=0):
    _lib, ops, _ = _mods()
    s2, H, Ci, Co, _, _ = _LAYERS[name]
    kind = _lib.LAYER_CONV3_S2 if s2 else _lib.LAYER_CONV3_S1
    q = dict(n_img=n, Hin=H, Win=H, Cin=Ci, Cout=Co, out_split=out_split)
    return ops.gemm_tile_m(kind, **q), ops.gemm_tile_n(kind, **q)


@pytest.mark.parametrize("name,n", _CASES)
def test_packed_group_bit_equal(name, n):
    """Images 0 .. n - 1 at n_img = n are bit-equal to the same inputs at the next multiple of the tile's images."""
    _, _, packing = _mods()
    s2, H, Ci, Co, use_res, use_pe = _LAYERS[name]
    Ho = H // 2 if s2 else H
    bn = 8 if Ho % 8 else 2
    n_full = -(-n // bn) * bn
    assert n % bn, f"{name} at {n} images has no partial group"
    assert _tiles(name, n) == _tiles(name, n_full), "the two batch sizes take different tiles"
    x = _rand(n_full, H, H, Ci, seed=31).half()
    w = packing.pack_conv3(_rand(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=32).cpu()).cuda()
    b = _rand(Co, seed=33)
    res = _rand(n_full, Ho, Ho, Co, seed=34).half() if use_res else None
    pe = _rand(Ho * Ho, Co, seed=35) if use_pe else None
    full = _run(name, n_full, x, w, b, res, pe)
    part = _run(name, n, x, w, b, res, pe)
    torch.cuda.synchronize()
    _same(part, full[:n], f"{name} at {n} images")


def test_packed_group_out_split(monkeypatch):
    """The last encodeA layer writes A images into channels [0, C) and B images, from image Np on, into [C, 2 C) of
    the concat buffer.  Np is a multiple of the tile's images, so the packed group lies wholly among the B images.
    At 249 pairs the layer would take the swapped tile, which never packs: the 128 x 128 tile is forced."""
    monkeypatch.setenv("FPOSE_SWAP_TILE", "0")
    _, _, packing = _mods()
    name = "s1_128@40_res"
    _, H, Ci, Co, _, _ = _LAYERS[name]
    n_b = 249
    n_a = (n_b + 3) & ~3
    n, n_full = n_a + n_b, n_a + n_b + 1
    assert _tiles(name, n, n_a) == _tiles(name, n_full, n_a), "the two batch sizes take different tiles"
    x = _rand(n_full, H, H, Ci, seed=41).half()
    w = packing.pack_conv3(_rand(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=42).cpu()).cuda()
    b = _rand(Co, seed=43)
    res = _rand(n_full, H, H, Co, seed=44).half()
    outs = []
    for m in (n_full, n):
        out = torch.zeros(n_a, H, H, 2 * Co, dtype=torch.float16, device="cuda")
        _run(name, m, x, w, b, res, None, out_split=n_a, out=out, out_ld=2 * Co)
        outs.append(out)
    torch.cuda.synchronize()
    full, part = outs
    # the buffer holds n_b pairs; A images n_b .. n_a - 1 are pads, which the output map (n_img - out_split
    # images) leaves unstored
    _same(part[:n_b, :, :, :Co], full[:n_b, :, :, :Co], f"A half at {n} images")
    _same(part[:n_b, :, :, Co:], full[:n_b, :, :, Co:], f"B half at {n} images")
