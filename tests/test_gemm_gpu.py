"""Parity of the wgmma implicit-GEMM kernel (csrc/fp_gemm.cu) against torch fp32 convolutions /
matmuls evaluated on the same fp16-rounded operands.  Tolerance: fp16 output rounding (rel 2e-3,
abs 2e-3 on O(1) activations); accumulation is fp32 on both sides.
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
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


@pytest.mark.parametrize("M,K,Co,relu,use_res", [(1000, 512, 1536, False, False), (400, 512, 512, True, True), (37, 64, 64, False, True)])
def test_linear(M, K, Co, relu, use_res):
    _lib, ops, packing = _mods()
    x = _rand(M, K, seed=1).half()
    w = _rand(Co, K, scale=K ** -0.5, seed=2)
    b = _rand(Co, seed=3)
    res = _rand(M, Co, seed=4).half() if use_res else None
    out = ops.gemm_layer(_lib.LAYER_LINEAR, x, packing.pack_linear(w.cpu()).cuda(), b, n_img=1, Hin=1, Win=M, Cin=K,
                         Cout=Co, res=res, res_ld=Co, relu=relu)
    ref = x.float() @ w.half().float().t() + b
    if use_res:
        ref = ref + res.float()
    if relu:
        ref = ref.relu()
    _cmp(out.reshape(M, Co), ref, "linear")


@pytest.mark.parametrize("n,H,Ci,Co,use_res,use_pe", [(3, 40, 128, 128, True, False), (2, 40, 256, 256, False, False),
                                                       (5, 20, 512, 512, True, True), (1, 40, 128, 128, False, False)])
def test_conv3_s1(n, H, Ci, Co, use_res, use_pe):
    _lib, ops, packing = _mods()
    x = _rand(n, Ci, H, H, seed=5).half()
    w = _rand(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=6)
    b = _rand(Co, seed=7)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    res = _rand(n, H, H, Co, seed=8).half() if use_res else None
    pe = _rand(H * H, Co, seed=9) if use_pe else None
    out = ops.gemm_layer(_lib.LAYER_CONV3_S1, x_nhwc, packing.pack_conv3(w.cpu()).cuda(), b, n_img=n, Hin=H, Win=H,
                         Cin=Ci, Cout=Co, res=res, res_ld=Co, post_add=pe, relu=True)
    ref = F.conv2d(x.float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1)
    if use_res:
        ref = ref + res.float()
    ref = ref.relu()
    if use_pe:
        ref = ref + pe.reshape(1, H, H, Co)
    _cmp(out, ref, "conv3_s1")


@pytest.mark.parametrize("n,H,Ci,Co", [(2, 80, 64, 128), (3, 40, 256, 512)])
def test_conv3_s2(n, H, Ci, Co):
    _lib, ops, packing = _mods()
    x = _rand(n, Ci, H, H, seed=10).half()
    w = _rand(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=11)
    b = _rand(Co, seed=12)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    out = ops.gemm_layer(_lib.LAYER_CONV3_S2, x_nhwc, packing.pack_conv3(w.cpu()).cuda(), b, n_img=n, Hin=H, Win=H,
                         Cin=Ci, Cout=Co, relu=True)
    ref = F.conv2d(x.float(), w.half().float(), b, stride=2, padding=1).relu().permute(0, 2, 3, 1)
    _cmp(out, ref, "conv3_s2")


def test_conv7_s2():
    _lib, ops, packing = _mods()
    n, H = 3, 160
    x = _rand(n, 6, H, H, seed=13).half()
    w = _rand(64, 6, 7, 7, scale=(49 * 6) ** -0.5, seed=14)
    b = _rand(64, seed=15)
    xp = packing.pad_image_c8(x)
    out = ops.gemm_layer(_lib.LAYER_CONV7_S2, xp, packing.pack_conv7(w.cpu()).cuda(), b, n_img=n, Hin=H, Win=H, Cin=8,
                         Cout=64, relu=True)
    ref = F.conv2d(x.float(), w.half().float(), b, stride=2, padding=3).relu().permute(0, 2, 3, 1)
    _cmp(out, ref, "conv7_s2")


_STEM_MAX_IMAGES = 504


@pytest.fixture(scope="module")
def _stem_outputs():
    """The stem at 3 images, at the 5 of track_one, and at the 501 / 504 of 249 / 252 hypotheses.  Inputs are drawn
    once at the largest size and sliced, so every batch starts with the same images.  504 images make 25 200 tiles,
    about 191 per CTA, so the six-stage patch ring wraps and its phase bit flips many times."""
    _lib, ops, packing = _mods()
    H = 160
    x = _rand(_STEM_MAX_IMAGES, 6, H, H, seed=23).half()
    w = _rand(64, 6, 7, 7, scale=(49 * 6) ** -0.5, seed=24)
    b = _rand(64, seed=25)
    w_packed = packing.pack_conv7(w.cpu()).cuda()
    outs = {}
    for n in (3, 5, 501, 504):
        outs[n] = ops.gemm_layer(_lib.LAYER_CONV7_S2, packing.pad_image_c8(x[:n]), w_packed, b, n_img=n, Hin=H, Win=H,
                                 Cin=8, Cout=64, relu=True)
    return x, w, b, outs


@pytest.mark.parametrize("n", [3, 5, 501, 504])
def test_conv7_s2_batch_sizes(n, _stem_outputs):
    """The stem at the image counts the product launches, against fp32 on the same fp16 inputs."""
    x, w, b, outs = _stem_outputs
    ref = F.conv2d(x[:n].float(), w.half().float(), b, stride=2, padding=3).relu().permute(0, 2, 3, 1)
    _cmp(outs[n], ref, "conv7_s2")
    # a tile's arithmetic does not depend on where in the ring it lands or how many tiles follow it
    assert torch.equal(outs[n][:3], outs[3]), "images 0..2 differ from the 3-image launch"


def test_out_split_concat():
    """torch.cat((a, b), 1) of refine_network.py:85 fused into the producing layer's store."""
    _lib, ops, packing = _mods()
    n, H, C = 4, 40, 128
    x = _rand(n, C, H, H, seed=16).half()
    w = _rand(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=17)
    b = _rand(C, seed=18)
    out = torch.zeros(n // 2, H, H, 2 * C, dtype=torch.float16, device="cuda")
    ops.gemm_layer(_lib.LAYER_CONV3_S1, x.permute(0, 2, 3, 1).contiguous(), packing.pack_conv3(w.cpu()).cuda(), b,
                   n_img=n, Hin=H, Win=H, Cin=C, Cout=C, out=out, out_ld=2 * C, out_split=n // 2, relu=True)
    y = F.conv2d(x.float(), w.half().float(), b, padding=1).relu()
    ref = torch.cat((y[: n // 2], y[n // 2:]), 1).permute(0, 2, 3, 1)
    _cmp(out, ref, "out_split")
