"""CPU: the encoder's weight preparation and the error bar of test_encoder_gpu.py, without a GPU.

  * packing.fold_bn + pack_conv3 / pack_conv7 (through engine.pack_network) against a float64 fold of the state dict;
  * the test's inverse packers round-trip;
  * a CPU emulation of one layer as the kernels round it (fp16 operands, fp32 sums of K = 16 slices added to an fp32
    accumulator, fp32 epilogue, one fp16 rounding) passes encoder_reference.bar, and every probe of the GPU test fails
    it on small shapes.
"""
import pytest
import torch

import encoder_reference as ref


def _ulp16(x):
    """fp16 ulp at |x| (normal range; 2^-24 below it)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return 2.0 ** (e - 10)


@pytest.mark.parametrize("kind", ["refine", "score"])
def test_fold_and_pack_against_float64(kind):
    """Every packed fp16 weight is within one fp16 ulp of the float64 fold w gamma / sqrt(var + eps), every fp32 bias
    within 4 fp32 ulps of the magnitude of its terms ((b - mean) gamma / sqrt(var + eps) + beta), and the inverse
    packers give back the packed bits."""
    from foundationpose_b200 import packing
    from foundationpose_b200.engine import encoder_convs, pack_network
    from foundationpose_b200.weights import random_state_dict

    sd = random_state_dict(kind, 5)
    packed = pack_network(sd, kind)
    for i, (cname, bname) in enumerate(encoder_convs(kind)):
        w = sd[f"{cname}.weight"].double()
        b = sd[f"{cname}.bias"].double()
        scale = sd[f"{bname}.weight"].double() / torch.sqrt(sd[f"{bname}.running_var"].double() + 1e-5)
        w64 = w * scale.reshape(-1, 1, 1, 1)
        t1 = (b - sd[f"{bname}.running_mean"].double()) * scale
        b64 = t1 + sd[f"{bname}.bias"].double()
        wp = torch.from_numpy(packed[f"enc.{i}.w"])
        wu = ref.unpack_conv7(wp) if i == 0 else ref.unpack_conv3(wp)
        repack = packing.pack_conv7(wu.float()) if i == 0 else packing.pack_conv3(wu.float())
        assert torch.equal(repack.view(torch.int16), wp.view(torch.int16)), f"layer {i}: unpack / re-pack changed bits"
        wu = wu[:, :w.shape[1]].double()
        if i == 0:
            assert not wp.reshape(7, 8, -1, 8)[:, 7].any() and not wp[..., w.shape[1]:].any(), "stem pad taps not zero"
        assert wu.shape == w64.shape
        assert ((wu - w64).abs() <= _ulp16(w64)).all(), f"layer {i}: a weight is more than one fp16 ulp off"
        bf = torch.from_numpy(packed[f"enc.{i}.b"]).double()
        assert ((bf - b64).abs() <= 4 * 2.0 ** -24 * (t1.abs() + sd[f"{bname}.bias"].double().abs())).all(), f"layer {i}: bias"


def test_inverse_packers_round_trip():
    from foundationpose_b200 import packing

    g = torch.Generator().manual_seed(1)
    w3 = torch.randn(128, 64, 3, 3, generator=g).half()
    assert torch.equal(ref.unpack_conv3(packing.pack_conv3(w3.float())), w3)
    w7 = torch.randn(64, 6, 7, 7, generator=g).half()
    u7 = ref.unpack_conv7(packing.pack_conv7(w7.float()))
    assert torch.equal(u7[:, :6], w7) and not u7[:, 6:].any()


def _emulate(x, wp, b, kind, H, res=None, pe=None):
    """One 3x3 layer as the kernel rounds it: x fp16 NHWC, wp the packed fp16 (Co, 9 Ci) with K ordered (r, s, c);
    fp32 products (exact), each K = 16 slice summed in fp32 and added to an fp32 accumulator, then + b, + res, ReLU,
    + pe in fp32 and one fp16 rounding."""
    n, _, _, ci = x.shape
    co = wp.shape[0]
    xc = x.permute(0, 3, 1, 2).float()
    cols = torch.nn.functional.unfold(xc, 3, padding=1, stride=1 if kind == ref.LK_CONV3_S1 else 2)
    L = cols.shape[-1]
    cols = cols.reshape(n, ci, 9, L).transpose(1, 2).reshape(n, 9 * ci, L)  # K as (r, s, c), the packed order
    w = wp.float()
    acc = torch.zeros(n, co, L, dtype=torch.float32)
    for k0 in range(0, 9 * ci, 16):
        acc += w[:, k0:k0 + 16] @ cols[:, k0:k0 + 16]
    ho = ref.out_hw(kind, H)
    a = acc.transpose(1, 2).reshape(n, ho, ho, co) + b.float()
    if res is not None:
        a = a + res.float()
    a = a.clamp_min(0.0)
    if pe is not None:
        a = a + pe.float()
    return a.half()


@pytest.mark.parametrize("kind", [ref.LK_CONV3_S1, ref.LK_CONV3_S2])
def test_bar_accepts_the_kernel_rounding_and_rejects_the_probes(kind):
    """4 images of 8 x 8 (stride 1: with a residual and an 8 x 8 positional embedding; stride 2: 16 x 16 input) with
    64 channels.  The emulation passes the bar; each probe of test_encoder_gpu fails it on a good part of the elements:
    (a) tap (2, 2) zeroed, (b) the residual taken from the layer's input, (c) the images' second half from the wrong
    image, (d) the positional embedding transposed, (e) the stride-2 window shifted one pixel."""
    from foundationpose_b200 import packing
    from foundationpose_b200.weights import positional_embedding

    g = torch.Generator().manual_seed(7 + kind)
    H = 8 if kind == ref.LK_CONV3_S1 else 16
    ci = co = 64
    x = torch.relu(torch.randn(4, H, H, ci, generator=g)).half()
    w = (torch.randn(co, ci, 3, 3, generator=g) * (2.0 / (9 * ci)) ** 0.5).half()
    wp = packing.pack_conv3(w.float())
    b = torch.randn(co, generator=g) * 0.1
    ho = ref.out_hw(kind, H)
    res = pe = None
    if kind == ref.LK_CONV3_S1:
        res = torch.relu(torch.randn(4, ho, ho, co, generator=g)).half()
        pe = positional_embedding(64, co)[0].reshape(8, 8, co)
    got = _emulate(x, wp, b, kind, H, res, pe).double()
    acc, mag, tap = ref.conv_terms(x, ref.unpack_conv3(wp), kind, H)
    y = ref.epilogue(acc, b, res, pe)
    bar = ref.bar(y, acc, mag, b, ref.k_steps(kind, ci), res, pe)
    err = (got - y).abs()
    assert (err <= bar).all(), f"emulated layer over the bar: worst error / bar {(err / bar).max().item():.3f}"
    assert (err / bar).max() > 0.01, "the bar is far looser than the rounding it bounds"
    frac = lambda probe: ((got - probe).abs() > bar).double().mean().item()
    assert frac(ref.epilogue(acc - tap, b, res, pe)) > 0.25
    assert frac(ref.epilogue(acc, b, res, pe)[[0, 1, 3, 2]]) > 0.25
    if kind == ref.LK_CONV3_S1:
        assert frac(ref.epilogue(acc, b, x, pe)) > 0.25
        assert frac(ref.epilogue(acc, b, res, pe.transpose(0, 1))) > 0.05
    else:
        acc_s, _, _ = ref.conv_terms(x, ref.unpack_conv3(wp), kind, H, shift=True)
        assert frac(ref.epilogue(acc_s, b)) > 0.25
