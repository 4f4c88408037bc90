"""float64 references and per-element error bars for the encoder's convolutions (test_encoder_cpu.py,
test_encoder_gpu.py).

A layer computes  y = relu(conv(x, w) + b + res) + pe  (the epilogue order of fp_gemm.cu and fp_stem.cu) from fp16
activations x, fp16 weights w, fp32 bias b, an optional fp16 residual res and an optional fp32 positional embedding
pe, and rounds y to fp16 once.  The references here take exactly those operands, so what is left between the kernel
and the reference is what the kernel rounds:

  * the products x w: exact (an fp16 x fp16 product has 22 significant bits);
  * their fp32 accumulation: each wgmma step adds one K = 16 slice, 16 exact products, to the fp32 accumulator.
    Tensor cores of earlier generations were found to do that as one multi-operand addition that aligns all 17
    addends to the largest exponent and truncates, so each addend may lose up to one fp32 ulp of the largest:
    17 2^-23 of the magnitudes summed so far per step, at most ADDENDS k_steps 2^-23 conv(|x|, |w|) in all.  A model
    of one rounding per step (k_steps 2^-23 conv(|x|, |w|)) is too tight on an H100: the printed ratio "beyond the
    output's rounding" measured up to 4 against it, so the H100's adder is taken to behave like the earlier ones;
  * the epilogue's fp32 adds (bias, residual, positional embedding): at most three roundings of partial sums bounded
    by |acc| + |b| + |res| + |pe|, taken four times;
  * the fp16 rounding of y: u16 |y| for normal outputs, at most 2^-25 below fp16's normal range (the 2^-24 term).

    bar = u16 |y_ref| + 17 k_steps 2^-23 conv(|x|, |w|) + 4 2^-24 (|acc| + |b| + |res| + |pe|) + 2^-24

ReLU does not add error (|relu(a) - relu(b)| <= |a - b|).  The bar is a bound derived from these roundings, not a
fit to a measurement: a layer that exceeds it has a defect to find.
"""
import torch
import torch.nn.functional as F

U16 = 2.0 ** -11  # unit roundoff of fp16
U32 = 2.0 ** -24  # unit roundoff of fp32
TC_ULP = 2.0 ** -23  # one fp32 ulp, truncated rather than rounded
ADDENDS = 17  # per wgmma step: the accumulator and one K = 16 slice of products

LK_CONV3_S1, LK_CONV3_S2, LK_CONV7_S2 = 1, 2, 3


def unpack_conv3(wp):
    """Inverse of packing.pack_conv3: (Co, 9 Ci) with K ordered (r, s, c) -> (Co, Ci, 3, 3), same dtype."""
    co = wp.shape[0]
    return wp.reshape(co, 3, 3, wp.shape[1] // 9).permute(0, 3, 1, 2).contiguous()


def unpack_conv7(wp):
    """Inverse of packing.pack_conv7: (7, 4, 2, Co, 8) = [filter row][tap pair][tap of the pair][Co][8 ch] ->
    (Co, 8, 7, 7), same dtype.  Tap 7 of each row is dropped (pack_conv7 writes zeros there; re-packing shows it) and
    all 8 input channels are kept (channels >= Ci are the zero pad)."""
    co = wp.shape[3]
    return wp.reshape(7, 8, co, 8)[:, :7].permute(2, 3, 0, 1).contiguous()


def k_steps(kind, cin):
    """K = 16 wgmma steps per output: 7 filter rows x 4 tap pairs of 8 channels for the stem (fp_stem.cu), 9 Cin / 16
    for a 3x3 convolution (fp_gemm.cu)."""
    return 28 if kind == LK_CONV7_S2 else 9 * cin // 16


def _columns(x, kind, shift):
    """x NHWC -> float64 im2col columns (n, Cin k k, Ho Wo), K ordered (c, r, s) like a (Co, Ci, k, k) filter.
    Stem: x is the padded crop canvas (n, 166, 168, 8) with the image at (3, 3), read without further padding.
    shift: the window one input pixel down and right (the probe of the stride-2 layers)."""
    xd = x.permute(0, 3, 1, 2).double()
    if kind == LK_CONV7_S2:
        o = 1 if shift else 0
        return F.unfold(xd[:, :, o:o + 165, o:o + 165], 7, stride=2)  # 7 + 2 x 79 = 165 rows and columns
    if kind == LK_CONV3_S1:
        return F.unfold(xd, 3, padding=1)
    if shift:
        return F.unfold(F.pad(xd, (0, 2, 0, 2)), 3, stride=2)
    return F.unfold(xd, 3, padding=1, stride=2)


def out_hw(kind, H):
    return H if kind == LK_CONV3_S1 else (80 if kind == LK_CONV7_S2 else H // 2)


def conv_terms(x, w, kind, H, shift=False):
    """float64 conv(x, w), conv(|x|, |w|) and the contribution of filter tap (2, 2) alone, each NHWC (n, Ho, Wo, Co),
    on x's device.  x fp16 NHWC (the stem: the padded canvas), w (Co, Ci, k, k) holding the kernel's fp16 values."""
    co, ci, kk = w.shape[0], w.shape[1], w.shape[2]
    cols = _columns(x, kind, shift)
    wd = w.to(device=x.device, dtype=torch.float64).reshape(co, -1)
    ho = out_hw(kind, H)
    nhwc = lambda t: t.transpose(1, 2).reshape(x.shape[0], ho, ho, co)
    acc = nhwc(wd @ cols)
    tap = torch.arange(ci, device=x.device) * kk * kk + 2 * kk + 2
    tap22 = nhwc(wd[:, tap] @ cols[:, tap])
    cols.abs_()
    mag = nhwc(wd.abs() @ cols)
    return acc, mag, tap22


def epilogue(acc, b, res=None, pe=None, relu=True):
    """relu(acc + b + res) + pe in float64; b (Co,), res like acc, pe (Ho, Wo, Co).  relu=False: the linear layers
    without ReLU (tests/heads_reference.py)."""
    y = acc + b.double()
    if res is not None:
        y = y + res.double()
    if relu:
        y = y.clamp_min(0.0)
    if pe is not None:
        y = y + pe.double()
    return y


def half_ulp16(y):
    """Half an fp16 ulp at the fp16 values y (2^-25 below fp16's normal range): the most rounding y to fp16 can move."""
    e = torch.floor(torch.log2(y.double().abs().clamp_min(2.0 ** -14)))
    return 2.0 ** (e - 11)


def bar(y_ref, acc, mag, b, steps, res=None, pe=None):
    """The per-element bound of the module docstring."""
    s = acc.abs() + b.double().abs()
    if res is not None:
        s = s + res.double().abs()
    if pe is not None:
        s = s + pe.double().abs()
    return U16 * y_ref.abs() + ADDENDS * steps * TC_ULP * mag + 4 * U32 * s + U32
