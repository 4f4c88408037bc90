"""float64 references and per-element error bars for the stages of the transformer heads (test_heads_gpu.py,
test_heads_stages_gpu.py, and their CPU self-check test_heads_reference_cpu.py).  Device-agnostic torch: the GPU tests
evaluate them in float64 on the device.

Each stage is referenced from the operands the kernel reads, so what remains between the kernel and the reference is
what the kernel itself rounds:

  * linear layers (in-projection, out-projection + residual, FF1 + ReLU, FF2 + residual) run on gemm_layer_launch
    (linear_ws_kernel, or gemm_tile_kernel's 128 x 128 tile) with the epilogue order of the encoder's convolutions
    (+bias, +residual, ReLU, one fp16 rounding) and K = 512, 32 wgmma steps of K = 16: encoder_reference.epilogue and
    encoder_reference.bar with steps = LINEAR_STEPS;
  * attention, LayerNorm and the token reductions: the bars below, each derived where it is defined.
"""
import math

import torch
import torch.nn.functional as F

import encoder_reference as enc

U16 = enc.U16  # unit roundoff of fp16
U32 = enc.U32  # unit roundoff of fp32
SCALE = 1.0 / math.sqrt(128)
LN_EPS = 1e-5
LINEAR_STEPS = 512 // 16  # K = 16 wgmma steps of a K = 512 linear layer


# ----------------------------------------------------------------------------------------------------------------------
# linear layers
# ----------------------------------------------------------------------------------------------------------------------
def linear_terms(x, w, k0=0, k1=512):
    """float64 x @ w^T and |x| @ |w|^T over input channels [k0, k1): x [rows, K] (any float dtype), w [Cout, K]."""
    xd, wd = x[:, k0:k1].double(), w[:, k0:k1].double()
    return xd @ wd.t(), xd.abs() @ wd.abs().t()


def linear(x, w, b, res=None, relu=False):
    """y = relu(x w^T + b + res) in float64 and its per-element bar (encoder_reference.bar, 32 steps)."""
    acc, mag = linear_terms(x, w)
    y = enc.epilogue(acc, b, res, relu=relu)
    return y, enc.bar(y, acc, mag, b, LINEAR_STEPS, res)


def neighbour_panel(b):
    """Bias whose 128-channel panels are swapped pairwise (panel p gets panel p ^ 1's): the probe of a wrong panel."""
    return b.reshape(-1, 128)[torch.arange(b.numel() // 128, device=b.device) ^ 1].reshape(-1)


# ----------------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------------
def attention(qkv, B, G, g, b0, b1):
    """float64 attention of sequences [b0, b1) of group g from the same fp16 q, k, v -> [b, 400, 4, 128] tensors:
    o_ref, P_ref @ |V| (row-normalised), the subnormal term, and the two probes (o with the last 80 keys dropped for
    query tile 3, o with P rounded through bfloat16).  qkv: [B*400, >= G*1536], group g's q | k | v at columns
    1536 g + (0, 512, 1024), 4 heads of 128 each."""
    x = qkv.view(B, 400, -1)[b0:b1, :, 1536 * g:1536 * (g + 1)].double().reshape(b1 - b0, 400, 3, 4, 128)
    x = x.permute(2, 0, 3, 1, 4)  # [3, b, head, 400, 128]
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-1, -2)) * SCALE
    p = torch.exp(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = p @ v / l
    pv_abs = p @ v.abs() / l
    sub = 2.0 ** -25 * v.abs().sum(-2, keepdim=True) / l + 2.0 ** -24
    o_bf16 = p.to(torch.bfloat16).double() @ v / l
    s3 = s[:, :, 384:, :320]  # query tile 3 (rows 384..399) without the last 80-key chunk
    p3 = torch.exp(s3 - s3.amax(-1, keepdim=True))
    o_drop = o.clone()
    o_drop[:, :, 384:] = p3 @ v[:, :, :320] / p3.sum(-1, keepdim=True)
    t = lambda a: a.permute(0, 2, 1, 3)  # -> [b, 400, head, 128]
    return t(o), t(pv_abs), t(sub.expand_as(o)), t(o_drop), t(o_bf16)


def attention_bar(o_ref, pv_abs, sub):
    """Per-element bound of attn_tc_kernel (fp_attn_tc.cu) against `attention`.  S = q k^T is exact products summed in
    fp32; P = exp(S - m) is kept in fp32 for the row sum l, but packed to fp16 (relative error <= u = 2^-11, or <= 2^-25
    absolute below fp16's normal range) before P V, which accumulates in fp32.  So O / l = sum_k p~_k v_k with
    |p~_k - p_k| <= u p_k + 2^-25 / l, hence |O / l - o_ref| <= u (P_ref @ |V|) + 2^-25 sum_k |v_k| / l.  The output is
    rounded to fp16: another u |o| (<= u |o_ref| + u^2 (...)), or 2^-24 absolute for subnormal outputs.  Together
        |o - o_ref| <= u (|o_ref| + P_ref @ |V|) + 2^-25 sum_k |v_k| / l + 2^-24.
    The fp32 parts (S, exp2f, alpha rescales, the sums) are a few 2^-24 relative to the same magnitudes; the safety
    factor 1.25 on the u term covers them."""
    return 1.25 * U16 * (o_ref.abs() + pv_abs) + sub


# ----------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ----------------------------------------------------------------------------------------------------------------------
def layernorm(x, gamma, beta):
    """float64 LayerNorm over 512 channels (eps 1e-5) of x [..., 512] and the per-element bound of layernorm_kernel
    (fp_attn.cu): the mean is an fp32 sum of 512 values in a chain 21 deep (16 in-lane adds, 5 shuffles), so
    |dmean| <= 21 u32 mean|x|; the variance sum the same, relative; rsqrtf is within 2 ulp; the affine step adds a few
    roundings.  With z = (x - mean) rstd:  |y - y_ref| <= u16 |y_ref| + |gamma| (|z| 32 u32 + rstd |dmean|) +
    |beta| 2 u32 + 2^-24, and a safety factor 1.25.  Returns (y_ref, bar)."""
    xd, g, b = x.double(), gamma.double(), beta.double()
    ref = F.layer_norm(xd, (512,), g, b, LN_EPS)
    mean = xd.mean(-1, keepdim=True)
    var = xd.var(-1, unbiased=False, keepdim=True)
    rstd = (var + LN_EPS).rsqrt()
    z = (xd - mean) * rstd
    dmean = 21 * U32 * xd.abs().mean(-1, keepdim=True)
    bar = 1.25 * (U16 * ref.abs() + g.abs() * (z.abs() * 32 * U32 + rstd * dmean) + b.abs() * 2 * U32) + 2.0 ** -24
    return ref, bar


def layernorm_var511(x, gamma, beta):
    """The LayerNorm probe: the variance divided by 511 instead of 512 (z off by 1/1022, about 2 u16)."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = xd.var(-1, unbiased=False, keepdim=True)
    return (xd - mean) * (var * 512 / 511 + LN_EPS).rsqrt() * gamma.double() + beta.double()


# ----------------------------------------------------------------------------------------------------------------------
# token reductions
# ----------------------------------------------------------------------------------------------------------------------
# Both reductions (token_reduce_kernel, then the read-out dot product or rowwise_linear_kernel) sum 400 tokens in fp32
# chains about 23 deep (per-warp rows, eight warps, eight token ranges), divide by 400 and take a dot product over 512
# channels 21 deep; the LayerNorm before it costs about 35 u32 relative.  The bound is therefore below 80 u32 of the L1
# magnitude M_j = sum_c |W_jc| mean_t |x_tc| + |b_j|; the bar is 128 u32 M.
TOKEN_BAR_U32 = 128


def token_readout(x, w=None, bias=None, tokens=None):
    """float64 w . mean_t x + bias of x [B, T, 512] (w None: the token mean itself) and its bar, TOKEN_BAR_U32 u32 of
    the L1 magnitude.  tokens: divide the token sum by this count instead of T (the probe of a mean over 399)."""
    xd = x.double()
    m = xd.mean(1) if tokens is None else xd.sum(1) / tokens
    a = xd.abs().mean(1)
    if w is None:
        return m, TOKEN_BAR_U32 * U32 * a
    wd, bd = w.double(), bias.double()
    return m @ wd.t() + bd, TOKEN_BAR_U32 * U32 * (a @ wd.abs().t() + bd.abs())


# ----------------------------------------------------------------------------------------------------------------------
# the stages composed (the CPU self-check ties them to oracle.nets)
# ----------------------------------------------------------------------------------------------------------------------
def refine_stages(tok, w, chunk=8):
    """The refiner heads' stages in float64 on tokens [N, 400, 512], each from the previous stage's float64 output,
    with w the buffers engine.pack_network uploads (torch tensors), in the layout of fp_op_heads: {qkv [M, 3072];
    att, x1pre, x1, ff, x2pre [2, M, 512]; head_out [2, N, 3]}, M = 400 N."""
    N = tok.shape[0]
    t = tok.reshape(N * 400, 512).double()
    qkv, _ = linear(t, w["heads.in_w"], w["heads.in_b"])
    out = {"qkv": qkv}
    for name in ("att", "x1pre", "x1", "ff", "x2pre", "head_out"):
        out[name] = []
    for g in range(2):
        h = lambda s: w[f"head{g}.{s}"]
        att = torch.cat([attention(qkv, N, 2, g, b0, min(N, b0 + chunk))[0] for b0 in range(0, N, chunk)])
        att = att.reshape(N * 400, 512)
        x1pre, _ = linear(att, h("out_w"), h("out_b"), res=t)
        x1, _ = layernorm(x1pre, h("ln1_g"), h("ln1_b"))
        ff, _ = linear(x1, h("ff1_w"), h("ff1_b"), relu=True)
        x2pre, _ = linear(ff, h("ff2_w"), h("ff2_b"), res=x1)
        x2, _ = layernorm(x2pre, h("ln2_g"), h("ln2_b"))
        head_out, _ = token_readout(x2.reshape(N, 400, 512), h("fin_w"), h("fin_b"))
        for name, v in (("att", att), ("x1pre", x1pre), ("x1", x1), ("ff", ff), ("x2pre", x2pre), ("head_out", head_out)):
            out[name].append(v)
    return {k: (torch.stack(v) if isinstance(v, list) else v) for k, v in out.items()}


def score_stages(tok, w, chunk=8):
    """The scorer's stages in float64 on tokens [N, 400, 512]: {qkv, att, tok_mean, feats}."""
    N = tok.shape[0]
    t = tok.reshape(N * 400, 512).double()
    qkv, _ = linear(t, w["att.in_w"], w["att.in_b"])
    att = torch.cat([attention(qkv, N, 1, 0, b0, min(N, b0 + chunk))[0] for b0 in range(0, N, chunk)])
    att = att.reshape(N * 400, 512)
    tok_mean, _ = token_readout(att.reshape(N, 400, 512))
    feats, _ = token_readout(tok_mean[:, None], w["att.out_w32"], w["att.out_b"])
    return {"qkv": qkv, "att": att, "tok_mean": tok_mean, "feats": feats}
