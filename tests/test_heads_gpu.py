"""The transformer-head kernels alone, at the batch sizes the product runs, against float64 references on the GPU.

Each kernel is called through its single-operator hook (fp_api_ops.cu), which runs the product's launcher with the
product's constants.  The bars are per element and derived from what each kernel rounds (see each test); every test
prints its worst ratio of error to bar and checks that its own comparison rejects a slightly wrong reference (a
defect probe) on a stated fraction of the elements.

Unit counts: the attention kernel walks B x 4 heads x G groups x 4 query tiles on 132 persistent CTAs of an H100 SXM,
so B = 1 with two groups (track_one's refiner: 32 units) leaves most CTAs idle and B = 252 with two groups (the
refiner at 252 hypotheses) gives every CTA 61 or 62 units, with the Q ring's phase flipping on every second unit.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import heads_reference as ref

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_cached_memory():
    # the float64 references are large: hand their cached blocks back to the device after each test
    yield
    torch.cuda.empty_cache()


def _report(what, err, bar):
    ratio = (err / bar).max().item()
    print(f"{what}: worst error / bar = {ratio:.3f}")
    return ratio


def _probe_fraction(err, bar):
    return (err > bar).double().mean().item()


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
def _attn_inputs(B, G, seed):
    """fp16 [B*400, G*1536]: group g's q | k | v at columns 1536 g + (0, 512, 1024), 4 heads of 128 each.  Head h of
    sequence b gets class (b + h) % 4:
      0  q, k, v of scale 1.5: moderate logits (std ~ 2), tens of keys share each row's weight
      1  scale 4: large logits (std ~ 16), nearly one-hot rows
      2  the keys of the last 80-key chunk three times larger: most rows meet their maximum in the last chunk, so
         the online softmax rescales everything accumulated before it
      3  q = 0 on odd rows: exactly uniform weights over the 400 keys"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 400, G, 3, 4, 128, generator=gen, device="cuda", dtype=torch.float16)
    cls = (torch.arange(B, device="cuda")[:, None] + torch.arange(4, device="cuda")[None]) % 4  # [B, head]
    x *= torch.tensor([1.5, 4.0, 1.0, 1.5], device="cuda", dtype=torch.float16)[cls][:, None, None, None, :, None]
    x[:, 320:, :, 1] *= torch.where(cls == 2, 3.0, 1.0).half()[:, None, None, :, None]
    odd = (torch.arange(400, device="cuda") % 2 == 1)[None, :, None, None, None]
    x[:, :, :, 0] *= torch.where((cls == 3)[:, None, None, :, None] & odd, 0.0, 1.0).half()
    return x.reshape(B * 400, G * 1536)


@pytest.mark.parametrize("G", [1, 2], ids=lambda g: f"G{g}")
@pytest.mark.parametrize("B", [1, 3, 66, 67, 249, 252], ids=lambda b: f"B{b}")
def test_attention_groups(B, G):
    """attn_tc_kernel (fp_attn_tc.cu) through fp_op_attention_groups, the launch of run_refine_heads (G = 2, ld 3072)
    and run_score_feats (G = 1, ld 1536), against float64 softmax(q k^T / sqrt(128)) v on the same fp16 q, k, v.

    Error bound per output element: heads_reference.attention_bar,
        |o - o_ref| <= 1.25 u (|o_ref| + P_ref @ |V|) + 2^-25 sum_k |v_k| / l + 2^-24,
    derived there.  Measured on an H100: at most 0.75 of this bar over the whole grid.

    Probes: dropping the last 80-key chunk for query tile 3 must fail on more than half of tile 3's elements (81 to 89 %
    measured); rounding P through bfloat16 (4x fp16's rounding) must fail on more than 1 % of all elements (3.6 to
    3.9 % measured: the rounding errors of many keys average out, so only rows with a few dominant keys
    show it).  Both launches must be bit-equal, and with two groups each group's output must equal, bit for bit, a
    one-group launch on that group's column block (pointer advanced by 1536 g columns, ld still 3072)."""
    from foundationpose_b200 import ops

    qkv = _attn_inputs(B, G, seed=1000 + 10 * B + G)
    out = ops.attention_groups(qkv, B, G)
    assert torch.equal(out, ops.attention_groups(qkv, B, G)), "two launches differ"
    if G == 2:
        for g in range(2):
            alone = ops.attention_groups(qkv[:, 1536 * g:], B, 1, ld=3072)
            assert torch.equal(alone[0], out[g]), f"group {g} differs from a one-group launch of its columns"
    worst, n_bf16, n_drop, n_all, n_tile3 = 0.0, 0, 0, 0, 0
    chunk = 12
    for g in range(G):
        got = out[g].view(B, 400, 4, 128)
        for b0 in range(0, B, chunk):
            b1 = min(B, b0 + chunk)
            o_ref, pv_abs, sub, o_drop, o_bf16 = ref.attention(qkv, B, G, g, b0, b1)
            bar = ref.attention_bar(o_ref, pv_abs, sub)
            o = got[b0:b1].double()
            err = (o - o_ref).abs()
            bad = err > bar
            if bad.any():
                idx = bad.nonzero()[0].tolist()
                pytest.fail(f"B={B} G={G} group {g}: {int(bad.sum())} elements over the bar, first at "
                            f"(sequence {b0 + idx[0]}, row {idx[1]}, head {idx[2]}, dim {idx[3]}): "
                            f"err {err[tuple(idx)].item():.3g} bar {bar[tuple(idx)].item():.3g}")
            worst = max(worst, (err / bar).max().item())
            n_bf16 += int(((o - o_bf16).abs() > bar).sum())
            n_drop += int(((o - o_drop).abs() > bar)[:, 384:].sum())
            n_all += o.numel()
            n_tile3 += o[:, 384:].numel()
    print(f"attention B={B} G={G}: worst error / bar = {worst:.3f}, bf16-P probe fails {n_bf16 / n_all:.2%}, "
          f"dropped-chunk probe fails {n_drop / n_tile3:.2%} of tile 3")
    assert n_drop > 0.5 * n_tile3, "the bar does not see query tile 3 missing its last key chunk"
    assert n_bf16 > 0.01 * n_all, "the bar does not see P rounded through bfloat16"


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [400, 67 * 400, 100800, 100803])
def test_layernorm(rows):
    """layernorm_kernel (fp_attn.cu) through fp_op_layernorm against float64 F.layer_norm on the same fp16 rows.
    100 800 rows = 252 hypotheses x 400 tokens; 100 803 gives some warps one more trip round the grid-stride loop.

    Edge rows: row 1 is constant (mean exact, variance 0: the output must be beta rounded to fp16, exactly); row 2 has
    mean ~1000 and spread ~1 (cancellation); row 3 has values near +-6e4 (squares near 4e9).

    Error bound: heads_reference.layernorm, derived there.  Probe: the variance divided by 511 instead of 512 (z off
    by 1/1022, about 2 u16) must fail on more than half of the elements (88 % measured; at most 0.80 of the bar
    reached)."""
    from foundationpose_b200 import ops

    gen = torch.Generator(device="cuda").manual_seed(rows)
    x = torch.randn(rows, 512, generator=gen, device="cuda")
    gamma = 1.0 + 0.1 * torch.randn(512, generator=gen, device="cuda")
    beta = 0.1 * torch.randn(512, generator=gen, device="cuda")
    x[1] = 0.7
    x[2] = 1000.0 + torch.randn(512, generator=gen, device="cuda")
    x[3] = torch.sign(torch.randn(512, generator=gen, device="cuda")) * (5e4 + 1.5e4 * torch.rand(512, generator=gen, device="cuda"))
    x16 = x.half()
    y = ops.layernorm(x16, gamma, beta).double()
    assert torch.equal(y[1], beta.half().double()), "a constant row must give beta rounded to fp16"
    y_ref, bar = ref.layernorm(x16, gamma, beta)
    err = (y - y_ref).abs()
    ratio = _report(f"layernorm rows={rows}", err, bar)
    assert ratio <= 1.0, f"layernorm rows={rows}: {int((err > bar).sum())} elements over the bar, first row {int((err > bar).any(-1).nonzero()[0])}"
    probe = ref.layernorm_var511(x16, gamma, beta)
    frac = _probe_fraction((y - probe).abs(), bar)
    print(f"layernorm rows={rows}: variance/511 probe fails {frac:.2%}")
    assert frac > 0.5, "the bar does not see the variance divided by 511"


# ------------------------------------------------------------------------------------------------------------------
# token reductions
# ------------------------------------------------------------------------------------------------------------------
def _tokens(B, seed):
    """fp16 [B, 400, 512]: a per-sequence channel profile plus per-token noise, so the token mean is of the order of
    the tokens themselves (as in trained features) rather than 1/20 of them."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(B, 1, 512, generator=gen, device="cuda")
    return (base + 0.5 * torch.randn(B, 400, 512, generator=gen, device="cuda")).half()


# Both reductions are held to heads_reference.TOKEN_BAR_U32 u32 of the L1 magnitude M_j = sum_c |W_jc| mean_t |x_tc| +
# |b_j| (derived there).


@pytest.mark.parametrize("B", [1, 66, 67, 252])
def test_head_final(B):
    """token_reduce_kernel<true> (fp_attn.cu) through fp_op_head_final with out_dim 3: norm2 -> token mean ->
    Linear(512, 3) of one refiner head, against float64.  B <= 66 takes the eight-CTA cluster launch on an H100 SXM's
    132 SMs, B >= 67 one CTA per sequence (token_split_for).  Bar: 128 u32 of the L1 magnitude (see TOKEN_BAR_U32).
    Probe: the mean over 399 tokens instead of 400 must fail on more than 60 % of the outputs (95 to 100 % measured;
    it misses only outputs whose token mean nearly cancels in the dot product).  The measured errors stay below 0.005
    of the bar: the bar is a worst-case bound on fp32 sums whose rounding errors mostly cancel."""
    from foundationpose_b200 import ops

    x = _tokens(B, 7 + B)
    gen = torch.Generator(device="cuda").manual_seed(B)
    gamma = 1.0 + 0.1 * torch.randn(512, generator=gen, device="cuda")
    beta = 0.1 * torch.randn(512, generator=gen, device="cuda")
    w = torch.randn(3, 512, generator=gen, device="cuda") / math.sqrt(512)
    bias = 0.01 * torch.randn(3, generator=gen, device="cuda")
    out = ops.head_final(x, gamma, beta, w, bias).double()
    ln = F.layer_norm(x.double(), (512,), gamma.double(), beta.double(), 1e-5)
    y_ref, bar = ref.token_readout(ln, w, bias)
    err = (out - y_ref).abs()
    assert _report(f"head_final B={B}", err, bar) <= 1.0
    probe, _ = ref.token_readout(ln, w, bias, tokens=399)
    frac = _probe_fraction((out - probe).abs(), bar)
    print(f"head_final B={B}: 399-token probe fails {frac:.2%}")
    assert frac > 0.6, "the bar does not see a mean over 399 tokens"


@pytest.mark.parametrize("B", [1, 66, 67, 249, 252])
def test_token_mean_proj(B):
    """token_reduce_kernel<false> + rowwise_linear_kernel (fp_attn.cu) through fp_op_token_mean_proj: the scorer's
    token mean -> out_proj, against float64.  B = 249 leaves a last block of 1 of rowwise_linear's 8-row blocks.  Bar
    and probe as in test_head_final."""
    from foundationpose_b200 import ops

    x = _tokens(B, 11 + B)
    gen = torch.Generator(device="cuda").manual_seed(100 + B)
    w = torch.randn(512, 512, generator=gen, device="cuda") / math.sqrt(512)
    bias = 0.01 * torch.randn(512, generator=gen, device="cuda")
    out = ops.token_mean_proj(x, w, bias).double()
    y_ref, bar = ref.token_readout(x, w, bias)
    err = (out - y_ref).abs()
    assert _report(f"token_mean_proj B={B}", err, bar) <= 1.0
    probe, _ = ref.token_readout(x, w, bias, tokens=399)
    frac = _probe_fraction((out - probe).abs(), bar)
    print(f"token_mean_proj B={B}: 399-token probe fails {frac:.2%}")
    assert frac > 0.6, "the bar does not see a mean over 399 tokens"


# ------------------------------------------------------------------------------------------------------------------
# both heads at product N, from the GPU's own tokens
# ------------------------------------------------------------------------------------------------------------------
# weights the engine keeps in fp16 (engine.pack_network); the float64 reference uses the same rounded values, so what
# remains is the heads' fp16 activations and the glue between the kernels
_FP16_WEIGHTS = ("self_attn.in_proj_weight", "self_attn.out_proj.weight", "linear1.weight", "linear2.weight",
                 "att.in_proj_weight")


@pytest.fixture(scope="module")
def heads_engine():
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    sds = {}
    for kind in ("refine", "score"):
        sd = random_state_dict(kind, 0)
        e.load_network(kind, sd)
        sds[kind] = {k: (v.half() if k.endswith(_FP16_WEIGHTS) else v).double().cuda() for k, v in sd.items()
                     if torch.is_floating_point(v)}
    yield e, sds
    e.close()


def _random_crops(N, seed):
    from foundationpose_b200.engine import crops_from_planar

    gen = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.rand(N, 6, 160, 160, generator=gen, device="cuda")
    B = torch.rand(N, 6, 160, 160, generator=gen, device="cuda")
    for T in (A, B):
        T[:, 3:] = (T[:, 3:] - 0.5) * 2
        T[:, 3:, :30] = 0
    return crops_from_planar(A, B)


def _refine_heads_reference(tok, sd, chunk=24):
    """oracle.nets' refiner heads (encoder layer -> Linear(512, 3) -> token mean) in float64 on fp16 tokens."""
    from oracle import nets

    outs = {"trans": [], "rot": []}
    for b0 in range(0, tok.shape[0], chunk):
        t = tok[b0:b0 + chunk].double()
        for name, head in (("trans", "trans_head"), ("rot", "rot_head")):
            y = nets.encoder_layer(t, sd, f"{head}.0")
            outs[name].append((y @ sd[f"{head}.1.weight"].t() + sd[f"{head}.1.bias"]).mean(dim=1))
    return torch.cat(outs["trans"]), torch.cat(outs["rot"])


def _score_feats_reference(tok, sd, chunk=24):
    from oracle import nets

    return torch.cat([nets.mha(tok[b0:b0 + chunk].double(), sd, "att").mean(dim=1) for b0 in range(0, tok.shape[0], chunk)])


# Absolute bars.  Worst errors measured on an H100 80GB HBM3 (700 W) with these weights and inputs, at N = 67 / 252:
# trans 4.6e-6 / 4.3e-6, rot 3.5e-6 / 3.9e-6, scorer features 7.9e-4 / 1.13e-3 (features up to 7.2 in magnitude).
# Each bar is under three times the worst of them.
HEADS_BAR = {"trans": 1.2e-5, "rot": 1.2e-5, "feats": 3e-3}


@pytest.mark.parametrize("N", [67, 252])
def test_heads_at_product_n(N, heads_engine):
    """fp_op_refine_net / fp_op_score_feats at N = 252 (the refiner's heads one after the other) and N = 67 (heads
    forked onto two streams) against oracle.nets' heads run in float64 on the tokens fp_op_encoder returns for the same
    crops.  This isolates the glue at product N: the 3072-wide in_proj, the group offsets of run_refine_heads and the
    out_proj -> LayerNorm -> feed-forward -> LayerNorm chain with its fp16 intermediates.  Bars: absolute, HEADS_BAR.
    Probe: a reference whose rot head is fed the trans head's attention output (the rot head's in_proj replaced by the
    trans head's) must fail on more than half of the rot outputs."""
    e, sds = heads_engine
    crops = _random_crops(N, 40 + N)
    tok = e.op_encoder("refine", crops, N).reshape(N, 400, 512)
    trans, rot = e.op_refine_net(crops, N)
    sd = sds["refine"]
    ref_t, ref_r = _refine_heads_reference(tok, sd)
    err_t = (trans.double() - ref_t).abs().max().item()
    err_r = (rot.double() - ref_r).abs().max().item()
    tok_s = e.op_encoder("score", crops, N).reshape(N, 400, 512)
    feats = e.op_score_feats(crops, N)
    ref_f = _score_feats_reference(tok_s, sds["score"])
    err_f = (feats.double() - ref_f).abs().max().item()
    print(f"heads N={N}: max |err| trans {err_t:.3e}, rot {err_r:.3e}, scorer features {err_f:.3e} "
          f"(|feats| max {ref_f.abs().max().item():.3g}); worst error / bar = "
          f"{max(err_t / HEADS_BAR['trans'], err_r / HEADS_BAR['rot'], err_f / HEADS_BAR['feats']):.3f}")
    assert err_t <= HEADS_BAR["trans"] and err_r <= HEADS_BAR["rot"] and err_f <= HEADS_BAR["feats"]
    crossed = dict(sd)
    for k in ("in_proj_weight", "in_proj_bias"):
        crossed[f"rot_head.0.self_attn.{k}"] = sd[f"trans_head.0.self_attn.{k}"]
    _, probe_r = _refine_heads_reference(tok, crossed)
    frac = _probe_fraction((rot.double() - probe_r).abs(), HEADS_BAR["rot"])
    print(f"heads N={N}: crossed-group probe fails {frac:.2%} of the rot outputs")
    assert frac > 0.5, "the bar does not see the rot head reading the trans head's attention"
