"""CPU: the stage-by-stage references of tests/heads_reference.py, composed, are the heads of oracle.nets.

test_heads_stages_gpu.py holds every stage of the heads to its own float64 reference, each computed from the previous
stage's GPU output.  Those references only add up to the network if their composition is the network: here, in float64
on seeded weights held as engine.pack_network uploads them (fp16 projection weights, fp32 the rest), the refiner's
stages must give oracle.nets.encoder_layer -> Linear(512, 3) -> token mean of both heads, and the scorer's
oracle.nets.mha -> token mean, to float64 rounding.  oracle.nets is itself held to the reference's network classes
(tests/test_oracle_golden.py).
"""
import pytest
import torch

import heads_reference as ref

N = 3
# weights the engine keeps in fp16: the oracle runs on their rounded values
_FP16_WEIGHTS = ("self_attn.in_proj_weight", "self_attn.out_proj.weight", "linear1.weight", "linear2.weight",
                 "att.in_proj_weight")


def _setup(kind):
    from foundationpose_b200.engine import pack_network
    from foundationpose_b200.weights import random_state_dict

    sd = random_state_dict(kind, 6)
    packed = {k: torch.from_numpy(v) for k, v in pack_network(sd, kind).items()}
    sd64 = {k: (v.half() if k.endswith(_FP16_WEIGHTS) else v).double() for k, v in sd.items() if torch.is_floating_point(v)}
    g = torch.Generator().manual_seed(11)
    base = torch.randn(N, 1, 512, generator=g)
    tok = (base + torch.randn(N, 400, 512, generator=g)).half()
    return tok, packed, sd64


def _close(got, want, what):
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    print(f"{what}: max |composition - oracle| = {err:.3g} (max |oracle| {scale:.3g})")
    assert err <= 1e-12 * max(1.0, scale), f"{what}: the stages do not compose to the oracle ({err:.3g})"


def test_refine_stages_compose_to_the_oracle():
    from oracle import nets

    tok, w, sd = _setup("refine")
    st = ref.refine_stages(tok, w)
    assert st["qkv"].shape == (N * 400, 3072) and st["x2pre"].shape == (2, N * 400, 512) and st["head_out"].shape == (2, N, 3)
    t = tok.double()
    for g, head in enumerate(("trans_head", "rot_head")):
        p = f"{head}.0"
        # the in-projection and attention of the oracle's mha, written out to reach its intermediate values
        qkv = t @ sd[f"{p}.self_attn.in_proj_weight"].t() + sd[f"{p}.self_attn.in_proj_bias"]
        _close(st["qkv"][:, 1536 * g:1536 * (g + 1)].reshape(N, 400, 1536), qkv, f"{head} qkv")
        y = nets.encoder_layer(t, sd, p)
        ln2 = torch.nn.functional.layer_norm(st["x2pre"][g].reshape(N, 400, 512), (512,), sd[f"{p}.norm2.weight"],
                                             sd[f"{p}.norm2.bias"], 1e-5)
        _close(ln2, y, f"{head} LayerNorm 2 of x2pre")
        out = (y @ sd[f"{head}.1.weight"].t() + sd[f"{head}.1.bias"]).mean(dim=1)
        _close(st["head_out"][g], out, f"{head} head_out")


def test_score_stages_compose_to_the_oracle():
    from oracle import nets

    tok, w, sd = _setup("score")
    st = ref.score_stages(tok, w)
    t = tok.double()
    qkv = t @ sd["att.in_proj_weight"].t() + sd["att.in_proj_bias"]
    _close(st["qkv"].reshape(N, 400, 1536), qkv, "scorer qkv")
    _close(st["feats"], nets.mha(t, sd, "att").mean(dim=1), "scorer features")


@pytest.mark.parametrize("relu", [False, True])
def test_linear_bar_accepts_the_kernel_rounding(relu):
    """A CPU emulation of one K = 512 linear layer as the kernels round it (fp16 operands, each K = 16 slice summed in
    fp32 and added to an fp32 accumulator, + bias, + residual, ReLU, one fp16 rounding) passes the bar of
    heads_reference.linear, and dropping K block 448..511 fails it on most elements."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(256, 512, generator=g).half()
    w = (torch.randn(384, 512, generator=g) / 512 ** 0.5).half()
    b = torch.randn(384, generator=g) * 0.05
    res = torch.randn(256, 384, generator=g).half()
    acc = torch.zeros(256, 384)
    for k0 in range(0, 512, 16):
        acc += x[:, k0:k0 + 16].float() @ w[:, k0:k0 + 16].float().t()
    a = acc + b + res.float()
    got = (a.clamp_min(0) if relu else a).half().double()
    y, bar = ref.linear(x, w, b, res=res, relu=relu)
    err = (got - y).abs()
    assert (err <= bar).all(), f"emulated layer over the bar: worst error / bar {(err / bar).max().item():.3f}"
    assert (err / bar).max() > 0.01, "the bar is far looser than the rounding it bounds"
    acc_d, _ = ref.linear_terms(x, w)
    drop, _ = ref.linear_terms(x, w, 448, 512)
    probe = ref.enc.epilogue(acc_d - drop, b, res, relu=relu)
    frac = ((got - probe).abs() > bar).double().mean().item()
    assert frac > (0.4 if relu else 0.9), f"dropping K block 448..511 fails only {frac:.1%}"
