"""GPU parity of the whole network paths (15 wgmma conv layers + attention heads) against the fp32
CPU oracle (oracle/nets.py, pinned to the reference classes by tests/test_oracle_golden.py) on
identical pre-built crops and identical seeded weights.

Tolerances (stated per BASELINE.json north_star): the engine computes in fp16 with fp32 accumulation
like the reference's autocast path; against the fp32 oracle the raw network outputs agree to 5e-3
absolute (|outputs| ~ 0.5), i.e. < 1e-3 on the SE(3) delta after the x(diameter/2) / x0.349
scaling (checked in test_pipeline_gpu.py).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _crops(n, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.rand(n, 6, 160, 160, generator=g)
    B = torch.rand(n, 6, 160, 160, generator=g)
    for T in (A, B):
        T[:, 3:] = (T[:, 3:] - 0.5) * 2
        T[:, 3:, :30] = 0
    return A, B


@pytest.fixture(scope="module")
def engine():
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    sd_r = random_state_dict("refine", 0)
    sd_s = random_state_dict("score", 0)
    e.load_network("refine", sd_r)
    e.load_network("score", sd_s)
    return e, sd_r, sd_s


def test_refine_tokens(engine):
    from foundationpose_b200.engine import crops_from_planar
    from oracle import nets

    e, sd_r, _ = engine
    A, B = _crops(3, 11)
    tok = e.op_encoder("refine", crops_from_planar(A.cuda(), B.cuda()), 3).reshape(3, 400, 512).float().cpu()
    # oracle sees the same fp16-rounded inputs
    A16, B16 = A.half().float(), B.half().float()
    x = nets.encode_a(torch.cat([A16, B16], 0), sd_r, "encodeA")
    ab = nets.encode_ab(torch.cat((x[:3], x[3:]), 1), sd_r, "encodeAB")
    ref = nets._tokens(ab, sd_r)
    err = (tok - ref).abs()
    scale = ref.abs().max().item()
    assert err.max().item() < 0.02 * scale, f"token max err {err.max().item()} vs scale {scale}"
    assert err.mean().item() < 2e-3 * scale


def test_refine_net_outputs(engine):
    from foundationpose_b200.engine import crops_from_planar
    from oracle import nets

    e, sd_r, _ = engine
    A, B = _crops(3, 12)
    trans, rot = e.op_refine_net(crops_from_planar(A.cuda(), B.cuda()), 3)
    ref = nets.refine_forward(sd_r, A.half().float(), B.half().float())
    np.testing.assert_allclose(trans.cpu().numpy(), ref["trans"].numpy(), atol=5e-3, rtol=0)
    np.testing.assert_allclose(rot.cpu().numpy(), ref["rot"].numpy(), atol=5e-3, rtol=0)


def test_token_reduction_is_bitwise_the_same_as_cluster_or_single_cta(engine):
    """fp_attn.cu token_reduce_kernel: a cluster of eight CTAs per hypothesis while B * 8 <= 4 * SMs
    (token_split_for), one CTA walking the same eight token ranges above.  Same partial sums, same order: the read-outs
    of the largest batch that takes the cluster launch must not change by a bit when 8 more hypotheses push the batch
    onto the single-CTA launch (refiner heads and scorer features)."""
    from foundationpose_b200.engine import crops_from_planar

    e, _, _ = engine
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_cluster = (4 * sms) // 8  # largest B with B * 8 <= 4 * SMs
    n_single = n_cluster + 8
    assert n_cluster * 8 <= 4 * sms < n_single * 8
    A, B = _crops(n_single, 21)
    big = crops_from_planar(A.cuda(), B.cuda())
    small = crops_from_planar(A[:n_cluster].cuda(), B[:n_cluster].cuda())
    t_big, r_big = e.op_refine_net(big, n_single)
    t_small, r_small = e.op_refine_net(small, n_cluster)
    assert torch.equal(t_big[:n_cluster], t_small) and torch.equal(r_big[:n_cluster], r_small)
    f_big = e.op_score_feats(big, n_single)
    f_small = e.op_score_feats(small, n_cluster)
    assert torch.equal(f_big[:n_cluster], f_small)


def test_refine_net_golden(engine):
    """Same crops as the reference-generated golden fixture (tools/make_golden.py)."""
    import os

    from foundationpose_b200.engine import crops_from_planar

    e, _, _ = engine
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "nets_golden.npz"))
    g = torch.Generator().manual_seed(123)
    A = torch.rand(2, 6, 160, 160, generator=g)
    B = torch.rand(2, 6, 160, 160, generator=g)
    for T in (A, B):
        T[:, 3:] = (T[:, 3:] - 0.5) * 2
        T[:, 3:, :30] = 0
    trans, rot = e.op_refine_net(crops_from_planar(A.cuda(), B.cuda()), 2)
    np.testing.assert_allclose(trans.cpu().numpy(), gold["refine_trans"], atol=5e-3, rtol=0)
    np.testing.assert_allclose(rot.cpu().numpy(), gold["refine_rot"], atol=5e-3, rtol=0)


def test_score_feats_and_tail(engine):
    from foundationpose_b200.engine import crops_from_planar
    from oracle import nets

    e, _, sd_s = engine
    A, B = _crops(5, 13)
    feats = e.op_score_feats(crops_from_planar(A.cuda(), B.cuda()), 5)
    ref_feats = nets.score_features(sd_s, A.half().float(), B.half().float())
    scale = ref_feats.abs().max().item()
    assert (feats.cpu() - ref_feats).abs().max().item() < 0.01 * scale
    # tail on identical (oracle) features: fp32 SIMT vs fp32 torch
    scores, best = e.score_tail(ref_feats.cuda())
    ref_logits = nets.score_tail(sd_s, ref_feats, 5).reshape(-1)
    # fp32 on both sides: the bar is relative to the magnitude of the logits (the stand-in read-out is scaled x60)
    np.testing.assert_allclose(scores.cpu().numpy() - 100.0, ref_logits.numpy(), atol=2e-5 * float(ref_logits.abs().max()) + 2e-5, rtol=0)
    assert int(best.item()) == int(ref_logits.argmax())


def test_score_tail_252(engine):
    """Cross-hypothesis attention at the real L=252 with random features; index must match."""
    from oracle import nets

    e, _, sd_s = engine
    g = torch.Generator().manual_seed(5)
    feats = torch.randn(252, 512, generator=g) * 2
    scores, best = e.score_tail(feats.cuda())
    ref = nets.score_tail(sd_s, feats, 252).reshape(-1)
    np.testing.assert_allclose(scores.cpu().numpy() - 100.0, ref.numpy(), atol=2e-5 * float(ref.abs().max()) + 2e-5, rtol=0)
    assert int(best.item()) == int(ref.argmax())


def test_attention_core(impl=1):
    """softmax(QK^T/sqrt(128))V for 400 tokens x 4 heads vs torch fp32 on the same fp16 q, k, v."""
    from foundationpose_b200 import ops

    g = torch.Generator().manual_seed(21 + impl)
    B = 3
    qkv = (torch.randn(B * 400, 1536, generator=g) * 1.5).half().cuda()
    out = ops.attention(qkv, impl=impl).float()
    q, k, v = qkv.float().reshape(B, 400, 3, 4, 128).permute(2, 0, 3, 1, 4)
    att = torch.softmax(q @ k.transpose(-1, -2) / 128 ** 0.5, dim=-1)
    ref = (att @ v).permute(0, 2, 1, 3).reshape(B * 400, 512)
    err = (out - ref).abs().max().item()
    assert err < 4e-3, f"attention impl {impl}: max err {err}"
