"""CPU self-checks of the float64 references of tests/tail_reference.py, which tests/test_selection_gpu.py holds the
scorer tail and the pose update to."""
import numpy as np
import torch

import tail_reference as tr


def _sd64():
    from foundationpose_b200.weights import random_state_dict

    return tr.state_dict64(random_state_dict("score", 0), "cpu")


def test_tail_reference_matches_the_oracle_on_equal_segments():
    """Segments of equal length are the batch of oracle.nets.score_tail (score_network.py:84-88)."""
    from oracle import nets

    sd64 = _sd64()
    g = torch.Generator().manual_seed(1)
    for n, bs in ((1, 5), (20, 3), (63, 2)):
        x = (torch.randn(n * bs, 512, generator=g) * 2).double()
        ref = tr.tail_ref(sd64, x, list(range(0, n * bs + 1, n)))
        want = nets.score_tail(sd64, x, n).reshape(-1) + tr.OFFSET
        np.testing.assert_allclose(ref.numpy(), want.numpy(), atol=1e-12, rtol=0)


def test_tail_bar_holds_for_an_fp32_evaluation_and_rejects_the_probes():
    """The derived bar covers an fp32 evaluation of the same operation (torch on the CPU, another summation order than
    the kernel's), and it is tight enough that each wrong reference of the GPU test's probes fails it."""
    from foundationpose_b200.weights import random_state_dict

    sd = random_state_dict("score", 0)
    sd32 = {k: v.float() for k, v in tr.state_dict64(sd, "cpu").items()}
    sd64 = _sd64()
    g = torch.Generator().manual_seed(2)
    seg = [0, 63, 83, 84, 213]
    x32 = torch.randn(seg[-1], 512, generator=g) * 2
    x = x32.double()
    ref = tr.tail_ref(sd64, x, seg)
    bar = tr.tail_bar(sd64, x, seg)
    fp32 = tr.tail_ref(sd32, x32, seg).double()
    assert ((fp32 - ref).abs() / bar).max() < 1
    probes = {"neighbour key": tr.tail_ref(sd64, x, seg, extra_key=0)}
    sd_scale = dict(sd64)
    sd_scale["att_cross.in_proj_weight"] = sd64["att_cross.in_proj_weight"].clone()
    sd_scale["att_cross.in_proj_bias"] = sd64["att_cross.in_proj_bias"].clone()
    sd_scale["att_cross.in_proj_weight"][:512] *= 0.5  # q / 2: the logits of a 1 / sqrt(512) scale
    sd_scale["att_cross.in_proj_bias"][:512] *= 0.5
    probes["1/sqrt(512)"] = tr.tail_ref(sd_scale, x, seg)
    sd_nob = dict(sd64)
    sd_nob["att_cross.out_proj.bias"] = torch.zeros_like(sd64["att_cross.out_proj.bias"])
    probes["no out_proj bias"] = tr.tail_ref(sd_nob, x, seg)
    for name, p in probes.items():
        assert ((fp32 - p).abs() > bar).any(), name


def test_pose_update_bars_hold_for_an_fp32_evaluation():
    """oracle.geometry.pose_update (fp32 torch) stays inside the bars of the float64 restatement."""
    from oracle import geometry

    g = torch.Generator().manual_seed(3)
    N = 64
    poses = torch.eye(4).repeat(N, 1, 1)
    poses[:, :3, :3] = geometry.so3_exp_map(torch.randn(N, 3, generator=g))
    poses[:, :3, 3] = torch.randn(N, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 0.7])
    trans = torch.randn(N, 3, generator=g) * 0.3
    rot = torch.randn(N, 3, generator=g) * 2
    rot[:4] = 0
    rn, d = 0.3490658503988659, 0.8
    out, td, rd = geometry.pose_update(poses, trans, rot, d, rn)
    ref, td_ref, rd_ref = tr.pose_update_ref(poses, trans, rot, torch.full((N,), np.float32(d) / 2), np.float32(rn))
    bar_R, bar_td, bar_t = tr.pose_update_bars(poses, rd_ref, td_ref)
    assert ((rd.double() - rd_ref).abs() <= tr.ROT_DELTA_BAR).all()
    assert ((out[:, :3, :3].double() - ref[:, :3, :3]).abs() <= bar_R).all()
    assert ((td.double() - td_ref).abs() <= bar_td).all()
    assert ((out[:, :3, 3].double() - ref[:, :3, 3]).abs() <= bar_t).all()
