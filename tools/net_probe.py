"""On-GPU probe of the network paths: prints per-stage errors against the fp32 oracle and times the
refiner / scorer networks at the C2 batch (252 hypotheses)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from foundationpose_b200.engine import Engine, crops_from_planar  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402
from oracle import nets  # noqa: E402


def crops(n, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.rand(n, 6, 160, 160, generator=g)
    B = torch.rand(n, 6, 160, 160, generator=g)
    for T in (A, B):
        T[:, 3:] = (T[:, 3:] - 0.5) * 2
        T[:, 3:, :30] = 0
    return A, B


def main():
    e = Engine()
    sd_r = random_state_dict("refine", 0)
    sd_s = random_state_dict("score", 0)
    e.load_network("refine", sd_r)
    e.load_network("score", sd_s)
    n = 3
    A, B = crops(n, 11)
    cb = crops_from_planar(A.cuda(), B.cuda())
    A16, B16 = A.half().float(), B.half().float()

    tok = e.op_encoder("refine", cb, n).reshape(n, 400, 512).float().cpu()
    x = nets.encode_a(torch.cat([A16, B16], 0), sd_r, "encodeA")
    ab = nets.encode_ab(torch.cat((x[:n], x[n:]), 1), sd_r, "encodeAB")
    ref_tok = nets._tokens(ab, sd_r)
    err = (tok - ref_tok).abs()
    print(f"[tokens] max_err {err.max():.4g} mean_err {err.mean():.4g} ref_absmax {ref_tok.abs().max():.4g} nan {torch.isnan(tok).sum()}")

    trans, rot = e.op_refine_net(cb, n)
    ref = nets.refine_forward(sd_r, A16, B16)
    print("[refine] trans", trans.cpu().numpy().round(4).tolist())
    print("[refine]   ref", ref["trans"].numpy().round(4).tolist())
    print("[refine] rot  ", rot.cpu().numpy().round(4).tolist())
    print("[refine]   ref", ref["rot"].numpy().round(4).tolist())
    print(f"[refine] max_err trans {(trans.cpu() - ref['trans']).abs().max():.4g} rot {(rot.cpu() - ref['rot']).abs().max():.4g}")

    feats = e.op_score_feats(cb, n)
    ref_feats = nets.score_features(sd_s, A16, B16)
    print(f"[score feats] max_err {(feats.cpu() - ref_feats).abs().max():.4g} ref_absmax {ref_feats.abs().max():.4g}")
    scores, best = e.score_tail(ref_feats.cuda())
    ref_logits = nets.score_tail(sd_s, ref_feats, n).reshape(-1)
    print("[score tail] got", (scores.cpu() - 100).numpy().round(4).tolist(), "ref", ref_logits.numpy().round(4).tolist(), "best", int(best.item()), int(ref_logits.argmax()))

    # timing at N = 252
    N = 252
    big = torch.zeros(2 * N, 166, 168, 8, dtype=torch.float16, device="cuda")
    big[:, 3:163, 3:163, :6] = torch.rand(2 * N, 160, 160, 6, device="cuda").half()
    for name, fn in (("refine_net", lambda: e.op_refine_net(big, N)), ("score_feats", lambda: e.op_score_feats(big, N))):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        gf = 23.946 if name == "refine_net" else 21.94
        print(f"[perf] {name} N={N}: {ms:.3f} ms/pass -> {N / ms * 1e3:.0f} hyp-pass/s, {gf * N / ms / 1e3:.1f} TFLOP/s algorithmic")


if __name__ == "__main__":
    main()
