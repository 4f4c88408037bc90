"""On-GPU probe of the attention kernel: error vs torch fp32 + timing at B=252."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from foundationpose_b200 import ops


def ref_attn(qkv, B):
    q, k, v = qkv.float().reshape(B, 400, 3, 4, 128).permute(2, 0, 3, 1, 4)
    att = torch.softmax(q @ k.transpose(-1, -2) / 128 ** 0.5, dim=-1)
    return (att @ v).permute(0, 2, 1, 3).reshape(B * 400, 512)


def main():
    impls = [int(x) for x in sys.argv[1:]] or [0, 1]
    torch.manual_seed(0)
    B = 3
    qkv = (torch.randn(B * 400, 1536, device="cuda") * 1.5).half()
    ref = ref_attn(qkv, B)
    for impl in impls:
        out = ops.attention(qkv, impl=impl).float()
        torch.cuda.synchronize()
        err = (out - ref).abs()
        print(f"[attn impl {impl}] max_err {err.max().item():.4g} mean_err {err.mean().item():.4g} ref_absmax {ref.abs().max().item():.4g} nan {torch.isnan(out).sum().item()}")
        if err.max().item() > 4e-3:
            bad = (err > 4e-3)
            rows = bad.any(1).nonzero().flatten()
            cols = bad.any(0).nonzero().flatten()
            print("   bad rows", rows.numel(), rows[:12].tolist(), "bad cols", cols.numel(), cols[:12].tolist())
            print("   got", out[rows[0], :6].tolist())
            print("   ref", ref[rows[0], :6].tolist())
    B = 252
    qkv = (torch.randn(B * 400, 1536, device="cuda")).half()
    for impl in impls:
        for _ in range(3):
            ops.attention(qkv, impl=impl)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.attention(qkv, impl=impl)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        fl = 2 * 2.0 * B * 4 * 400 * 400 * 128
        print(f"[attn impl {impl}] B=252: {ms:.3f} ms  {fl / ms / 1e9:.1f} TFLOP/s")


if __name__ == "__main__":
    main()
