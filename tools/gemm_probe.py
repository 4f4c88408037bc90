"""Verbose on-GPU probe of the implicit-GEMM kernel: one case per process (so a hang in one case
cannot take the others down), prints an error map instead of a bare assert.

    python tools/gemm_probe.py <case>        # case in CASES
    python tools/gemm_probe.py all           # runs every case in a subprocess with a timeout
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = ["linear_small", "linear", "conv3_s1_128", "conv3_s1_256", "conv3_s1_512", "conv3_s2_64", "conv3_s2_256", "conv7", "perf"]


def report(name, got, ref):
    import torch

    got = got.float()
    err = (got - ref).abs()
    tol = 3e-3 + 2e-3 * ref.abs()
    bad = err > tol
    print(f"[{name}] shape {tuple(got.shape)} max_err {err.max().item():.4g} ref_absmax {ref.abs().max().item():.4g} "
          f"bad {bad.sum().item()}/{bad.numel()} got_absmax {got.abs().max().item():.4g} nan {torch.isnan(got).sum().item()}")
    if bad.any():
        b = bad.reshape(-1, bad.shape[-1])
        rows = b.any(1).nonzero().flatten()
        cols = b.any(0).nonzero().flatten()
        print(f"   bad rows: {rows.numel()} (first {rows[:16].tolist()}), bad cols: {cols.numel()} (first {cols[:16].tolist()})")
        g = got.reshape(-1, got.shape[-1])
        r = ref.reshape(-1, ref.shape[-1])
        i = rows[0].item()
        print("   got[row0,:8]", g[i, :8].tolist())
        print("   ref[row0,:8]", r[i, :8].tolist())
    return not bad.any().item()


def run_case(case):
    import torch
    import torch.nn.functional as F

    from foundationpose_b200 import _lib, ops, packing

    torch.manual_seed(0)
    dev = "cuda"
    ok = True
    if case in ("linear_small", "linear"):
        M, K, Co = (128, 64, 64) if case == "linear_small" else (1000, 512, 1536)
        x = torch.randn(M, K, device=dev).half()
        w = (torch.randn(Co, K, device=dev) * K ** -0.5)
        b = torch.randn(Co, device=dev)
        out = ops.gemm_layer(_lib.LAYER_LINEAR, x, packing.pack_linear(w.cpu()).cuda(), b, n_img=1, Hin=1, Win=M, Cin=K, Cout=Co)
        torch.cuda.synchronize()
        ok = report(case, out.reshape(M, Co), x.float() @ w.half().float().t() + b)
    elif case.startswith("conv3_s1"):
        C = int(case.split("_")[-1])
        H = 20 if C == 512 else 40
        n = 3
        x = torch.randn(n, C, H, H, device=dev).half()
        w = torch.randn(C, C, 3, 3, device=dev) * (9 * C) ** -0.5
        b = torch.randn(C, device=dev)
        res = torch.randn(n, H, H, C, device=dev).half()
        out = ops.gemm_layer(_lib.LAYER_CONV3_S1, x.permute(0, 2, 3, 1).contiguous(), packing.pack_conv3(w.cpu()).cuda(), b,
                             n_img=n, Hin=H, Win=H, Cin=C, Cout=C, res=res, res_ld=C, relu=True)
        torch.cuda.synchronize()
        ref = (F.conv2d(x.float(), w.half().float(), b, padding=1).permute(0, 2, 3, 1) + res.float()).relu()
        ok = report(case, out, ref)
    elif case.startswith("conv3_s2"):
        C = int(case.split("_")[-1])
        H = 80 if C == 64 else 40
        n = 3
        x = torch.randn(n, C, H, H, device=dev).half()
        w = torch.randn(2 * C, C, 3, 3, device=dev) * (9 * C) ** -0.5
        b = torch.randn(2 * C, device=dev)
        out = ops.gemm_layer(_lib.LAYER_CONV3_S2, x.permute(0, 2, 3, 1).contiguous(), packing.pack_conv3(w.cpu()).cuda(), b,
                             n_img=n, Hin=H, Win=H, Cin=C, Cout=2 * C, relu=True)
        torch.cuda.synchronize()
        ref = F.conv2d(x.float(), w.half().float(), b, stride=2, padding=1).relu().permute(0, 2, 3, 1)
        ok = report(case, out, ref)
    elif case == "conv7":
        n, H = 2, 160
        x = torch.randn(n, 6, H, H, device=dev).half()
        w = torch.randn(64, 6, 7, 7, device=dev) * (294) ** -0.5
        b = torch.randn(64, device=dev)
        out = ops.gemm_layer(_lib.LAYER_CONV7_S2, packing.pad_image_c8(x), packing.pack_conv7(w.cpu()).cuda(), b,
                             n_img=n, Hin=H, Win=H, Cin=8, Cout=64, relu=True)
        torch.cuda.synchronize()
        ref = F.conv2d(x.float(), w.half().float(), b, stride=2, padding=3).relu().permute(0, 2, 3, 1)
        ok = report(case, out, ref)
    elif case == "perf":
        # per-layer throughput at the C2 batch (252 hypotheses): CUDA events, 3 warm-up + 5 windows of 10 timed launches,
        # the median window reported.  The 128-channel convolutions run both tiles in alternating windows: the 128 x 128
        # tile (FPOSE_SWAP_TILE=0) and whatever the plan picks by default.
        name_dev = torch.cuda.get_device_name()
        try:
            power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                    str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            power = "unknown"
        print(f"[perf] {name_dev}, power limit {power}")
        shapes = [("conv7 6->64 @160 (504 img)", _lib.LAYER_CONV7_S2, 504, 160, 8, 64, 294),
                  ("conv3s2 64->128 @80 (504)", _lib.LAYER_CONV3_S2, 504, 80, 64, 128, 576),
                  ("conv3 128 @40 (504)", _lib.LAYER_CONV3_S1, 504, 40, 128, 128, 1152),
                  ("conv3 128 @40 (249+252) +res split", _lib.LAYER_CONV3_S1, 501, 40, 128, 128, 1152),
                  ("conv3 256 @40 (252)", _lib.LAYER_CONV3_S1, 252, 40, 256, 256, 2304),
                  ("conv3 256 @40 (249, odd M tiles)", _lib.LAYER_CONV3_S1, 249, 40, 256, 256, 2304),
                  ("conv3s2 256->512 @40 (252)", _lib.LAYER_CONV3_S2, 252, 40, 256, 512, 2304),
                  ("conv3 512 @20 (252)", _lib.LAYER_CONV3_S1, 252, 20, 512, 512, 4608),
                  ("linear 512->1536 (100800 rows)", _lib.LAYER_LINEAR, 1, 100800, 512, 1536, 512),
                  ("linear 512->3072 (100800 rows)", _lib.LAYER_LINEAR, 1, 100800, 512, 3072, 512),
                  ("conv3 128 @40 (504) +res", _lib.LAYER_CONV3_S1, 504, 40, 128, 128, 1152),
                  ("conv3 256 @40 (252) +res", _lib.LAYER_CONV3_S1, 252, 40, 256, 256, 2304),
                  ("conv3 512 @20 (252) +res", _lib.LAYER_CONV3_S1, 252, 20, 512, 512, 4608),
                  ("conv3 512 @20 (252) +res +pe", _lib.LAYER_CONV3_S1, 252, 20, 512, 512, 4608),
                  ("linear 512->512 (100800) +res", _lib.LAYER_LINEAR, 1, 100800, 512, 512, 512)]
        for name, kind, n, H, Ci, Co, Kreal in shapes:
            use_res = "+res" in name
            use_pe = "+pe" in name
            if kind == _lib.LAYER_LINEAR:
                x = torch.randn(H, Ci, device=dev).half()
                w = torch.randn(Co, Ci, device=dev).half()
                kw = dict(n_img=1, Hin=1, Win=H, Cin=Ci, Cout=Co)
                M = H
            elif kind == _lib.LAYER_CONV7_S2:
                x = torch.zeros(n, H + 6, H + 8, 8, device=dev, dtype=torch.float16)
                w = torch.randn(Co, 7 * 64, device=dev).half()
                kw = dict(n_img=n, Hin=H, Win=H, Cin=8, Cout=Co)
                M = n * (H // 2) ** 2
            else:
                x = torch.randn(n, H, H, Ci, device=dev).half()
                w = torch.randn(Co, 9 * Ci, device=dev).half()
                kw = dict(n_img=n, Hin=H, Win=H, Cin=Ci, Cout=Co)
                M = n * H * H if kind == _lib.LAYER_CONV3_S1 else n * (H // 2) ** 2
            b = torch.zeros(Co, device=dev)
            Ho = 1 if kind == _lib.LAYER_LINEAR else (H if kind == _lib.LAYER_CONV3_S1 else H // 2)
            out_ld = Co
            if "split" in name:  # the last encodeA layer: A images 0..248, B from 252, into the 256-channel concat
                kw.update(out_split=252)
                out_ld = 2 * Co
                out = torch.empty((n - 252) * Ho * Ho * out_ld, device=dev, dtype=torch.float16)
            else:
                out = torch.empty(M * Co, device=dev, dtype=torch.float16)
            if use_res:
                kw.update(res=torch.randn(M * Co, device=dev).half(), res_ld=Co)
            if use_pe:
                kw.update(post_add=torch.randn(Ho * Ho, Co, device=dev))
            q = dict(n_img=kw["n_img"], Hin=kw["Hin"], Win=kw["Win"], Cin=Ci, Cout=Co, out_split=kw.get("out_split", 0))
            variants = ["1"]
            if Co == 128 and kind in (_lib.LAYER_CONV3_S1, _lib.LAYER_CONV3_S2):
                variants = ["0", "1"]
            times = {v: [] for v in variants}
            tiles = {}
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for rep in range(5):
                for v in variants:
                    os.environ["FPOSE_SWAP_TILE"] = v
                    if rep == 0:
                        # tile configuration the layer runs with ("-" for a library that predates the query)
                        tile = "-"
                        if getattr(_lib.lib, "fp_op_gemm_tile_n", None) is not None:
                            tm = ops.gemm_tile_m(kind, **q) if getattr(_lib.lib, "fp_op_gemm_tile_m", None) else 128
                            tile = f"{tm}x{ops.gemm_tile_n(kind, **q)}"
                        tiles[v] = tile
                        for _ in range(3):
                            ops.gemm_layer(kind, x, w, b, out=out, out_ld=out_ld, relu=True, **kw)
                    e0.record()
                    for _ in range(10):
                        ops.gemm_layer(kind, x, w, b, out=out, out_ld=out_ld, relu=True, **kw)
                    e1.record()
                    torch.cuda.synchronize()
                    times[v].append(e0.elapsed_time(e1) / 10)
            os.environ.pop("FPOSE_SWAP_TILE", None)
            fl = 2.0 * M * Co * Kreal
            for v in variants:
                ms = sorted(times[v])[len(times[v]) // 2]
                rates = " ".join(f"{fl / t / 1e9:.0f}" for t in times[v])
                print(f"[perf] {name:34s} tile {tiles[v]:7s} {ms:8.3f} ms  {fl / ms / 1e9:8.1f} TFLOP/s (algorithmic, "
                      f"median of 5; windows {rates})")
    print(f"[{case}] {'OK' if ok else 'FAIL'}")
    return ok


if __name__ == "__main__":
    case = sys.argv[1] if len(sys.argv) > 1 else "all"
    if case == "all":
        rc = 0
        for c in CASES:
            try:
                p = subprocess.run([sys.executable, os.path.abspath(__file__), c], timeout=180, capture_output=True, text=True)
                print(p.stdout[-3000:])
                if p.returncode != 0:
                    print(f"[{c}] exit {p.returncode}\n{p.stderr[-3000:]}")
                    rc = 1
            except subprocess.TimeoutExpired as e:
                print(f"[{c}] TIMEOUT (hang?)\n{(e.stdout or b'')[-2000:]}")
                rc = 1
        sys.exit(rc)
    sys.exit(0 if run_case(case) else 1)
