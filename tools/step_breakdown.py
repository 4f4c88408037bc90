"""Where the time of one `register` step goes, per kernel kind: one steady-state `Engine.refine(poses, 5)` +
`Engine.score` at 252 hypotheses, run eagerly (no CUDA graphs, so every launch is its own trace record) under
`torch.profiler` with CUDA activities.

    python tools/step_breakdown.py [--hyp 252] [--iters 5] [--out DIR]

Kernels are named by what they run.  The implicit-GEMM launches (`gemm_tile_kernel`, `linear_ws_kernel`) are told apart
by their place in a pass, which is fixed: after the stem come the encoder's convolutions, the last GEMM ahead of the
attention kernel is the in-projection, and in a refiner pass the six GEMMs behind it are each head's out-projection,
FF1 and FF2.  The step itself is timed in a separate, unprofiled loop with CUDA events, eagerly and through the graphs
the product replays.  `--out` writes the table as JSON into DIR."""
import argparse
import json
import os
import subprocess
import sys

os.environ["FPOSE_NO_GRAPH"] = "1"  # read when the context is created: every launch stays a separate trace record

import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from foundationpose_b200 import hypotheses, synth  # noqa: E402
from foundationpose_b200.engine import Engine  # noqa: E402
from foundationpose_b200.estimater import make_mesh_tensors  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402

GEMM_KERNELS = ("gemm_tile_kernel", "linear_ws_kernel")
SIMPLE = [("crop_tile_kernel", "crop producer"), ("stem_conv_kernel", "stem 7x7/s2"), ("attn_tc_kernel", "attention"),
          ("layernorm_kernel", "LayerNorm"), ("token_reduce_kernel", "head final / token mean"),
          ("pose_update_kernel", "pose update"), ("rowwise_linear_kernel", "scorer tail"),
          ("cross_attn_score_kernel", "scorer tail")]
HEAD_LAYERS = ["out-proj 512->512 +res", "FF1 512->512 +ReLU", "FF2 512->512 +res"]


def device_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def label_kernels(kernels):
    """kernels: [(name, ms)] in launch order -> [(label, group, ms)]"""
    out = []
    gemms = []  # GEMM launches of the current pass not yet labelled: (index into out)
    state = {"attn_seen": False, "post": 0}

    def close_pass():
        # GEMMs behind the attention kernel exist only in a refiner pass
        for i in gemms:
            out[i] = ("scorer in-proj 512->1536", "linear", out[i][2])
        gemms.clear()

    for name, ms in kernels:
        if any(k in name for k in GEMM_KERNELS):
            if not state["attn_seen"]:
                gemms.append(len(out))
                out.append(("unlabelled GEMM", "conv", ms))
            else:
                if gemms:  # the pass has GEMMs after its attention: it is a refiner pass
                    for i in gemms:
                        out[i] = ("in-proj 512->3072 (both heads)", "linear", out[i][2])
                    gemms.clear()
                out.append((HEAD_LAYERS[state["post"] % 3], "linear", ms))
                state["post"] += 1
            continue
        simple = next((lab for key, lab in SIMPLE if key in name), None)
        if simple == "stem 7x7/s2" or simple == "crop producer":
            close_pass()
            state["attn_seen"] = False
            state["post"] = 0
        if simple == "attention" and not state["attn_seen"]:
            state["attn_seen"] = True
            # every GEMM before the in-projection is an encoder convolution, numbered after the stem (layer 0)
            for k, i in enumerate(gemms[:-1]):
                out[i] = (f"encoder conv layer {k + 1}", "conv", out[i][2])
            gemms[:] = gemms[-1:]
        if simple is None:
            out.append((name.split("(")[0][:60], "other", ms))
        else:
            out.append((simple, "attention" if simple == "attention" else "other", ms))
    close_pass()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hyp", type=int, default=252)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10, help="timed steps of the unprofiled loop")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "step_breakdown needs a CUDA device"

    mesh, gt, K, rgb, depth, mask = synth.default_scene(5, 0)
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt["uv"], tex=mt["tex"])
    e.set_frame(rgb, depth, K, filter_depth=True)
    d, _ = e.get_depth()
    poses = hypotheses.make_rotation_grid()[:a.hyp].copy()
    poses[:, :3, 3] = hypotheses.guess_translation(d.cpu().numpy(), mask, K)
    poses = torch.from_numpy(poses).cuda()

    def step():
        p, _, _ = e.refine(poses, a.iters)
        return e.score(p)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.reps):
        step()
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / a.reps

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    kern = [ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
    kern.sort(key=lambda ev: ev.time_range.start)
    kernels = [(ev.name, (ev.time_range.end - ev.time_range.start) / 1000.0) for ev in kern
               if "Memcpy" not in ev.name and "Memset" not in ev.name]
    rows = label_kernels(kernels)

    table = {}
    for label, group, ms in rows:
        t = table.setdefault(label, {"group": group, "ms": 0.0, "launches": 0})
        t["ms"] += ms
        t["launches"] += 1
    busy = sum(t["ms"] for t in table.values())
    groups = {}
    for t in table.values():
        groups[t["group"]] = groups.get(t["group"], 0.0) + t["ms"]

    name, power = device_info()
    print(f"device: {name}, power limit {power}")
    print(f"step ({a.hyp} hypotheses x {a.iters} iterations + score), eager: {step_ms:.2f} ms over {a.reps} steps; "
          f"kernel time in the traced step {busy:.2f} ms")
    print(f"{'kernel':42s} {'launches':>8s} {'ms':>9s} {'share':>7s}")
    for label, t in sorted(table.items(), key=lambda kv: -kv[1]["ms"]):
        print(f"{label:42s} {t['launches']:8d} {t['ms']:9.3f} {100 * t['ms'] / busy:6.1f}%")
    print("by group:")
    for g, ms in sorted(groups.items(), key=lambda kv: -kv[1]):
        print(f"  {g:40s} {ms:9.3f} ms {100 * ms / busy:6.1f}%")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "step_breakdown.json"), "w") as fh:
            json.dump({"device": name, "power_limit": power, "hyp": a.hyp, "iters": a.iters, "step_ms_eager": step_ms,
                       "kernel_ms": busy, "kernels": table, "groups": groups}, fh, indent=1)


if __name__ == "__main__":
    main()
