"""Where does the scorer-feature error come from?  For a subset of the golden final poses (tests/golden/register_252x5.npz):
  crops: CUDA producer vs oracle (pixel statistics per channel group),
  features: CUDA net on CUDA crops | CUDA net on ORACLE crops | oracle net on oracle crops (= golden)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from foundationpose_b200 import synth  # noqa: E402
from foundationpose_b200.engine import Engine, crops_from_planar  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402
from oracle import geometry, nets, pipeline  # noqa: E402


def main():
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "register_252x5.npz")))
    mesh = synth.make_mesh(3)
    rgb, depth, mask = synth.make_scene(mesh.visual.image, g["gt_pose"])
    d = synth.mesh_diameter(mesh.vertices)
    mt = pipeline.mesh_tensors(mesh)
    sd_s = random_state_dict("score", 0)
    e = Engine()
    e.load_network("score", sd_s)
    e.load_network("refine", random_state_dict("refine", 0))
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt["uv"], tex=mt["tex"])
    e.set_frame(rgb, depth, synth.DEFAULT_K, filter_depth=True)
    depth_f = e.get_depth()[0].cpu().numpy()
    ref_depth_f = geometry.bilateral_filter_depth(geometry.erode_depth(depth))
    print("filtered depth max diff", np.abs(depth_f - ref_depth_f).max())
    idx = np.arange(0, 252, 16)
    poses = g["poses"][5][idx]
    for mode in (1, 0):
        _, dbg, _ = e.make_crops(poses, mode=mode, want_dbg=True)
        xyz = geometry.depth2xyzmap(ref_depth_f, synth.DEFAULT_K)
        A, B, _ = pipeline.make_crops(poses, mt, rgb, ref_depth_f, xyz, synth.DEFAULT_K, d, mode)
        gA = dbg[:, 0].permute(0, 3, 1, 2).cpu()
        gB = dbg[:, 1].permute(0, 3, 1, 2).cpu()
        for name, x, y in (("A rgb", gA[:, :3], A[:, :3]), ("A xyz", gA[:, 3:], A[:, 3:]), ("B rgb", gB[:, :3], B[:, :3]), ("B xyz", gB[:, 3:], B[:, 3:])):
            dd = (x - y).abs()
            print(f"mode {mode} {name}: max {dd.max():.3e} mean {dd.mean():.3e}  pixels > 1e-3: {(dd.amax(1) > 1e-3).sum().item()} of {dd.shape[0] * 160 * 160}"
                  f"  > 1e-2: {(dd.amax(1) > 1e-2).sum().item()}")
        if mode == 1:
            f_gpu = e.score_features(poses).cpu()
            f_gpu_oraclecrops = e.op_score_feats(crops_from_planar(A.cuda(), B.cuda()), len(poses)).cpu()
            f_gpu_gpucrops_planar = e.op_score_feats(crops_from_planar(gA.cuda(), gB.cuda()), len(poses)).cpu()
            f_ref = nets.score_features(sd_s, A, B)
            gold = torch.from_numpy(g["feats"][idx])
            rms = lambda t: float(t.pow(2).mean().sqrt())
            print("golden vs recomputed oracle feats", rms(f_ref - gold))
            print("CUDA net + CUDA crops (product path) vs golden: rms", rms(f_gpu - gold), "max", float((f_gpu - gold).abs().max()))
            print("CUDA net + ORACLE crops vs golden: rms", rms(f_gpu_oraclecrops - gold), "max", float((f_gpu_oraclecrops - gold).abs().max()))
            print("CUDA net + CUDA crops re-imported (fp32 dbg) vs product path: rms", rms(f_gpu_gpucrops_planar - f_gpu))
            f_ref_gpucrops = nets.score_features(sd_s, gA, gB)
            print("ORACLE net + CUDA crops vs golden: rms", rms(f_ref_gpucrops - gold), "max", float((f_ref_gpucrops - gold).abs().max()))
            print("feature spread across these hypotheses (std per dim, mean)", float(gold.std(0).mean()))


def outliers():
    """Per-hypothesis feature error over all 252 golden poses; stage-wise comparison for the worst ones."""
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "register_252x5.npz")))
    mesh = synth.make_mesh(3)
    rgb, depth, mask = synth.make_scene(mesh.visual.image, g["gt_pose"])
    d = synth.mesh_diameter(mesh.vertices)
    mt = pipeline.mesh_tensors(mesh)
    sd_s = random_state_dict("score", 0)
    e = Engine()
    e.load_network("score", sd_s)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt["uv"], tex=mt["tex"])
    e.set_frame(rgb, depth, synth.DEFAULT_K, filter_depth=True)
    poses = g["poses"][5]
    f = e.score_features(poses).cpu().numpy()
    err = np.abs(f - g["feats"])
    per = err.max(1)
    order = np.argsort(-per)
    print("per-hypothesis max feature error: median %.2e, 90%% %.2e, worst %s" % (np.median(per), np.quantile(per, 0.9), [(int(i), float(per[i])) for i in order[:8]]))
    # batch-size dependence: the same poses scored alone / in a small batch
    for n in (1, 8, 64):
        idx = order[:n] if n > 1 else order[:1]
        fs = e.score_features(poses[idx]).cpu().numpy()
        print(f"  worst {n} scored as a batch of {n}: max err {np.abs(fs - g['feats'][idx]).max():.2e} (in the 252 batch: {err[idx].max():.2e})")
    worst = order[:4]
    ref_depth_f = geometry.bilateral_filter_depth(geometry.erode_depth(depth))
    A, B, _ = pipeline.make_crops(poses[worst], mt, rgb, ref_depth_f, None, synth.DEFAULT_K, d, 1)
    cb = crops_from_planar(A.cuda(), B.cuda())
    tok = e.op_encoder("score", cb, len(worst)).reshape(len(worst), 400, 512).float().cpu()
    x = nets.encode_a(torch.cat([A, B], 0), sd_s, "encoderA")
    ab = nets.encode_ab(torch.cat((x[:len(worst)], x[len(worst):]), 1), sd_s, "encoderAB")
    ref_tok = nets._tokens(ab, sd_s)
    te = (tok - ref_tok).abs()
    print("tokens of the worst 4: max err", te.amax(dim=(1, 2)).tolist(), "ref absmax", ref_tok.abs().amax(dim=(1, 2)).tolist())
    f4 = e.op_score_feats(cb, len(worst)).cpu()
    print("feats of the worst 4 through op_score_feats (batch 4, oracle crops): max err", (f4 - torch.from_numpy(g["feats"][worst])).abs().amax(1).tolist())
    # attention on the ORACLE tokens (fp16) vs oracle attention
    qkv = (ref_tok.half().float() @ sd_s["att.in_proj_weight"].half().float().t() + sd_s["att.in_proj_bias"])
    from foundationpose_b200 import ops

    o = ops.attention(qkv.reshape(-1, 1536).half().cuda()).float().cpu().reshape(len(worst), 400, 512)
    q, k, v = qkv.reshape(len(worst), 400, 3, 4, 128).permute(2, 0, 3, 1, 4)
    att = torch.softmax(q @ k.transpose(-1, -2) / 128 ** 0.5, dim=-1)
    ref_o = (att @ v).permute(0, 2, 1, 3).reshape(len(worst), 400, 512)
    print("attention core on oracle tokens: max err", (o - ref_o).abs().amax(dim=(1, 2)).tolist(), "absmax", ref_o.abs().amax(dim=(1, 2)).tolist(),
          "max logit", (q @ k.transpose(-1, -2) / 128 ** 0.5).abs().amax(dim=(1, 2, 3)).tolist())


def worst_crops():
    """Pixel comparison of the CUDA and oracle scorer crops for the hypotheses with the largest feature error."""
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "register_252x5.npz")))
    mesh = synth.make_mesh(3)
    rgb, depth, mask = synth.make_scene(mesh.visual.image, g["gt_pose"])
    d = synth.mesh_diameter(mesh.vertices)
    mt = pipeline.mesh_tensors(mesh)
    e = Engine()
    e.load_network("score", random_state_dict("score", 0))
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt["uv"], tex=mt["tex"])
    e.set_frame(rgb, depth, synth.DEFAULT_K, filter_depth=True)
    poses = g["poses"][5]
    f = e.score_features(poses).cpu().numpy()
    per = np.abs(f - g["feats"]).max(1)
    worst = np.argsort(-per)[:3]
    print("worst", worst, per[worst], "poses t", poses[worst][:, :3, 3])
    ref_depth_f = geometry.bilateral_filter_depth(geometry.erode_depth(depth))
    for mode in (1, 0):
        _, dbg, win = e.make_crops(poses[worst], mode=mode, want_dbg=True)
        xyz = geometry.depth2xyzmap(ref_depth_f, synth.DEFAULT_K)
        A, B, owin = pipeline.make_crops(poses[worst], mt, rgb, ref_depth_f, xyz, synth.DEFAULT_K, d, mode)
        print("windows gpu", win.cpu().numpy().tolist(), "oracle", [owin[k].tolist() for k in ("left", "top", "sx", "sy")])
        gA = dbg[:, 0].permute(0, 3, 1, 2).cpu()
        gB = dbg[:, 1].permute(0, 3, 1, 2).cpu()
        for name, x, y in (("A rgb", gA[:, :3], A[:, :3]), ("A xyz", gA[:, 3:], A[:, 3:]), ("B rgb", gB[:, :3], B[:, :3]), ("B xyz", gB[:, 3:], B[:, 3:])):
            dd = (x - y).abs().amax(1)  # (n,160,160)
            for i in range(len(worst)):
                bad = (dd[i] > 1e-3).nonzero()
                msg = ""
                if len(bad):
                    r0, r1, c0, c1 = bad[:, 0].min().item(), bad[:, 0].max().item(), bad[:, 1].min().item(), bad[:, 1].max().item()
                    msg = f" rows {r0}-{r1} cols {c0}-{c1}; gpu-zero there: {(x[i].abs().sum(0)[bad[:, 0], bad[:, 1]] == 0).float().mean():.2f}, oracle-zero: {(y[i].abs().sum(0)[bad[:, 0], bad[:, 1]] == 0).float().mean():.2f}"
                print(f"mode {mode} hyp {worst[i]} {name}: max {dd[i].max():.3e}, pixels > 1e-3: {len(bad)}{msg}")


if __name__ == "__main__":
    if os.environ.get("PROBE_WORST"):
        worst_crops()
    elif os.environ.get("PROBE_OUTLIERS"):
        outliers()
    else:
        main()
