"""Golden vectors of the debug canvases, produced by the reference's own, unmodified code:

  * the three helpers (Utils.py:293-300 make_grid_image, :456-479 depth_to_vis, :630-655 cv_draw_text) on fixed inputs;
  * the canvases of PoseRefinePredictor.predict(get_vis=True) (predict_pose_refine.py:241-293) and
    ScorePredictor.predict(get_vis=True) (predict_score.py:27-52, :219-224, vis_batch_data_scores) on the scene of
    tools/make_golden_flow.py: its 5 start poses, 2 refiner iterations, then the scorer on the refined poses.

The reference's Utils.py cannot be imported here (it pulls in nvdiffrast, pytorch3d, warp, ...), so the function bodies
are extracted with `ast` (tools/make_golden_geometry.py::extract) and run with numpy, cv2, torch and torchvision; the
predictors run in the harness of tools/make_golden_flow.py (its rasteriser and warp substitutions, on the CPU).

    python tools/make_golden_vis.py        # needs /root/reference; writes tests/golden/vis_golden.npz (~1 min)

tests/test_vis_cpu.py holds foundationpose_b200/vis.py (which the drop-in Utils re-exports) and the host composer
tests/vis_compose.py to these vectors; tests/test_vis_gpu.py holds the CUDA canvases to them.
"""
import os
import sys

import cv2
import numpy as np
import torch
import torchvision

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
REF = os.environ.get("FPOSE_REFERENCE", "/root/reference")


def reference_helpers():
    from make_golden_geometry import extract

    ns = dict(np=np, cv2=cv2, torch=torch, torchvision=torchvision)
    for name in ("make_grid_image", "depth_to_vis", "cv_draw_text"):
        exec(extract(os.path.join(REF, "Utils.py"), name), ns)
    return ns["make_grid_image"], ns["depth_to_vis"], ns["cv_draw_text"]


def cases():
    """Fixed inputs: name -> kwargs.  Shared with the test, which rebuilds them from the same seed."""
    rng = np.random.default_rng(7)
    depth = rng.uniform(0.3, 0.9, (48, 40)).astype(np.float32)
    depth[:5] = 0.0
    depth[10, :] = 0.3
    norm = rng.uniform(-0.6, 0.6, (48, 40)).astype(np.float32)
    norm[20:30, 5:15] = 0.0
    rgb_f = (rng.uniform(0, 1, (3, 32, 24, 3)).astype(np.float32) * np.float32(255))
    rgb_u = rng.integers(0, 256, (3, 32, 24, 3), dtype=np.uint8)
    return dict(depth=depth, norm=norm, rgb_f=rgb_f, rgb_u=rgb_u)


def reference_canvases(make_grid_image, depth_to_vis, cv_draw_text):
    """predict(get_vis=True) of both reference predictors, as register (estimater.py:203-221) calls them."""
    import make_golden_flow as mgf
    from make_golden_geometry import extract

    from foundationpose_b200.weights import DEFAULT_CFG, random_state_dict
    from oracle import geometry

    torch.set_num_threads(os.cpu_count())
    mesh, mt, _, rgb, depth, mask, K, d, _ = mgf.scene()
    cfg = mgf.Cfg(DEFAULT_CFG, input_resize=(160, 160))
    _, refiner, scorer = mgf.reference_objects(random_state_dict("refine", 0), random_state_dict("score", 0), cfg)
    helpers = dict(make_grid_image=make_grid_image, depth_to_vis=depth_to_vis, cv_draw_text=cv_draw_text, cv2=cv2)
    refiner.predict.__globals__.update(helpers)
    scorer.predict.__globals__.update(helpers)
    exec(extract(os.path.join(REF, "learning/training/predict_score.py"), "vis_batch_data_scores"), scorer.predict.__globals__)
    depth_f = geometry.bilateral_filter_depth(geometry.erode_depth(depth))
    poses = mgf.start_grid().copy()
    poses[:, :3, 3] = geometry.guess_translation(depth_f, mask, K)
    xyz_map = geometry.depth2xyzmap(depth_f, K)
    with torch.inference_mode():
        refined, vis_r = refiner.predict(mesh=mesh, mesh_tensors=mt, rgb=rgb, depth=depth_f, K=K, ob_in_cams=poses, normal_map=None,
                                         xyz_map=xyz_map, glctx=None, mesh_diameter=d, iteration=mgf.REGISTER_ITERS, get_vis=True)
        scores, vis_s = scorer.predict(mesh=mesh, rgb=rgb, depth=depth_f, K=K, ob_in_cams=refined.numpy(), normal_map=None,
                                       mesh_tensors=mt, glctx=None, mesh_diameter=d, get_vis=True)
    print(f"reference canvases: refiner {vis_r.shape}, scorer {vis_s.shape}, scores {scores.numpy()}")
    return dict(canvas_start=poses, canvas_refined=refined.numpy(), canvas_scores=scores.numpy(), canvas_refine=vis_r,
                canvas_score=vis_s)


def main():
    make_grid_image, depth_to_vis, cv_draw_text = reference_helpers()
    c = cases()
    out = dict(c)
    out["d2v_inverse"] = depth_to_vis(c["depth"])
    out["d2v_range"] = depth_to_vis(c["depth"], zmin=np.float32(0.3), zmax=np.float32(0.7), inverse=False)
    out["d2v_norm"] = depth_to_vis(c["norm"], zmin=c["norm"].min(), zmax=c["norm"].max(), inverse=False)
    out["d2v_flat"] = depth_to_vis(np.zeros((8, 8), np.float32), zmin=np.float32(0), zmax=np.float32(0), inverse=False)
    out["d2v_gray"] = depth_to_vis(c["depth"], mode="gray")
    mixed = [c["rgb_f"][0], c["rgb_f"][1], c["rgb_u"][0], c["rgb_u"][1]]
    out["grid_mixed"] = make_grid_image(mixed, nrow=4, padding=2, pad_value=255)
    out["grid_rows"] = make_grid_image(list(c["rgb_u"]), nrow=2, padding=5, pad_value=255)
    out["grid_one"] = make_grid_image([c["rgb_f"][2]], nrow=1, padding=2, pad_value=255)
    out["grid_col"] = make_grid_image(list(c["rgb_f"]), nrow=1, padding=2, pad_value=0)
    base = c["rgb_u"][0].repeat(4, axis=0).repeat(8, axis=1)  # 128 x 192
    out["text_u8"] = cv_draw_text(base.copy(), text="id:7", uv_top_left=(10, 10), color=(0, 255, 0), fontScale=0.5)
    out["text_edge"] = cv_draw_text(base.copy(), text="id:123, score:101.234\nline two", uv_top_left=(150, 120),
                                    color=(255, 0, 0), fontScale=0.5, outline_color=(0, 0, 0))
    out["text_f64"] = cv_draw_text(base.astype(np.float64), text="id:3, score:100.500", uv_top_left=(10, 10),
                                   color=(0, 255, 0), fontScale=0.5)
    out.update(reference_canvases(make_grid_image, depth_to_vis, cv_draw_text))
    path = os.path.join(ROOT, "tests", "golden", "vis_golden.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
