"""run_demo.py's flow (run_demo.py:38-63) with one tracking call always in flight: register on the first frame, then
submit frame i with `track_objects(..., wait=False)` and only then collect frame i - 1's pose and write it.  The host
reads and decodes frame i + 1 while the device tracks frame i, so a frame costs about the larger of the host time and
the device time instead of their sum.  The poses written are exactly those of run_demo.py's blocking track_one loop.

Reads a YCBInEOAT-layout scene (cam_K.txt, rgb/, depth/, masks/) through the drop-in YcbineoatReader and writes one
ob_in_cam/<frame id>.txt per frame, as run_demo.py does:

    python examples/track_sequence_pipelined.py --mesh_file SCENE/mesh/textured_simple.obj --test_scene_dir SCENE \\
        --out_dir /tmp/fpose_pipelined
"""
import argparse
import logging
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "foundationpose_b200", "dropin")):
    if p not in sys.path:
        sys.path.insert(0, p)

from datareader import YcbineoatReader  # noqa: E402
from Utils import trimesh  # noqa: E402

from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor, track_objects  # noqa: E402


def run(mesh_file, scene_dir, out_dir, est_refine_iter=5, track_refine_iter=2):
    mesh = trimesh.load(mesh_file)
    est = FoundationPose(model_pts=mesh.vertices, model_normals=mesh.vertex_normals, mesh=mesh, scorer=ScorePredictor(),
                         refiner=PoseRefinePredictor())
    reader = YcbineoatReader(video_dir=scene_dir, shorter_side=None, zfar=np.inf)
    os.makedirs(f"{out_dir}/ob_in_cam", exist_ok=True)

    def write(i, pose):
        np.savetxt(f"{out_dir}/ob_in_cam/{reader.id_strs[i]}.txt", pose.reshape(4, 4))

    pending = None  # (frame, PendingTrack) of the call in flight
    for i in range(len(reader.color_files)):
        color, depth = reader.get_color(i), reader.get_depth(i)
        if i == 0:
            mask = reader.get_mask(0).astype(bool)
            write(0, est.register(K=reader.K, rgb=color, depth=depth, ob_mask=mask, iteration=est_refine_iter))
            continue
        # est.pose_last already holds frame i - 1's pose on the device: frame i is submitted before i - 1 is collected
        submitted = (i, track_objects([est], color, depth, reader.K, iteration=track_refine_iter, wait=False))
        if pending is not None:
            write(pending[0], pending[1].result()[0])
        pending = submitted
    if pending is not None:
        write(pending[0], pending[1].result()[0])
    logging.info(f"{len(reader.color_files)} poses written to {out_dir}/ob_in_cam")


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--mesh_file", type=str, required=True)
    parser.add_argument("--test_scene_dir", type=str, required=True)
    parser.add_argument("--est_refine_iter", type=int, default=5)
    parser.add_argument("--track_refine_iter", type=int, default=2)
    parser.add_argument("--out_dir", type=str, default="/tmp/fpose_b200_pipelined")
    args = parser.parse_args()
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    run(args.mesh_file, args.test_scene_dir, args.out_dir, args.est_refine_iter, args.track_refine_iter)
