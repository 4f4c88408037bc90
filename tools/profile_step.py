"""One hot-path step (register: 252 hyp x 5 iters + score) bracketed by cudaProfilerStart/Stop, for

    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv \
        --log-file launches.csv python tools/profile_step.py
    ncu --profile-from-start off --set full --clock-control none --import-source on \
        -k regex:gemm_tile_kernel -s 6 -c 1 -o prof_gemm python tools/profile_step.py

Numbers printed under ncu are never bench values (replay serialises and cold-caches every launch)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from foundationpose_b200 import hypotheses, synth  # noqa: E402
from foundationpose_b200.engine import Engine  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402


def main():
    n_hyp = int(os.environ.get("FP_PROFILE_HYP", "252"))
    iters = int(os.environ.get("FP_PROFILE_ITERS", "5"))
    mesh, gt, K, rgb, depth, mask = synth.default_scene(5, 0)
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    from foundationpose_b200.estimater import make_mesh_tensors

    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt["uv"], tex=mt["tex"])
    e.set_frame(rgb, depth, K, filter_depth=True)
    d, _ = e.get_depth()
    poses = hypotheses.make_rotation_grid()[:n_hyp].copy()
    poses[:, :3, 3] = hypotheses.guess_translation(d.cpu().numpy(), mask, K)
    poses = torch.from_numpy(poses).cuda()
    for _ in range(2):
        p, _, _ = e.refine(poses, iters)
        e.score(p)
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    p, _, _ = e.refine(poses, iters)
    s, b = e.score(p)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    print("best", int(b.item()))


if __name__ == "__main__":
    main()
