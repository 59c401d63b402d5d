"""Worker of tests/test_gpu_surface_points.py's multi-GPU case — launched with torchrun, one process per GPU (NCCL).  The
pose-sharded surface point cloud must equal the single-block one, array for array and bit for bit, on every rank.  Prints
`SURFACE_MULTI_OK <world>` from rank 0."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from conftest import load_npz  # noqa: E402
from test_gpu_parity import LEGO_CFG  # noqa: E402


def main():
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    from nerfmeshes_b200 import parallel as par
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lego = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval().cuda()
    focal = float(0.5 * 64 / np.tan(0.5 * 0.6911112))
    poses = mesh.surface_ray_poses(5, 2)                # 10 views: uneven blocks on 3 or 4 ranks
    thr = 0.002 * (800 / 64) ** 2                       # the default scaled with the pixel footprint, as the GPU tests do
    for kw in (dict(min_acc=0.99, dist_threshold=thr), dict(network_normals=True, dist_threshold=thr)):
        one = par.surface_points_sharded(lego, poses, 64, 64, focal, 2.0, 6.0, group=par.SINGLE, **kw)
        many = par.surface_points_sharded(lego, poses, 64, 64, focal, 2.0, 6.0, **kw)
        assert one["counts"] == many["counts"], (kw, one["counts"], many["counts"])
        for k in ("points", "normals", "colors", "view", "pixel"):
            assert torch.equal(one[k], many[k]), (kw, k)
        assert one["points"].shape[0] > 0
    dist.barrier()
    if rank == 0:
        print(f"SURFACE_MULTI_OK {world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
