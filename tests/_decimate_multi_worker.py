"""Worker of tests/test_gpu_mesh_decimate.py's multi-GPU case — launched with torchrun, one process per GPU (NCCL).  Slab-sharded
extraction with decimation (every rank decimates the identical gathered mesh) must equal the single-shard extraction with the
switch, array for array, on every rank.  Prints `DECIMATE_MULTI_OK <world>` from rank 0."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from conftest import load_npz  # noqa: E402
from test_gpu_parity import LEGO_CFG  # noqa: E402


def main():
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import parallel as par
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lego = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval().cuda()
    for s, net in ((0, False), (2, True)):
        class Args:
            res, limit, iso_level, super_sampling, network_normals, min_component_faces, decimate_faces = 64, 1.2, 32.0, s, net, 40, 1500
        v1, f1, n1, _ = par.extract_geometry_sharded(lego, Args, group=par.SINGLE, to_host=False)
        v1, f1, n1 = v1.clone(), f1.clone(), n1.clone()
        vN, fN, nN, _ = par.extract_geometry_sharded(lego, Args, to_host=False)
        assert torch.equal(vN, v1) and torch.equal(fN, f1) and torch.equal(nN, n1), f"s={s}: decimated mesh differs"
    dist.barrier()
    if rank == 0:
        print(f"DECIMATE_MULTI_OK {world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
