"""Worker of tests/test_gpu_sigma_grad.py's multi-GPU case — launched with torchrun, one process per GPU (NCCL).  Slab-sharded
extraction with network normals (every rank evaluates its own vertices before the gather) must equal the single-GPU
extraction with the switch, array for array, at s = 0 and s = 2.  Prints `SIGMA_GRAD_MULTI_OK <world>` from rank 0."""
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
    for s in (0, 2):
        class Args:
            res, limit, iso_level, super_sampling, network_normals = 40, 1.2, 32.0, s, True
        v1, f1, n1, _ = par.extract_geometry_sharded(lego, Args, group=par.SINGLE, to_host=False)
        vN, fN, nN, _ = par.extract_geometry_sharded(lego, Args, to_host=False)
        assert torch.equal(vN, v1) and torch.equal(fN, f1), f"s={s}: gathered mesh differs from the single-GPU one"
        assert torch.equal(nN, n1), f"s={s}: gathered network normals differ from the single-GPU ones"
    dist.barrier()
    if rank == 0:
        print(f"SIGMA_GRAD_MULTI_OK {world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
