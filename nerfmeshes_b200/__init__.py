"""nerfmeshes_b200 — H100-native (sm_90a) NeRF render / dense-grid hot path of qway/nerfmeshes (the name is historical).

Layout: csrc/ (CUDA kernels + C ABI, built into lib/libnerfmeshes_b200.so), _lib.py (ctypes binding), engine.py (handle +
torch plumbing), models.py / nerf_api.py / mesh.py / train.py / eval.py (host mirror of the reference's interface for this path).
"""
from . import _lib
from ._lib import NmError, PREC_EXACT, PREC_FAST, PREC_FP32
from .cfgnode import CfgNode, flatten_dict, nest_dict
from .engine import Engine, RenderSettings
from .models import (BaseModel, BuFFModel, FlexibleNeRFModel, NeRFModel, OutputBundle, TreeSampling,
                     load_lightning_checkpoint)
from .nerf_api import get_ray_bundle, meshgrid_xy, ndc_rays, pose_spherical
from .mesh import (extract_geometry, extract_geometry_with_super_sampling, extract_iso_level, extract_radiance, load_obj,
                   marching_cubes, super_sampling_tables)
from .chamfer import Meshes, chamfer_distance, create_mesh, sample_points_from_meshes
from .train import training_step

__all__ = [n for n in dir() if not n.startswith("_")]
