"""`nerf` namespace of the reference (src/nerf/__init__.py:1-5) for the hot path: compute entry points are the H100
implementation, the rest is the small host-side glue the scripts import by name."""
from nerfmeshes_b200.cfgnode import CfgNode  # noqa: F401
from nerfmeshes_b200.models import FlexibleNeRFModel, OutputBundle, PositionalEncoding, TreeSampling  # noqa: F401
from nerfmeshes_b200.nerf_api import get_ray_bundle, meshgrid_xy, ndc_rays  # noqa: F401
from . import models, nerf_helpers  # noqa: F401
from .nerf_helpers import *  # noqa: F401,F403
