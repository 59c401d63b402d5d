"""pytorch3d.ops.sample_points_from_meshes (src/models/model_base.py:94-96) backed by nerfmeshes_b200.chamfer (nm_mesh_sample)."""
from nerfmeshes_b200.chamfer import sample_points_from_meshes

__all__ = ["sample_points_from_meshes"]
