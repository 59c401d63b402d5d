"""pytorch3d.structures.Meshes, reduced to verts_list / faces_list / isempty (what mesh_nerf.create_mesh and the chamfer
branch of validation_epoch_end use): nerfmeshes_b200.chamfer.Meshes."""
from nerfmeshes_b200.chamfer import Meshes

__all__ = ["Meshes"]
