"""pytorch3d.loss.chamfer_distance (src/models/model_base.py:99) backed by nerfmeshes_b200.chamfer (nm_chamfer)."""
from nerfmeshes_b200.chamfer import chamfer_distance

__all__ = ["chamfer_distance"]
