"""Chamfer-distance mesh evaluation — the pieces of pytorch3d that the chamfer branch of validation_epoch_end
(src/models/model_base.py:82-102) calls, plus create_mesh (src/mesh_nerf.py:14-24).  The sampling and the nearest-neighbour
search run in the library (nm_mesh_sample, nm_chamfer; DESIGN 4.7).  The definitions are recalled from pytorch3d ~v0.2 and
not verified against it (it is not installable here); parity is distributional, like `perturb`."""
from __future__ import annotations

from typing import List, Optional

import torch


class Meshes:
    """pytorch3d.structures.Meshes reduced to what the chamfer branch reads: lists of (V,3) vertices and (F,3) faces."""

    def __init__(self, verts: List[torch.Tensor], faces: List[torch.Tensor]):
        if len(verts) != len(faces):
            raise ValueError("verts and faces lists must have the same length")
        self._verts = [torch.as_tensor(v) for v in verts]
        self._faces = [torch.as_tensor(f) for f in faces]

    def verts_list(self):
        return self._verts

    def faces_list(self):
        return self._faces

    def isempty(self) -> bool:
        return len(self._verts) == 0 or all(v.shape[0] == 0 or f.shape[0] == 0 for v, f in zip(self._verts, self._faces))

    def __len__(self):
        return len(self._verts)


def create_mesh(vertices, faces_idx) -> Meshes:
    """src/mesh_nerf.py:14-24: centre the vertices on their mean and scale by the largest absolute coordinate (float32, on
    the host)."""
    v = torch.as_tensor(vertices).detach().cpu().to(torch.float32)
    v = v - v.mean(0)
    scale = max(v.abs().max(0)[0])
    v = v / scale
    return Meshes(verts=[v], faces=[torch.as_tensor(faces_idx).detach().cpu()])


def _engine(engine):
    if engine is not None:
        return engine
    from .nerf_api import _engine as util
    return util()


def sample_points_from_meshes(meshes: Meshes, num_samples: int = 10000, seed: Optional[int] = None, engine=None):
    """pytorch3d.ops.sample_points_from_meshes(meshes, num_samples) without normals / textures: (B, num_samples, 3)
    area-weighted surface points on the device.  Mesh b uses seed + b; with no seed one is drawn from torch's default
    generator, so torch.manual_seed makes runs reproducible."""
    if meshes.isempty():
        raise ValueError("Meshes are empty.")
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    eng = _engine(engine)
    return torch.stack([eng.mesh_sample(v, f, int(num_samples), int(seed) + b)
                        for b, (v, f) in enumerate(zip(meshes.verts_list(), meshes.faces_list()))])


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                     batch_reduction: str = "mean", point_reduction: str = "mean", engine=None):
    """pytorch3d.loss.chamfer_distance(x, y) for (B,N,3) / (B,M,3) point tensors with point and batch reduction "mean":
    mean over the batch of mean_i d2(x_i, Y) + mean_j d2(y_j, X), d2 the squared distance to the nearest point.  Returns
    (loss, None) like pytorch3d; the loss is a float64 0-dim device tensor.  Padded batches, weights and normals raise."""
    if x_lengths is not None or y_lengths is not None or weights is not None or x_normals is not None or y_normals is not None:
        raise NotImplementedError("chamfer_distance: lengths, weights and normals are not supported")
    if batch_reduction != "mean" or point_reduction != "mean":
        raise NotImplementedError("chamfer_distance: only batch_reduction = point_reduction = 'mean'")
    x, y = torch.as_tensor(x), torch.as_tensor(y)
    if x.dim() != 3 or y.dim() != 3 or x.shape[0] != y.shape[0] or x.shape[2] != 3 or y.shape[2] != 3:
        raise ValueError(f"chamfer_distance: expected (B,N,3) and (B,M,3), got {tuple(x.shape)} and {tuple(y.shape)}")
    eng = _engine(engine)
    loss = sum(eng.chamfer(x[b], y[b]).sum() for b in range(x.shape[0])) / x.shape[0]
    return loss, None
