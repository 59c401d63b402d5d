"""The body of NeRFModel.training_step (src/models/model_nerf.py:88-151) on the fused path: manual batching over
`cfg.nerf.train.chunksize` rays, loss = mse(coarse.rgb_map, target) + mse(fine.rgb_map, target) averaged over the chunks,
PSNR log values — with forward, loss and backward of a chunk in ONE library call (nm_loss_backward), so the forward runs
once per chunk (the autograd route of `NeRFModel.forward` re-runs it inside backward).  Gradients land in `.grad` of
the CUDA parameters; the optimiser / scheduler stay the caller's (model_base.py:150-177)."""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import parallel


def mse2psnr(mse: float) -> float:
    """src/nerf/nerf_helpers.py: -10 log10(mse) (1e-5 substituted for an exact 0)."""
    return -10.0 * math.log10(mse if mse != 0 else 1e-5)


def training_step(model, ray_batch, ray_targets, *, chunksize: Optional[int] = None, seed: Optional[int] = None,
                  group=None, allreduce: bool = True, global_step: Optional[int] = None):
    """ray_batch = (ray_origins (3,) | (R,3), ray_directions (R,3), (near, far)); ray_targets (R,3).  All CUDA tensors.
    Returns the reference's dict {"loss", "log": {...}} with python floats; parameters' .grad hold d loss / d theta
    (averaged over ranks when torch.distributed is initialised).
    NeRFModel: manual batching over `chunksize`, {"train/loss", "train/coarse_loss", "train/coarse_psnr", "train/fine_*"}
    (model_nerf.py:88-151).  BuFFModel: one batch, {"train/loss", "train/psnr"}, the sample weights are integrated into the
    voxel tree and the tree is consolidated when its schedule ticks (model_buff.py:75-110)."""
    if not model.training:
        raise RuntimeError("training_step needs model.train()")
    if global_step is not None:
        model.global_step = int(global_step)
    # empty-space skipping (BaseModel.enable_training_skip): the schedule ticks once per step, here, before any render
    ts = model._train_skip
    tskip = model._train_skip_tick(None if global_step is None else int(global_step))
    if ts is not None:
        ts["in_step"] = True
    try:
        return _step(model, ray_batch, ray_targets, chunksize, seed, group, allreduce, tskip)
    finally:
        if ts is not None:
            ts["in_step"] = False


def _step(model, ray_batch, ray_targets, chunksize, seed, group, allreduce, tskip):
    named = model._named_net_params()
    if type(model).__name__ == "BuFFModel":
        # through forward(): it owns the tree-integration hook (model_buff.py:65-66); gradients via the autograd bridge
        for _, _, p in named:
            p.grad = None
        out = model.forward(ray_batch, seed=seed)
        loss = torch.nn.functional.mse_loss(out.rgb_map, ray_targets.to(out.rgb_map.device))
        loss.backward()
        if allreduce:
            parallel.allreduce_gradients([p for _, _, p in named], group)
        if model.tree.ticked(model.global_step):
            model.tree.consolidate()
        value = float(loss)
        return {"loss": value, "log": {"train/loss": value, "train/psnr": mse2psnr(value)}}
    ray_origins, ray_directions, near, far = model._unpack(ray_batch)
    eng = model._engine()
    R = ray_directions.shape[0]
    chunk = int(chunksize or model.cfg.nerf.train.get("chunksize", R) or R)
    n_chunks = R / chunk                                         # the reference divides by this float (model_nerf.py:93)
    per_ray_o = torch.as_tensor(ray_origins).numel() != 3
    eng.zero_grad()
    loss = torch.zeros(2, dtype=torch.float32, device=ray_directions.device)
    base_seed = model._pick_seed(seed)
    for i in range(0, R, chunk):
        sl = slice(i, i + chunk)
        o = ray_origins[sl] if per_ray_o else ray_origins
        loss += eng.loss_backward(o, ray_directions[sl], near, far, ray_targets[sl], training=True, seed=base_seed + i,
                                  train_skip=tskip)
    for which, name, p in named:
        g = eng.get_grad(which, name, p)
        p.grad = g.div_(n_chunks) if p.grad is None else p.grad.add_(g.div_(n_chunks))
    if allreduce:
        parallel.allreduce_gradients([p for _, _, p in named], group)
    terms = (loss / n_chunks).tolist()
    two = len(model._nets()) > 1 and model._nets()[1] is not None
    log = {"train/coarse_loss": terms[0], "train/coarse_psnr": mse2psnr(terms[0])}
    total = terms[0]
    if two:
        log.update({"train/fine_loss": terms[1], "train/fine_psnr": mse2psnr(terms[1])})
        total += terms[1]
    log["train/loss"] = total
    return {"loss": total, "log": log}
