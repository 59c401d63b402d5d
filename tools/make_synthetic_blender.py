#!/usr/bin/env python
"""Write a tiny Blender-format dataset (transforms_{train,val,test}.json + PNGs) and a config in the reference's live schema
(config/nerf-synthetic-lego.yml) so that train_nerf.py / eval_nerf.py can be driven without the real datasets (none ship
with the reference).  Images are rendered from the lego checkpoint re-packed under tests/golden/ when an H100 is available
(`--render`), else filled with noise (enough for the no-GPU plumbing test, which stops at the first compute call).

    python tools/make_synthetic_blender.py OUT_DIR [--size 40] [--views 6 2 2] [--render] [--tiny-net]
Returns (as a module: make(...)) the path of the config file."""
import argparse
import json
import math
import os
import sys

import numpy as np
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ANGLE_X = 0.6911112070083618


def net(tiny):
    return dict(num_layers=4 if tiny else 8, skip_step=4, encoding="positional", num_layers_view=-1, hidden_size=128 if tiny else 256,
                include_input_xyz=True, log_sampling_xyz=True, num_encoding_fn_xyz=6 if tiny else 10, include_input_dir=True,
                num_encoding_fn_dir=4, log_sampling_dir=True, use_viewdirs=True)


def config(out_dir, model="NeRFModel", tiny=True, train_iters=24, rays=512, size=40):
    buff = model == "BuFFModel"
    cfg = {
        "experiment": dict(id="synthetic-lego", model=model, description="synthetic plumbing run", logdir=os.path.join(out_dir, "logs"),
                           randomseed=42, train_iters=train_iters, validate_every=12, print_every=6, meshdir=os.path.join(out_dir, "meshes"),
                           use_early_stopping=False, early_stopping_step=25, chamfer_loss=False, chamfer_sampling_size=2400),
        "logging": dict(use_acronyms=True, use_projection=False, projection_step_size=5000),
        "dataset": dict(type="blender", basedir=os.path.join(out_dir, "data"), reduced_resolution=1, testskip=1, use_ndc=False, near=2, far=6,
                        empty=0.0, num_workers=0, llff_downsample_factor=8, llff_hold_step=8, white_background=False,
                        caching=dict(use_caching=False, override_caching=False, cache_dir=os.path.join(out_dir, "cache"), num_variations=4,
                                     sample_all=True)),
        "models": dict(coarse_type="FlexibleNeRFModel", coarse=net(tiny), fine_type="FlexibleNeRFModel", use_fine=not buff, fine=net(tiny)),
        "optimizer": dict(type="Adam", lr=5.0e-3 if tiny else 5.0e-4),
        "scheduler": dict(type="DefaultScheduler", options=dict(gamma=0.1, step_size=450000)),
        "nerf": dict(use_viewdirs=True, encode_position_fn="positional_encoding", encode_direction_fn="positional_encoding",
                     train=dict(num_random_rays=rays, chunksize=rays, perturb=True, num_coarse=192 if buff else 64, num_fine=128,
                                radiance_field_noise_std=0.2, lindisp=False),
                     validation=dict(chunksize=size * size, perturb=False, num_coarse=192 if buff else 64, num_fine=128,
                                     radiance_field_noise_std=0.0, lindisp=False, num_samples=1)),
    }
    if buff:
        cfg["tree"] = dict(subdivision_outer_count=2, subdivision_inner_count=2, max_depth=1, eps=0.0, max_voxel_count=64, step_size_tree=12,
                           step_size_integration_offset=0)
    return cfg


def make(out_dir, size=40, views=(6, 2, 2), render=False, **cfg_kw):
    from PIL import Image
    data = os.path.join(out_dir, "data")
    eng = None
    if render:
        import torch
        import nerfmeshes_b200 as nm
        from bench import load_npz, model_cfg
        model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
        eng = model._engine()
    focal = 0.5 * size / math.tan(0.5 * ANGLE_X)
    rng = np.random.default_rng(0)
    from nerfmeshes_b200.nerf_api import pose_spherical
    angle = 0.0
    for split, n in zip(("train", "val", "test"), views):
        os.makedirs(os.path.join(data, split), exist_ok=True)
        frames = []
        for i in range(n):
            pose = pose_spherical(-180.0 + angle, -30.0, 4.0)
            angle += 360.0 / sum(views)
            if eng is not None:
                rgb = eng.render_image(pose, size, size, focal, 2.0, 6.0, want=["rgb"])["rgb"].view(size, size, 3).clamp(0, 1)
                img = (rgb.cpu().numpy() * 255).astype(np.uint8)
            else:
                img = rng.integers(0, 255, (size, size, 3), dtype=np.uint8)
            Image.fromarray(np.concatenate([img, np.full((size, size, 1), 255, np.uint8)], -1)).save(os.path.join(data, split, f"r_{i}.png"))
            frames.append({"file_path": f"./{split}/r_{i}", "rotation": 0.0, "transform_matrix": pose.tolist()})
        with open(os.path.join(data, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": ANGLE_X, "frames": frames}, f)
    path = os.path.join(out_dir, "config.yml")
    with open(path, "w") as f:
        yaml.dump(config(out_dir, size=size, **cfg_kw), f)
    return path


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--size", type=int, default=40)
    ap.add_argument("--views", type=int, nargs=3, default=[6, 2, 2])
    ap.add_argument("--render", action="store_true")
    ap.add_argument("--full-net", action="store_true")
    a = ap.parse_args()
    print(make(a.out_dir, a.size, tuple(a.views), a.render, tiny=not a.full_net))
