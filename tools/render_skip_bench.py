"""Empty-space skipping (NM_FLAG_SKIP_EMPTY, DESIGN 4.15) against the dense render: lego NeRF at --size^2 over --poses ring
poses (theta = 45 k, phi = -30, radius 4), lego BuFF at the same size over two of them, and fern NDC at its golden pose and
size (box --fern-box).  For each grid setting (--settings res:threshold:dilate, the first is the one reported as chosen):
grid build ms, then per scene the dense and the skipping image time (render_image: rgb, depth, acc, disp; host clock around
synchronised calls; the median of --reps after one warm-up of each), the evaluated fraction of the coarse and fine pass
(nm_skip_stats), the PSNR of the skipping image against the dense one, and the fraction of pixels whose rgb is the same
bits.  With --split, one more skipping render per scene with MLP timing on (nm_set_timing) splits its time into the network
launches and everything else (marks, scan, compaction, count read-back, expansion, the unfused compositor, the samplers).

Prints one JSON line with the card's name, power limit and SM clocks read in the same run.

    python tools/render_skip_bench.py [--size 800] [--poses 8] [--reps 5] [--settings 128:-10:2,128:0:2] [--out f.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.mesh_render_bench import card  # noqa: E402

LEGO_FOCAL = float(0.5 * 800 / np.tan(0.5 * 0.6911112))


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def median_ms(fn, reps):
    fn()
    return float(np.median([clock(fn)[1] for _ in range(reps)]))


def psnr(a, b):
    mse = float(((a - b) ** 2).mean())
    return float("inf") if mse == 0 else -10.0 * np.log10(mse)


def scene(eng, name, poses, render, reps, split):
    dense_ms, skip_ms, fracs, psnrs, ident, mlp_ms = [], [], [], [], [], []
    for P in poses:
        dense_ms.append(median_ms(lambda: render(P, False), reps))
        skip_ms.append(median_ms(lambda: render(P, True), reps))
        d = render(P, False)["rgb"].clone()
        eng.skip_stats()
        s = render(P, True)["rgb"].clone()
        st = eng.skip_stats()
        fracs.append([st["coarse_evaluated"] / max(1, st["coarse_seen"]), st["fine_evaluated"] / max(1, st["fine_seen"]),
                      (st["coarse_evaluated"] + st["fine_evaluated"]) / max(1, st["coarse_seen"] + st["fine_seen"])])
        psnrs.append(psnr(d.double(), s.double()))
        ident.append(float((d.view(torch.int32) == s.view(torch.int32)).all(1).float().mean()))
        if split:
            eng.set_timing(True)
            _, tot = clock(lambda: render(P, True))
            mlp = eng.mlp_time_ms()[0]
            eng.set_timing(False)
            mlp_ms.append([tot, mlp])
    f = np.array(fracs)
    r = dict(scene=name, images=len(poses), dense_ms=float(np.median(dense_ms)), skip_ms=float(np.median(skip_ms)),
             speedup=float(np.median(dense_ms) / np.median(skip_ms)), eval_coarse=float(f[:, 0].mean()),
             eval_fine=float(f[:, 1].mean()), eval_all=float(f[:, 2].mean()), psnr_min=float(min(psnrs)),
             identical_pixels=float(np.mean(ident)), identical_min=float(min(ident)))
    if split:
        m = np.array(mlp_ms)
        r.update(split_total_ms=float(m[:, 0].mean()), split_mlp_ms=float(m[:, 1].mean()))
    print(json.dumps(r), file=sys.stderr)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--poses", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--settings", default="128:-10:2")
    ap.add_argument("--fern-box", default="-1.5,-1.5,-1,1.5,1.5,1")
    ap.add_argument("--split", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_skip_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import BUFF_CFG, LEGO_CFG
    lego = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()
    buff = nm.BuFFModel.from_npz(BUFF_CFG, load_npz("weights_lego_buff.npz")).eval()
    fern = nm.NeRFModel.from_npz({**LEGO_CFG, "dataset.use_ndc": True}, load_npz("weights_fern_nerf.npz")).eval()
    g = load_npz("golden_fern_nerf.npz")
    fern_box = [float(x) for x in a.fern_box.split(",")]
    S, F = a.size, LEGO_FOCAL * a.size / 800
    poses = [np.asarray(nm.pose_spherical(45.0 * k, -30.0, 4.0), np.float32) for k in range(a.poses)]
    want = ("rgb", "depth", "acc", "disp")
    results = []
    for setting in a.settings.split(","):
        res, thr, dil = setting.split(":")
        res, thr, dil = int(res), float(thr), int(dil)
        row = dict(res=res, threshold=thr, dilate=dil, scenes=[])
        for name, model, box in (("lego", lego, None), ("buff", buff, None), ("fern_ndc", fern, fern_box)):
            model.skip_empty = False
            eng = model._engine()
            if name == "buff":
                model._sync_tree(eng)
            model.build_occupancy_grid(res=res, box=box, threshold=thr, dilate=dil)         # warm-up
            _, ms = clock(lambda: model.build_occupancy_grid(res=res, box=box, threshold=thr, dilate=dil))
            model.skip_empty = False
            eng = model._engine()
            row[f"build_ms_{name}"] = ms
            if name == "lego":
                r = scene(eng, name, poses, lambda P, s: eng.render_image(P, S, S, F, 2.0, 6.0, want=want, skip_empty=s), a.reps, a.split)
            elif name == "buff":
                r = scene(eng, name, poses[:2], lambda P, s: eng.render_image(P, S, S, F, 2.0, 6.0, buff=True, want=want, skip_empty=s),
                          a.reps, a.split)
            else:
                H, W, ff = int(g["H"]), int(g["W"]), float(g["focal"])
                r = scene(eng, name, [np.asarray(g["pose"], np.float32)],
                          lambda P, s: eng.render_image(P, H, W, ff, 0.0, 1.0, ndc=True, want=want, skip_empty=s), a.reps, a.split)
            row["scenes"].append(r)
        results.append(row)
    out = dict(card=card(), size=a.size, poses=a.poses, reps=a.reps, results=results)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
