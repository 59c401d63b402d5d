"""Empty-space skipping in training (NM_FLAG_SKIP_EMPTY_TRAIN, BaseModel.enable_training_skip; DESIGN 4.15) against the
dense training step, in two parts.

1. Step time: the lego checkpoint (tests/golden/weights_lego_nerf.npz) fine-tuned on its own dense renders of --views ring
   poses at --size^2 (theta = 360 k / views, phi = -30, radius 4), --rays random pixels per step, training noise 0.2, perturb
   on.  A dense and a skipping copy (every --every steps a rebuild at the default grid) take alternate steps in one process,
   each with its own Adam; a step is training_step + the optimiser step, host clock around synchronised calls.  Reports the
   median and the 10-90 % spread of each, the evaluated fraction of each pass over the skipping steps (nm_skip_stats), and
   the grid rebuild time amortised over --every (the median of 5 rebuilds; the skipping steps' median does not include it).
2. Convergence: distillation from scratch as tools/train_demo.py does it (same architecture, seed, views and schedule), dense
   against --every, for --conv-steps steps each; held-out PSNR against the teacher on --heldout ring poses between the
   training views at every --eval-every steps, and each run's wall time.

Prints one JSON line, with the card's name, power limit and SM clocks read in the same run.

    python tools/train_skip_bench.py [--steps 200] [--conv-steps 3000] [--every 16] [--out f.json]"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfmeshes_b200 as nm  # noqa: E402
from tools.mesh_render_bench import card  # noqa: E402
from tools.train_demo import CFG as DEMO_CFG  # noqa: E402

FOV = 0.6911112070083618


def lego_weights():
    raw = np.load(os.path.join(ROOT, "tests", "golden", "weights_lego_nerf.npz"))
    return {k: torch.from_numpy(raw[k]) for k in raw.files if raw[k].dtype.kind in "fiub"}


def sync_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def dataset(teacher, student, size, thetas):
    focal = 0.5 * size / np.tan(0.5 * FOV)
    views = []
    with torch.no_grad():
        for th in thetas:
            p = nm.pose_spherical(float(th), -30.0, 4.0)
            o, d = student._engine().ray_bundle(p, size, size, focal)
            rgb = teacher._engine().render_image(p, size, size, focal, 2.0, 6.0, want=["rgb"])["rgb"]
            views.append((o, d.reshape(-1, 3), rgb))
    return views, focal


def spread(ts):
    return dict(median=float(np.median(ts)), p10=float(np.percentile(ts, 10)), p90=float(np.percentile(ts, 90)),
                mean=float(np.mean(ts)), n=len(ts))


def step_time(a):
    z = lego_weights()
    teacher = nm.NeRFModel.from_npz(DEMO_CFG, z).cuda().eval()
    models = {"dense": nm.NeRFModel.from_npz(DEMO_CFG, z).cuda().train(),
              "skip": nm.NeRFModel.from_npz(DEMO_CFG, z).cuda().train()}
    models["skip"].enable_training_skip(every=a.every)
    views, _ = dataset(teacher, models["dense"], a.size, np.linspace(0, 360, a.views, endpoint=False))
    opts = {k: torch.optim.Adam(m.parameters(), lr=5e-4) for k, m in models.items()}
    g = torch.Generator(device="cuda").manual_seed(1)
    times = {"dense": [], "skip": []}
    stats = np.zeros(4, np.int64)
    losses = {"dense": [], "skip": []}
    for step in range(a.warmup + a.steps):
        o, d, rgb = views[step % len(views)]
        sel = torch.randint(0, d.shape[0], (a.rays,), device="cuda", generator=g)
        for k in ("dense", "skip") if step % 2 == 0 else ("skip", "dense"):
            m, opt = models[k], opts[k]

            def one():
                opt.zero_grad(set_to_none=True)
                out = nm.training_step(m, (o, d[sel], (2.0, 6.0)), rgb[sel], global_step=step)
                opt.step()
                return out
            out, ms = sync_ms(one)
            if step >= a.warmup:
                times[k].append(ms)
                losses[k].append(out["loss"])
        st = models["skip"]._engine().skip_stats()
        if step >= a.warmup:
            stats += np.array([st["coarse_seen"], st["coarse_evaluated"], st["fine_seen"], st["fine_evaluated"]])
    sk = models["skip"]
    ts = sk._train_skip
    rebuild = [sync_ms(lambda: sk._build_grids(ts["res"], ts["box"], ts["threshold"], ts["dilate"]))[1] for _ in range(6)][1:]
    # the rebuild steps are in the skipping list (every `every`-th step): their median is the plain step's
    skip_plain = [t for i, t in enumerate(times["skip"]) if (a.warmup + i) % a.every != 0]
    return dict(rays=a.rays, size=a.size, views=a.views, steps=a.steps, every=a.every,
                dense_ms=spread(times["dense"]), skip_ms=spread(times["skip"]), skip_ms_without_rebuild_steps=spread(skip_plain),
                rebuild_ms=float(np.median(rebuild)), rebuild_ms_amortised=float(np.median(rebuild)) / a.every,
                evaluated_fraction=dict(coarse=float(stats[1] / max(stats[0], 1)), fine=float(stats[3] / max(stats[2], 1)),
                                        all=float((stats[1] + stats[3]) / max(stats[0] + stats[2], 1))),
                final_loss=dict(dense=float(np.mean(losses["dense"][-20:])), skip=float(np.mean(losses["skip"][-20:]))))


def convergence(a, every):
    z = lego_weights()
    teacher = nm.NeRFModel.from_npz(DEMO_CFG, z).cuda().eval()
    torch.manual_seed(a.seed)
    student = nm.NeRFModel(DEMO_CFG).cuda().train()
    if every:
        student.enable_training_skip(every=every)
    opt = torch.optim.Adam(student.parameters(), lr=5e-4)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=lambda s: 0.1 ** (s / 250000))
    H = 200
    views, focal = dataset(teacher, student, H, np.linspace(-180, 180, 24, endpoint=False))
    held = [nm.pose_spherical(float(th), -30.0, 4.0) for th in np.linspace(-180, 180, a.heldout, endpoint=False) + 7.5]
    with torch.no_grad():
        refs = [teacher._engine().render_image(p, H, H, focal, 2.0, 6.0, want=["rgb"])["rgb"].clone() for p in held]

    def heldout_psnr():
        student.eval()
        with torch.no_grad():
            mse = [float(torch.mean((student._engine().render_image(p, H, H, focal, 2.0, 6.0, want=["rgb"])["rgb"] - r) ** 2))
                   for p, r in zip(held, refs)]
        student.train()
        return float(-10 * np.log10(np.mean(mse)))
    g = torch.Generator(device="cuda").manual_seed(1)
    curve, wall = [], 0.0
    for step in range(a.conv_steps):
        o, d, rgb = views[step % len(views)]
        sel = torch.randint(0, d.shape[0], (a.rays,), device="cuda", generator=g)

        def one():
            opt.zero_grad(set_to_none=True)
            nm.training_step(student, (o, d[sel], (2.0, 6.0)), rgb[sel], global_step=step)
            opt.step()
            sched.step()
        wall += sync_ms(one)[1] / 1e3
        if (step + 1) % a.eval_every == 0 or step + 1 == a.conv_steps:
            curve.append((step + 1, heldout_psnr()))
    st = student._engine().skip_stats()
    return dict(every=every, steps=a.conv_steps, wall_s=wall, heldout_psnr=curve,
                evaluated_fraction=(st["coarse_evaluated"] + st["fine_evaluated"]) / max(1, st["coarse_seen"] + st["fine_seen"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--every", type=int, default=16)
    ap.add_argument("--conv-steps", type=int, default=3000)
    ap.add_argument("--eval-every", type=int, default=500)
    ap.add_argument("--heldout", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    if a.steps > 0:
        res["step_time"] = step_time(a)
        print(json.dumps(res["step_time"]), flush=True)
    if a.conv_steps > 0:
        res["convergence"] = []
        for every in (0, a.every):
            gc.collect()                   # the previous part's engines (a model and its engine form a cycle) and their
            torch.cuda.empty_cache()       # training workspaces
            res["convergence"].append(convergence(a, every))
            print(json.dumps(res["convergence"][-1]), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
