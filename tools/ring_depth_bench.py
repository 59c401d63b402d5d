"""Lego render time against the fused MLP's weight-ring depth, and with the coarse pass on the sigma-only or the full program.

Renders bench.py's lego image (800x800, 64 + 128 samples) with the ring capped at each depth in --caps (NM_MLP_RING_SLOTS;
"max" is the layout's own depth), once with the maps bench.py asks for (rgb, depth, acc, disp: the coarse pass runs the
sigma-only program) and once with coarse_rgb as well (the coarse pass runs the full program).  Every variant runs --runs
times, alternating, each run timing --images images with CUDA events; the median ms per image and the range are reported
with the SM clock, power and power-capped fraction sampled during the runs, the card's name and its power limit, as one
JSON line.

    python tools/ring_depth_bench.py [--caps 2,3,max] [--runs 3] [--images 4] [--precision exact]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--caps", default="2,3,max")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--precision", default="exact", choices=["exact", "fast"])
    a = ap.parse_args()
    import nerfmeshes_b200 as nm
    wl = bench.WORKLOADS["lego"]
    model = nm.NeRFModel.from_npz(bench.model_cfg(wl["near"], wl["far"]), bench.load_npz(wl["weights"])).eval()
    model.precision = {"exact": nm.PREC_EXACT, "fast": nm.PREC_FAST}[a.precision]
    model.cuda(0)
    eng = model._engine()
    poses = bench.poses120()
    variants = [(cap, coarse_rgb) for cap in a.caps.split(",") for coarse_rgb in (False, True)]

    def render(i, coarse_rgb):
        want = ["rgb", "depth", "acc", "disp"] + (["coarse_rgb"] if coarse_rgb else [])
        return eng.render_image(poses[i % len(poses)], wl["H"], wl["W"], wl["focal"], wl["near"], wl["far"], want=want)

    def set_cap(cap):
        if cap == "max":
            os.environ.pop("NM_MLP_RING_SLOTS", None)
        else:
            os.environ["NM_MLP_RING_SLOTS"] = cap

    for cap, coarse_rgb in variants:           # warm-up of every variant
        set_cap(cap)
        render(0, coarse_rgb)
    torch.cuda.synchronize()
    ms = {v: [] for v in variants}
    clocks = {v: [] for v in variants}
    for _ in range(a.runs):
        for v in variants:
            set_cap(v[0])
            clk = bench.ClockSampler(0)
            clk.start()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.images):
                render(i, v[1])
            e1.record()
            torch.cuda.synchronize()
            ms[v].append(e0.elapsed_time(e1) / a.images)
            clocks[v].append(clk.stop())
    set_cap("max")
    props = torch.cuda.get_device_properties(0)
    res = {"card": props.name, "precision": a.precision, "images_per_run": a.images, "runs": a.runs, "variants": []}
    for v in variants:
        c = clocks[v]
        sm = [x["sm_mhz"] for x in c if x.get("sm_mhz")]
        med = float(np.median(ms[v]))
        sm_med = float(np.median(sm)) if sm else None
        res["variants"].append({
            "ring_slots": v[0], "coarse": "full" if v[1] else "sigma-only", "ms_per_image_median": round(med, 2),
            "ms_range": [round(min(ms[v]), 2), round(max(ms[v]), 2)],
            "sm_mhz_median": sm_med, "mcycles_per_image": round(med * sm_med / 1e3, 1) if sm_med else None,
            "power_w_median": float(np.median([x["power_w_median"] for x in c if x.get("power_w_median")] or [0])),
            "power_capped_frac": float(np.mean([x["power_capped_frac"] for x in c if x.get("power_capped_frac") is not None] or [0])),
            "power_limit_w": max([x["power_limit_w"] for x in c if x.get("power_limit_w")] or [0])})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
