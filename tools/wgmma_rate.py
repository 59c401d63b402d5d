"""Sustained wgmma rate of the fused MLP's exact-mode pattern (hi*hi, lo*hi, hi*lo per K = 16 step) across 256 output columns
as 4 x m64n64k16, 2 x m64n128k16 or 1 x m64n256k16 per pass (tools/wgmma_rate.cu): one CTA per SM, two warpgroups,
operands resident in shared memory; and the m64n128k16 pattern issued by one warpgroup per SM ("n128_1wg").  Each variant runs twice in alternation; the best of the two is reported, with the
card's name and power limit, as one JSON line.

    python tools/wgmma_rate.py [--seconds 2] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLOP_PER_ITER = 2 * 64 * 256 * 64 * 3          # one warpgroup, K = 64 across 256 columns, three passes
NAMES = {0: "n64", 1: "n128", 2: "n256", 3: "n128_1wg"}
WARPGROUPS = {0: 2, 1: 2, 2: 2, 3: 1}


def run(exe, iters):
    out = subprocess.run([exe, str(iters)], check=True, capture_output=True, text=True).stdout.split("\n")
    sms = int(out[0].split()[1])
    name = out[1].split(" ", 1)[1]
    ms = {}
    for line in out[2:]:
        if line.strip():
            v, t = line.split()
            ms.setdefault(int(v), []).append(float(t))
    return sms, name, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0, help="target time per timed launch")
    ap.add_argument("--out", default=None, help="directory for the binary (default: a temporary one)")
    a = ap.parse_args()
    out_dir = a.out or tempfile.mkdtemp(prefix="wgmma_rate_")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "wgmma_rate")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                    "-I", os.path.join(ROOT, "nerfmeshes_b200", "csrc"), os.path.join(ROOT, "tools", "wgmma_rate.cu"),
                    "-o", exe], check=True)
    sms, name, ms = run(exe, 2000)                                   # calibration
    iters = max(2000, int(2000 * a.seconds * 1e3 / max(ms[0])))
    sms, name, ms = run(exe, iters)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().split("\n")[0]
    res = {"card": name, "power_limit_and_max_sm_clock": smi, "sms": sms, "iters": iters}
    for v, ts in sorted(ms.items()):
        flop = FLOP_PER_ITER * WARPGROUPS[v] * sms * iters
        res[NAMES[v] + "_tflops"] = round(flop / (min(ts) * 1e-3) / 1e12, 1)
        res[NAMES[v] + "_ms"] = ts
    res["n256_over_n64"] = round(res["n256_tflops"] / res["n64_tflops"], 3)
    res["n128_over_n64"] = round(res["n128_tflops"] / res["n64_tflops"], 3)
    res["n128_1wg_over_2wg"] = round(res["n128_1wg_tflops"] / res["n128_tflops"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
