"""Per-launch time of the backward's weight-gradient GEMM (nm_gemm_tc.cu) through nm_debug_gemm: the pack kernels run
once, the GEMM NM_GEMM_REPEAT times; (t(repeat=R) - t(repeat=1)) / (R-1).

    python tools/gemm_bench.py M N K REPEAT        (A: (K,M), B: (K,N), K = points)
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import nerfmeshes_b200 as nm


ARCH = dict(num_layers=8, hidden_size=256, skip_step=4, num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True,
            include_input_dir=True, log_sampling_xyz=True, log_sampling_dir=True, use_viewdirs=True)


def run(M, N, K, rep):
    os.environ["NM_GEMM_REPEAT"] = str(rep)
    eng = nm.Engine(ARCH, None, nm.RenderSettings())
    a = torch.randn((K, M), device="cuda")
    b = torch.randn((K, N), device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    out = torch.zeros(M, N, device="cuda")
    ts = []
    for _ in range(3):
        ev[0].record()
        eng.debug_gemm(a, b, out=out)
        ev[1].record(); torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]))
    return min(ts)


if __name__ == "__main__":
    M, N, K, rep = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    t = run(M, N, K, rep)
    print(f"M={M} N={N} K={K} repeat={rep}: {t * 1e3:.1f} us total")
