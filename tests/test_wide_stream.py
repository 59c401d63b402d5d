"""CPU tests of the wide weight stream the fused MLP kernel reads (nm_program.h wide_offset): every element equals the
canonical 64x64 block image's, the image has, per layer, K-block and 128-column half, a hi and a lo stage (one [hi | lo]
block for a 64-wide layer), and the stage ring stays free of deadlock and early refills with the per-layer stage runs the
kernel walks in exact and in fast precision."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import nerf_oracle as O

import nerfmeshes_b200 as nm
from nerfmeshes_b200 import _lib as L

sys.path.insert(0, os.path.join(ROOT, "tools"))
from protocol_sim import simulate  # noqa: E402
from test_host_logic import NetProgram, debug_pack  # noqa: E402

ARCHS = [
    (dict(), False), (dict(), True),
    (dict(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6), False),
    (dict(num_layers=6, hidden_size=256, skip_step=2, num_encoding_fn_xyz=8, num_encoding_fn_dir=2, include_input_dir=False), False),
    (dict(num_layers=3, hidden_size=128, num_encoding_fn_xyz=5, use_viewdirs=False), False),
    (dict(num_layers=1, hidden_size=128, num_encoding_fn_xyz=4, use_viewdirs=False), False),
]


def debug_pack_wide(cfg: O.NetCfg, sd, sigma_only=False):
    lib = L.load()
    desc = nm.engine.net_desc(**cfg.__dict__)
    names = [k.encode() for k in sd]
    arrs = [np.ascontiguousarray(v.numpy(), dtype=np.float32) for v in sd.values()]
    n = len(names)
    prog = NetProgram()
    need = C.c_size_t(0)
    args = (C.byref(desc), n, (C.c_char_p * n)(*names), (C.c_void_p * n)(*[a.ctypes.data for a in arrs]),
            (C.c_int64 * n)(*[a.size for a in arrs]), int(sigma_only), C.byref(prog), C.sizeof(prog))
    L.check(lib.nm_debug_pack_wide(*args, None, 0, C.byref(need)))
    buf = np.zeros(need.value, dtype=np.uint8)
    L.check(lib.nm_debug_pack_wide(*args, buf.ctypes.data, buf.size, C.byref(need)))
    return prog, buf


def layer_stages(Lp, fast=False):
    """(MMA width, K-blocks, stages the kernel walks) of one layer."""
    W = min(Lp.n_out, 128)
    kbs = (1 if Lp.pe_src else 0) + Lp.k_act // 64
    return W, kbs, kbs * (Lp.n_out // W) * (2 if W == 128 and not fast else 1)


def wide_runs(prog, fast=False):
    return [layer_stages(prog.layers[i], fast)[2] for i in range(prog.n_layers) if prog.layers[i].kind != 4]


def unswizzle_rows(tile):
    """K-major 128B-swizzled tile of R rows x 64 16-bit columns -> (R, 64) uint16 (chunk c of row r stored at c ^ (r % 8))."""
    t = tile.view(np.uint16).reshape(-1, 8, 8)
    r = np.arange(t.shape[0])
    return np.concatenate([t[r, c ^ (r & 7)] for c in range(8)], axis=1)


@pytest.mark.parametrize("arch,sigma_only", ARCHS)
def test_wide_stream_holds_the_canonical_blocks(arch, sigma_only):
    cfg = O.NetCfg(**{**O.NetCfg().__dict__, **arch})
    sd = O.init_weights(cfg, seed=3)
    prog, canon = debug_pack(cfg, sd, sigma_only)
    progw, wide = debug_pack_wide(cfg, sd, sigma_only)
    assert bytes(progw) == bytes(prog)                 # the same program; only the image differs
    total = sum(wide_runs(prog))
    assert wide.size == total * 16384
    s0 = 0
    for li in range(prog.n_layers):
        Lp = prog.layers[li]
        N = Lp.n_out
        W, kbs, n_st = layer_stages(Lp)
        # the canonical blocks as (hi/lo, N rows, K-block, 64 columns); K-block 0 is the encoding when the layer has one
        ref = np.zeros((2, N, kbs, 64), np.uint16)
        for b in range(Lp.blk_begin, Lp.blk_end):
            B = prog.blocks[b]
            kbi = (B.kb + (1 if Lp.pe_src else 0)) if B.src == 0 else 0
            for h in range(2):
                ref[h, B.nc * 64:(B.nc + 1) * 64, kbi] = unswizzle_rows(canon[b * 16384 + h * 8192:b * 16384 + (h + 1) * 8192])
        got = np.full((2, N, kbs, 64), 0xFFFF, np.uint16)
        st = wide[s0 * 16384:(s0 + n_st) * 16384].reshape(n_st, 16384)
        if W == 128:                                   # stage ((kb * halves + half) * 2 + lo): 128 rows x 64 columns
            for s in range(n_st):
                kbi, half, lo = (s // 2) // (N // 128), (s // 2) % (N // 128), s % 2
                got[lo, half * 128:(half + 1) * 128, kbi] = unswizzle_rows(st[s])
        else:                                          # stage kb: [hi | lo] of 64 rows
            for s in range(n_st):
                for lo in range(2):
                    got[lo, :, s] = unswizzle_rows(st[s, lo * 8192:(lo + 1) * 8192])
        np.testing.assert_array_equal(got, ref)
        if Lp.pe_src:
            assert not ref[:, :, 0, Lp.k_pe:].any()    # encoding columns past its width are zero
        s0 += n_st
    assert s0 == total
    if not arch:
        # 8x256: as many stages as canonical blocks, and each is read from L2 once per 128 points in either precision
        assert total == (146 if not sigma_only else 120) == prog.n_blocks


@pytest.mark.parametrize("arch", [dict(), dict(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6),
                                  dict(num_layers=3, hidden_size=128, use_viewdirs=False)])
@pytest.mark.parametrize("sigma_only", [False, True])
def test_ring_protocol_with_wide_stage_runs(arch, sigma_only):
    cfg = O.NetCfg(**{**O.NetCfg().__dict__, **arch})
    prog, _ = debug_pack(cfg, O.init_weights(cfg, 1), sigma_only)
    for fast in (False, True):
        runs = wide_runs(prog, fast)
        for ns in (2, 3, 5, 8):
            for tiles in (1, 2, 3, 4):
                ok, info = simulate(prog, tiles=tiles, NS=ns, runs=runs)
                assert ok, (fast, ns, tiles, info)
