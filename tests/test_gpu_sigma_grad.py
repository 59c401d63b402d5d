"""The density gradient nm_sigma_grad (DESIGN 4.8) on the GPU: against the float64 reference of tests/_sigma_grad_ref.py
at the tile and round edges of test_gpu_mlp_edges, its sigma output, determinism, side effects, and the mesh path's
network normals (single GPU and sharded).

Agreement: |g - g_ref| <= tau * S per entry, S the reference's error scale, on the points whose relu gates lie further
than MU from their threshold (_mlp_ref.gate_margin; exact / fp32 against the truth's margins MU_EXACT, fast mode
MU_FAST).  tau: _sigma_grad_ref.TAU_*, >= 4x the worst ratio measured on an H100.
"""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _mlp_ref as R
import _sigma_grad_ref as SG
from conftest import ROOT
from oracle import nerf_oracle as O
from test_gpu_mlp_edges import PREC, _engine, _points, _rows, _sizes

pytestmark = pytest.mark.gpu


def _report(test, key, value):
    print(f"RATIO {test} {key} {value:.3e}")


@pytest.mark.parametrize("prec", ["exact", "fast", "fp32"])
@pytest.mark.parametrize("net", list(R.NETS))
def test_sigma_grad_matches_float64(net, prec):
    if prec == "fast" and net not in SG.FAST_NETS:
        pytest.skip("no point of a 256-wide net clears fast mode's gate margin")
    cfg = R.net_cfg(net)
    sd = O.init_weights(cfg, 13)
    eng = _engine(cfg, prec)
    eng.load_weights(0, sd)
    sizes = _sizes()
    pool, _ = _points(max(sizes), 17)
    pool = pool * 0.6                                      # the scene box of the shipped checkpoints (|p| <= 1.5)
    rows = {M: _rows(M) for M in sizes}
    U = np.unique(np.concatenate(list(rows.values())))
    pos = np.full(max(sizes), -1)
    pos[U] = np.arange(U.size)
    g_ref, S, sig_ref, rec = SG.sigma_grad_ref(cfg, sd, pool[U].double().numpy())
    keep = R.gate_margin(rec) >= (R.MU_FAST if prec == "fast" else R.MU_EXACT)
    assert keep.mean() >= (0.02 if prec == "fast" else 0.3), keep.mean()
    tau = dict(exact=SG.TAU_EXACT, fast=SG.TAU_FAST, fp32=SG.TAU_FP32)[prec]
    worst = 0.0
    for M in sizes:
        sigma, g = eng.sigma_grad(0, pool[:M].cuda())
        g = g.cpu().double().numpy()
        assert np.isfinite(g).all(), (net, prec, M)
        ix = pos[rows[M]]
        k = keep[ix]
        r = R.forward_ratio(g[rows[M]][k], g_ref[ix][k], S[ix][k])
        worst = max(worst, r)
        assert r <= tau, (net, prec, M, r)
    _report("sigma-grad", f"{net} {prec}", worst)
    eng.close()


@pytest.mark.parametrize("prec", ["exact", "fast", "fp32"])
def test_sigma_output_is_point_mlp_sigma(prec):
    """The sigma output is nm_point_mlp's sigma-only forward of the same precision, bit for bit."""
    for net in R.NETS:
        cfg = R.net_cfg(net)
        sd = O.init_weights(cfg, 5)
        eng = _engine(cfg, prec)
        eng.load_weights(0, sd)
        p, _ = _points(4097, 6)
        sigma, _ = eng.sigma_grad(0, p.cuda())
        ref = eng.point_mlp(0, p.cuda(), None, sigma_only=True)
        assert torch.equal(sigma, ref), (net, prec)
        eng.close()


@pytest.mark.parametrize("prec", ["exact", "fast", "fp32"])
def test_sigma_grad_is_deterministic_and_batch_independent(prec, monkeypatch):
    cfg = R.net_cfg("nerf256")
    sd = O.init_weights(cfg, 23)
    eng = _engine(cfg, prec)
    eng.load_weights(0, sd)
    p, _ = _points(4097, 24)
    p = p.cuda()
    _, full = eng.sigma_grad(0, p)
    _, again = eng.sigma_grad(0, p)
    assert torch.equal(full, again), "second run differs"
    for i in (0, 63, 64, 2049, 4096):
        _, alone = eng.sigma_grad(0, p[i:i + 1])
        assert torch.equal(alone[0], full[i]), (prec, i)
    _, shifted = eng.sigma_grad(0, p[5:])                 # every point at another tile position
    assert torch.equal(shifted, full[5:])
    monkeypatch.setenv("NM_SIGMA_GRAD_CHUNK_POINTS", "1000")   # chunk boundaries at 1000, 2000, ... (not tile aligned)
    _, chunked = eng.sigma_grad(0, p)
    assert torch.equal(chunked, full), "chunked walk differs"
    eng.close()


@pytest.mark.parametrize("prec", ["exact", "fp32"])
def test_sigma_grad_leaves_gradients_and_renders_untouched(prec):
    cfg = R.net_cfg("nerf256")
    sd = O.init_weights(cfg, 31)
    eng = _engine(cfg, prec)
    eng.load_weights(0, sd)
    p, d = _points(2000, 32)
    dout = torch.randn(2000, 4, generator=torch.Generator().manual_seed(33))
    eng.zero_grad()
    eng.debug_mlp_backward(0, p.cuda(), d.cuda(), dout.cuda())
    before = {k: eng.get_grad(0, k, torch.as_tensor(v)).cpu() for k, v in sd.items()}
    g = torch.Generator().manual_seed(34)
    dirs = torch.nn.functional.normalize(torch.randn(512, 3, generator=g), dim=-1).cuda()
    origins = (-4.0 * dirs).contiguous()
    r0 = eng.render_rays(origins, dirs, 2.0, 6.0)
    eng.sigma_grad(0, p.cuda() * 0.5)
    r1 = eng.render_rays(origins, dirs, 2.0, 6.0)
    after = {k: eng.get_grad(0, k, torch.as_tensor(v)).cpu() for k, v in sd.items()}
    for k in before:
        assert torch.equal(before[k], after[k]), k
    for k in r0:
        assert torch.equal(r0[k], r1[k]), k
    eng.close()


def test_sigma_grad_argument_checks():
    cfg = R.net_cfg("tiny")
    eng = _engine(cfg, "exact")
    eng.load_weights(0, O.init_weights(cfg, 1))
    import nerfmeshes_b200._lib as L
    p = torch.zeros(4, 3, device="cuda")
    g = torch.empty(4, 3, device="cuda")
    lib, h, st = eng.lib, eng._h, eng._stream()
    ptr = lambda t: t.data_ptr()
    assert lib.nm_sigma_grad(h, 0, None, 4, None, ptr(g), st) != 0
    assert lib.nm_sigma_grad(h, 0, ptr(p), 4, None, None, st) != 0
    assert lib.nm_sigma_grad(h, 0, ptr(p), -1, None, ptr(g), st) != 0
    assert lib.nm_sigma_grad(h, L.NET_FINE, ptr(p), 4, None, ptr(g), st) != 0      # coarse-only handle
    assert lib.nm_sigma_grad(h, 0, ptr(p), 0, None, ptr(g), st) == 0
    s, gg = eng.sigma_grad(0, torch.zeros(0, 3))
    assert s.shape == (0,) and gg.shape == (0, 3)
    eng.close()


def test_density_gradient_uses_the_sweep_network():
    """BaseModel.density_gradient is Engine.sigma_grad on the net sample_points and the grid sweep use: the fine slot of a
    coarse + fine NeRFModel (which differs from the coarse slot there), the only (coarse) slot of a BuFFModel."""
    import nerfmeshes_b200 as nm
    import nerfmeshes_b200._lib as L
    from conftest import load_npz
    from test_gpu_parity import BUFF_CFG, LEGO_CFG
    p, _ = _points(3000, 41)
    p = (p * 0.5).cuda()
    nerf = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()
    sig, g = nerf.density_gradient(p)
    eng = nerf._engine()
    sf, gf = eng.sigma_grad(L.NET_FINE, p)
    _, gc = eng.sigma_grad(L.NET_COARSE, p)
    assert torch.equal(sig, sf) and torch.equal(g, gf) and not torch.equal(g, gc)
    buff = nm.BuFFModel.from_npz(BUFF_CFG, load_npz("weights_lego_buff.npz")).eval()
    sig, g = buff.density_gradient(p)
    sb, gb = buff._engine().sigma_grad(L.NET_COARSE, p)
    assert torch.equal(sig, sb) and torch.equal(g, gb)


# ----------------------------------------------------------------------------------------------------- mesh path
@pytest.fixture(scope="module")
def lego_model():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    return nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()


# Fraction of vertices whose network normal points the grid normal's way, measured on the lego weights at res 48 on an H100:
# 0.707 at s = 0, 0.784 at s = 2.  Which one is wrong where they disagree is measured by tools/mesh_normals_bench.py against
# the oriented face normals of the 512^3 s = 7 mesh (DESIGN 4.8): at 256^3 s = 0 the network normal is right in 43 % of the
# disagreements (it is evaluated up to a cell off the network's surface), at s = 3 in 82 %.  This bound only pins the
# present behaviour; the directional finite difference below is what checks the normals are the network's gradient.
MIN_SAME_SIDE = 0.65


@pytest.mark.parametrize("s", [0, 2])
def test_mesh_network_normals(lego_model, s):
    import nerfmeshes_b200 as nm
    base = dict(limit=1.2, res=48, iso_level=32.0, super_sampling=s)
    v0, f0, n0, d0 = nm.extract_geometry(lego_model, "cuda", SimpleNamespace(**base))
    vd, fd, nd, _ = nm.extract_geometry(lego_model, "cuda", SimpleNamespace(**base, network_normals=False))
    assert torch.equal(v0, vd) and torch.equal(f0, fd) and torch.equal(n0, nd)        # default path unchanged
    v1, f1, n1, d1 = nm.extract_geometry(lego_model, "cuda", SimpleNamespace(**base, network_normals=True))
    assert torch.equal(v0, v1) and torch.equal(f0, f1) and np.array_equal(d0, d1)
    assert v1.shape[0] > 100
    norm = n1.double().norm(dim=1)
    assert (norm - 1).abs().max() < 1e-5
    same = float(((n1 * n0).sum(1) > 0).double().mean())
    _report("mesh-same-side", f"s={s}", same)
    assert same >= MIN_SAME_SIDE, same
    # directional finite difference of sigma along the normal at the sweep coordinates: d sigma / dn = g . n = -|g|
    eng = lego_model._engine()
    which = lego_model.get_model()._owner[1]
    lins = [torch.linspace(-1.2, 1.2, 48) for _ in range(3)]
    # the index coordinates of the vertices: invert the exported rescale on the host (exact enough for a finite difference)
    vidx = ((v1.double() / 1.2 + 1.0) * 24.0).float().cuda()
    x = nm.mesh.sweep_coordinates(vidx, lins)
    _, g = eng.sigma_grad(which, x, want_sigma=False)
    gn = g.double().norm(dim=1)
    ok = torch.isfinite(gn) & (gn > 0)                     # the few vertices that keep their grid normal
    assert ok.double().mean() > 0.99
    x, g, gn = x[ok], g[ok], gn[ok]
    n = (-g.double() / gn[:, None]).float()
    h = 2e-4
    sp = eng.point_mlp(which, x + h * n, None, sigma_only=True).double()
    sm = eng.point_mlp(which, x - h * n, None, sigma_only=True).double()
    fd_ = (sp - sm) / (2 * h)
    rel = ((fd_ + gn).abs() / gn).cpu().numpy()
    _report("mesh-fd-median", f"s={s}", float(np.median(rel)))
    assert np.median(rel) < 0.05 and (rel < 0.25).mean() > 0.9, (np.median(rel), (rel < 0.5).mean())


def test_sharded_network_normals_match_single_gpu(lego_model):
    from nerfmeshes_b200 import parallel as par
    import nerfmeshes_b200 as nm
    A = SimpleNamespace(limit=1.2, res=40, iso_level=32.0, super_sampling=0, network_normals=True)
    v1, f1, n1, _ = par.extract_geometry_sharded(lego_model, A, group=par.SINGLE)
    v0, f0, n0, _ = nm.extract_geometry(lego_model, "cuda", A)
    assert torch.equal(v0, v1) and torch.equal(f0, f1) and torch.equal(n0, n1)


@pytest.mark.multigpu
def test_multi_gpu_network_normals():
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs 2 GPUs")
    port = 29900 + os.getpid() % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "_sigma_grad_multi_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and f"SIGMA_GRAD_MULTI_OK {world}" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
