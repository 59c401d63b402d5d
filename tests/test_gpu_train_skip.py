"""Empty-space skipping in training on the GPU (NM_FLAG_SKIP_EMPTY_TRAIN, DESIGN 4.15), in exact and NM_PREC_FP32 precision:
an all-occupied grid trains exactly as the dense step (outputs bit for bit, gradients within atomic-order noise) and an
all-empty one launches no network work and leaves the gradients zero; on lego NeRF and lego BuFF with the default grid, every
ray whose skipped samples all have a noisy pre-activation <= 0 keeps the dense step's outputs bit for bit and its gradients;
the results do not depend on the walk, the network launch size or the ray chunk; the rebuild schedule of
BaseModel.enable_training_skip, the stale-grid rule and the error paths."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_occupancy import LEGO_FOCAL, ROOT, bits, pose, sigma_at
from test_gpu_train import ATOMIC_NOISE, compare

pytestmark = pytest.mark.gpu

STD = 0.2                  # the training noise of the lego runs
BOX_MULLER = 5.7           # |randn| < sqrt(-2 ln 1e-7) = 5.68: sigma <= -5.7 std stays <= 0 whatever the noise draws
# lego, two 64x64 ring views, noise 0.2, perturb on, default grid (res 128, threshold -10, dilate 2): the share of rays proven
# to keep the dense step's bits and the fraction of network points evaluated, each with a margin over what an H100 run gave
# (printed by the test)
LEGO_CONFORM_BOUND = 0.99          # measured 0.9995 (NVIDIA H100 80GB HBM3, 700 W), exact and fp32
LEGO_TRAIN_EVAL_BOUND = 0.40       # measured 0.332
BUFF_CONFORM_BOUND = 0.99         # measured 0.9999


@pytest.fixture(autouse=True)
def _release():
    """the models hold a cycle to their engine: collect it after each test, so that the next one gets the training
    workspaces (tens of GB at these batch sizes) back"""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _lego(precision=None, **over):
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    m = nm.NeRFModel.from_npz({**LEGO_CFG, "nerf.train.perturb": True, "nerf.train.radiance_field_noise_std": STD, **over},
                              load_npz("weights_lego_nerf.npz")).cuda().train()
    if precision is not None:
        m.precision = precision
    return m


def _buff():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import BUFF_CFG
    m = nm.BuFFModel.from_npz({**BUFF_CFG, "nerf.train.perturb": True, "nerf.train.radiance_field_noise_std": STD},
                              load_npz("weights_lego_buff.npz")).cuda().train()
    return m


def ring_rays(eng, thetas, H=64):
    focal = LEGO_FOCAL * H / 800
    os_, ds = [], []
    for th in thetas:
        o, d = eng.ray_bundle(pose(th), H, H, focal)
        d = d.reshape(-1, 3)
        os_.append(o.reshape(1, 3).expand_as(d))
        ds.append(d)
    return torch.cat(os_).contiguous(), torch.cat(ds).contiguous()


def grads(model, eng):
    return {f"{w}.{k}": eng.get_grad(w, k, p).cpu() for w, k, p in model._named_net_params()}


def conservative(eng, which, o, d, t):
    """per ray: every sample network `which`'s grid skips among t has sigma <= -5.7 std (or NaN)"""
    sg, ev = sigma_at(eng, which, o.cpu().numpy(), d.cpu().numpy(), t.cpu().numpy())
    with np.errstate(invalid="ignore"):
        return (ev | ~(sg > -BOX_MULLER * STD)).all(1)


def set_all(eng, nets, value):
    G = 8
    w = torch.full((eng.occupancy_words(G),), value, dtype=torch.int32, device=eng.device)
    for which in nets:
        eng.set_occupancy(which, (-100, -100, -100, 100, 100, 100), G, w)


def _renders_and_grads(model, eng, o, d, target, seed, skip, buff=False, mask=None):
    want = ["rgb", "weights", "mask_weights", "t_vals"] + ([] if buff else ["coarse_rgb"])
    out = {k: v.clone() for k, v in eng.render_rays(o, d, 2.0, 6.0, training=True, buff=buff, seed=seed, want=want,
                                                     train_skip=skip).items()}
    g = torch.rand(d.shape[0], 3, generator=torch.Generator().manual_seed(seed)).cuda() - 0.5
    if mask is not None:
        g = g * mask[:, None].to(g)
    eng.zero_grad()
    eng.backward_rays(o, d, 2.0, 6.0, g, None if buff else g * 0.5, training=True, buff=buff, seed=seed, train_skip=skip)
    gr = grads(model, eng)
    loss = None
    if target is not None:
        eng.zero_grad()
        loss = eng.loss_backward(o, d, 2.0, 6.0, target, training=True, buff=buff, seed=seed, train_skip=skip).cpu()
        gr.update({"loss." + k: v for k, v in grads(model, eng).items()})
    return out, gr, loss


@pytest.mark.parametrize("prec", ["exact", "fp32"])
def test_all_occupied_grid_trains_as_dense(prec):
    import nerfmeshes_b200 as nm
    model = _lego(nm.PREC_FP32 if prec == "fp32" else None)
    eng = model._engine()
    o, d = ring_rays(eng, (40.0,), H=32)
    target = torch.rand(d.shape[0], 3, generator=torch.Generator().manual_seed(3)).cuda()
    set_all(eng, (0, 1), -1)
    dense, gd, ld = _renders_and_grads(model, eng, o, d, target, 11, False)
    skip, gs, ls = _renders_and_grads(model, eng, o, d, target, 11, True)
    st = eng.skip_stats()
    assert st["fine_evaluated"] == st["fine_seen"] > 0 and st["coarse_evaluated"] == st["coarse_seen"] > 0
    for k in dense:
        assert np.array_equal(bits(dense[k]), bits(skip[k])), k
    # the loss terms are atomic sums of block partials: equal up to their order
    assert torch.allclose(ls, ld, rtol=1e-6, atol=0), (ls, ld)
    compare(gs, gd, rel_max=ATOMIC_NOISE, name=f"all-occupied {prec}")


@pytest.mark.parametrize("prec", ["exact", "fp32"])
def test_all_empty_grid_launches_no_network_work(prec):
    import nerfmeshes_b200 as nm
    model = _lego(nm.PREC_FP32 if prec == "fp32" else None)
    eng = model._engine()
    o, d = ring_rays(eng, (40.0,), H=32)
    target = torch.rand(d.shape[0], 3, generator=torch.Generator().manual_seed(3)).cuda()
    set_all(eng, (0, 1), 0)
    for white in (False, True):
        eng.configure(white_background=white)
        eng.set_timing(True)
        n0 = eng.launch_count()
        out = eng.render_rays(o, d, 2.0, 6.0, training=True, seed=5, want=["rgb", "coarse_rgb"], train_skip=True)
        n1 = eng.launch_count()
        eng.zero_grad()
        eng.loss_backward(o, d, 2.0, 6.0, target, training=True, seed=5, train_skip=True)
        n2 = eng.launch_count()
        _, pts, launches = eng.mlp_time_ms()
        eng.set_timing(False)
        assert launches == 0 and pts == 0
        assert n2 - n1 == (n1 - n0) + 2, (n1 - n0, n2 - n1)     # the same forward, the two MSE gradients, no backward work
        bg = 1.0 if white else 0.0
        assert bool((out["rgb"] == bg).all()) and bool((out["coarse_rgb"] == bg).all())
        for k, v in grads(model, eng).items():
            assert bool((v == 0).all()), k
    assert eng.skip_stats()["fine_evaluated"] == 0


@pytest.mark.parametrize("prec", ["exact", "fp32"])
def test_lego_conforming_rays_train_as_dense(prec):
    import nerfmeshes_b200 as nm
    model = _lego(nm.PREC_FP32 if prec == "fp32" else None)
    model.build_occupancy_grid()
    model.skip_empty = False
    eng = model._engine()
    o, d = ring_rays(eng, (30.0, 210.0))
    seed = 1234
    dense, _, _ = _renders_and_grads(model, eng, o, d, None, seed, False)
    eng.skip_stats()
    skip, _, _ = _renders_and_grads(model, eng, o, d, None, seed, True)
    st = eng.skip_stats()
    frac = (st["coarse_evaluated"] + st["fine_evaluated"]) / (st["coarse_seen"] + st["fine_seen"])
    # coarse positions are a subset of the merged t_vals: checking the coarse net there too is conservative
    ok = conservative(eng, 0, o, d, dense["t_vals"]) & conservative(eng, 1, o, d, dense["t_vals"])
    share = float(ok.mean())
    print(f"lego training {prec}: evaluated fraction {frac:.4f} ({st}), conforming share {share:.4f}")
    assert share >= LEGO_CONFORM_BOUND, share
    assert frac < LEGO_TRAIN_EVAL_BOUND, frac
    for k in ("rgb", "coarse_rgb", "weights", "mask_weights", "t_vals"):
        a, b = bits(dense[k]).reshape(d.shape[0], -1), bits(skip[k]).reshape(d.shape[0], -1)
        bad = ~(a == b).all(1) & ok
        assert not bad.any(), (k, int(bad.sum()))
    # gradients of the conforming rays (d rgb = 0 on the others, in both runs)
    m = torch.from_numpy(ok).cuda()
    _, gd, _ = _renders_and_grads(model, eng, o, d, None, seed, False, mask=m)
    _, gs, _ = _renders_and_grads(model, eng, o, d, None, seed, True, mask=m)
    compare(gs, gd, rel_max=ATOMIC_NOISE, name=f"lego conforming {prec}")


def test_buff_conforming_rays_keep_weights_and_gradients():
    model = _buff()
    model.build_occupancy_grid()
    model.skip_empty = False
    eng = model._engine()
    model._sync_tree(eng)
    o, d = ring_rays(eng, (120.0, 300.0))
    seed = 77
    dense, _, _ = _renders_and_grads(model, eng, o, d, None, seed, False, buff=True)
    skip, _, _ = _renders_and_grads(model, eng, o, d, None, seed, True, buff=True)
    ok = conservative(eng, 0, o, d, dense["t_vals"])
    share = float(ok.mean())
    print(f"buff training: conforming share {share:.4f}")
    assert share >= BUFF_CONFORM_BOUND, share
    for k in ("rgb", "weights", "mask_weights", "t_vals"):
        a, b = bits(dense[k]).reshape(d.shape[0], -1), bits(skip[k]).reshape(d.shape[0], -1)
        assert not (~(a == b).all(1) & ok).any(), k
    m = torch.from_numpy(ok).cuda()
    _, gd, _ = _renders_and_grads(model, eng, o, d, None, seed, False, buff=True, mask=m)
    _, gs, _ = _renders_and_grads(model, eng, o, d, None, seed, True, buff=True, mask=m)
    compare(gs, gd, rel_max=ATOMIC_NOISE, name="buff conforming")


def _invariance_run(model, eng, o, d, target):
    r = eng.render_rays(o, d, 2.0, 6.0, training=True, seed=9, want=["rgb", "coarse_rgb", "t_vals"], train_skip=True)
    r = {k: v.cpu().numpy() for k, v in r.items()}
    eng.zero_grad()
    loss = eng.loss_backward(o, d, 2.0, 6.0, target, training=True, seed=9, train_skip=True)
    return r, loss.cpu().numpy(), {k: v.numpy() for k, v in grads(model, eng).items()}


def _invariance_setup(deterministic=False):
    """lego with noise 0.2 and jitter; `deterministic`: noise 0 and no jitter, whose samples and draws do not depend on
    the ray chunk (the chunk seed is seed + first ray: with noise or jitter, NM_CHUNK_RAYS moves the dense step's draws too)"""
    model = _lego(**({"nerf.train.perturb": False, "nerf.train.radiance_field_noise_std": 0.0} if deterministic else {}))
    model.build_occupancy_grid()
    model.skip_empty = False
    eng = model._engine()
    o, d = ring_rays(eng, (60.0,), H=48)
    target = torch.rand(d.shape[0], 3, generator=torch.Generator().manual_seed(4)).cuda()
    return model, eng, o, d, target


def test_independent_of_walk_launch_size_and_chunks(tmp_path, monkeypatch):
    model, eng, o, d, target = _invariance_setup()
    base = _invariance_run(model, eng, o, d, target)
    runs = {}
    monkeypatch.setenv("NM_TRAIN_DIRECT_GB", "0")
    runs["sub-chunk walk"] = _invariance_run(model, eng, o, d, target)
    monkeypatch.setenv("NM_SKIP_CHUNK_POINTS", "5000")
    runs["walk, 5000-point launches"] = _invariance_run(model, eng, o, d, target)
    monkeypatch.delenv("NM_TRAIN_DIRECT_GB")
    runs["direct, 5000-point launches"] = _invariance_run(model, eng, o, d, target)
    monkeypatch.delenv("NM_SKIP_CHUNK_POINTS")
    for name, run in runs.items():
        _same(name, run, base)
    # NM_CHUNK_RAYS is read once per process: a child trains with 333-ray chunks (draw-free configuration, see above)
    del model, eng
    gc.collect()
    model, eng, o, d, target = _invariance_setup(deterministic=True)
    base = _invariance_run(model, eng, o, d, target)
    out = tmp_path / "chunked.npz"
    code = f"""
import sys, numpy as np
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
import test_gpu_train_skip as T
model, eng, o, d, target = T._invariance_setup(deterministic=True)
r, loss, g = T._invariance_run(model, eng, o, d, target)
np.savez({str(out)!r}, loss=loss, **{{"r." + k: v for k, v in r.items()}}, **{{"g." + k: v for k, v in g.items()}})
"""
    subprocess.run([sys.executable, "-c", code], check=True, env={**os.environ, "NM_CHUNK_RAYS": "333"}, cwd=ROOT)
    z = np.load(out)
    _same("333-ray chunks", ({k[2:]: z[k] for k in z.files if k.startswith("r.")}, z["loss"],
                             {k[2:]: z[k] for k in z.files if k.startswith("g.")}), base)


def _same(name, run, base):
    """outputs the same bits, the loss and the gradients equal up to atomic order"""
    r, loss, g = run
    for k in base[0]:
        assert np.array_equal(r[k].view(np.int32), base[0][k].view(np.int32)), (name, k)
    assert np.allclose(loss, base[1], rtol=1e-6, atol=0), (name, loss, base[1])
    compare({k: torch.from_numpy(v) for k, v in g.items()}, {k: torch.from_numpy(v) for k, v in base[2].items()},
            rel_max=ATOMIC_NOISE, name=name)


def test_schedule_and_stale_grids():
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import train
    model = _lego(**{"nerf.train.chunksize": 1024})
    eng = model._engine()
    o, d = ring_rays(eng, (10.0, 100.0), H=32)
    target = torch.rand(d.shape[0], 3, generator=torch.Generator().manual_seed(6)).cuda()
    # training with the flag before any grid was built names the way to build one
    with pytest.raises(nm.NmError, match="enable_training_skip"):
        eng.loss_backward(o, d, 2.0, 6.0, target, training=True, seed=1, train_skip=True)
    model.enable_training_skip(every=3)
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    builds = []
    real = model._build_grids

    def spy(*a):
        builds.append(len(builds))
        return real(*a)
    model._build_grids = spy
    eng.skip_stats()
    for step in range(7):
        opt.zero_grad()
        out = train.training_step(model, (o, d, (2.0, 6.0)), target)
        assert np.isfinite(out["loss"])
        opt.step()
        if step in (0, 1):            # the weights moved: the grids are stale, and training keeps using them
            model._engine()
            assert eng._occupancy_stale == {0, 1} and not eng._occupancy
    assert model._train_skip["rebuilds"] == [0, 3, 6] and len(builds) == 3
    st = eng.skip_stats()
    assert 0 < st["fine_evaluated"] < st["fine_seen"]
    # eval-mode skipping is still build_occupancy_grid's: the grids predate the last weight update
    model.eval()
    model.skip_empty = True
    with pytest.raises(nm.NmError, match="build_occupancy_grid"):
        model.query((o[0], d[:64], (2.0, 6.0)))
    model.build_occupancy_grid()
    model.query((o[0], d[:64], (2.0, 6.0)))
    # the autograd route: forward in train mode ticks the schedule, its backward re-runs on the same grid
    model.train()
    model.enable_training_skip(every=2)
    model._build_grids = real
    for it in range(3):
        model.zero_grad(set_to_none=True)
        coarse, fine = model.forward((o, d, (2.0, 6.0)), seed=it)
        (torch.nn.functional.mse_loss(coarse.rgb_map, target) + torch.nn.functional.mse_loss(fine.rgb_map, target)).backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters() if p.requires_grad)
    assert model._train_skip["rebuilds"] == [0, 2]
    model.enable_training_skip(every=0)
    assert model._train_skip is None


def test_error_paths():
    import nerfmeshes_b200 as nm
    model = _lego()
    model.build_occupancy_grid()
    model.skip_empty = False
    eng = model._engine()
    o = torch.tensor([0.0, 0.0, 4.0]).cuda()
    d = torch.nn.functional.normalize(torch.randn(64, 3), dim=1).cuda()
    with pytest.raises(nm.NmError, match="needs NM_FLAG_TRAINING"):
        eng.render_rays(o, d, 2.0, 6.0, training=False, train_skip=True)
    with pytest.raises(nm.NmError, match="NM_FLAG_TEACHER_T"):
        eng.render_rays(o, d, 2.0, 6.0, training=True, train_skip=True,
                        teacher_t=torch.linspace(2, 6, 192).expand(64, 192).contiguous().cuda())
    with pytest.raises(nm.NmError, match="exclude each other"):
        eng.render_rays(o, d, 2.0, 6.0, training=True, skip_empty=True, train_skip=True)
    with pytest.raises(nm.NmError, match="NM_FLAG_TEACHER_T"):
        L = nm._lib
        import ctypes as C
        g = torch.zeros(64, 3).cuda()
        L.check(eng.lib.nm_backward_rays(eng._h, C.c_void_p(o.data_ptr()), 0, C.c_void_p(d.data_ptr()), 64,
                                         (C.c_float * 2)(2.0, 6.0), None, None,
                                         L.FLAG_TRAINING | L.FLAG_TEACHER_T | L.FLAG_SKIP_EMPTY_TRAIN, 0,
                                         C.c_void_p(g.data_ptr()), None, eng._stream()))
    # the library refuses a slot that never had a grid even when the binding is bypassed
    eng.set_occupancy(1, None, 0, None)
    eng._occupancy_stale.add(1)
    with pytest.raises(nm.NmError, match="no occupancy grid for network 1"):
        eng.render_rays(o, d, 2.0, 6.0, training=True, train_skip=True)
    with pytest.raises(nm.NmError, match="explicit box"):
        nm.NeRFModel.from_npz({**model.hparams, "dataset.use_ndc": True}, {}).enable_training_skip()
