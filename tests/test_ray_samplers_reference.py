"""The restatements of the ray samplers (tests/_sampler_ref.py) on the CPU: against the oracle and the reference-generated
goldens where those define the answer, against the float64 truth of SamplePDF over the edge matrix that
tests/test_gpu_ray_samplers.py runs bit for bit on the device, every fault variant visible on that matrix, and the
random streams of one render pairwise disjoint."""
import numpy as np
import pytest
import torch

import _sampler_ref as SR
from conftest import load_npz
from oracle import nerf_oracle as O

F32 = np.float32

# ----------------------------------------------------------------------------------------------------- edge matrices
PDF_SHAPES = [(Nc, Nf) for Nc in (3, 64, 256) for Nf in (1, 2, 31, 33, 128)] + [(256, 256), (3, 509)]
W_KINDS = ("zero", "spike", "equal", "tiny", "random")
T_KINDS = ("uniform", "lindisp", "equal", "per_ray")


def pdf_inputs(R, Nc, Nf, wkind, tkind, perturb, seed):
    """(t_c (R,Nc) ascending, w_c (R,Nc), u (Nf,) or None).  Weights: all zero; one spike (the other steps fall below the
    denom floor); equal; around 1e-5; random with zeros.  Depths: stratified [2, 6] jittered; lindisp [0.5, 100]; near ==
    far (every depth ties); per-ray near in [0, 2], far up to 5 beyond.  Deterministic u: linspace(Nf), or for the spike
    and equal weights the kernel's own cdf knots of row 0 (every row has that cdf), so u sits exactly on a knot."""
    rng = np.random.default_rng(seed)
    s = SR.linspace(Nc)
    if tkind == "uniform":
        t = SR.stratified(s, 2.0, 6.0, False, True, seed=seed, R=R)
    elif tkind == "lindisp":
        t = SR.stratified(s, 0.5, 100.0, True, False, R=R)
    elif tkind == "equal":
        t = np.full((R, Nc), 3.0, F32)
    else:
        near = rng.uniform(0, 2, R).astype(F32)
        t = SR.stratified(s, near, (near + rng.uniform(0.1, 5, R)).astype(F32), False, False)
    if wkind == "zero":
        w = np.zeros((R, Nc), F32)
    elif wkind == "spike":
        w = np.zeros((R, Nc), F32)
        w[:, rng.integers(1, Nc - 1)] = 1.0
    elif wkind == "equal":
        w = np.full((R, Nc), 0.5, F32)
    elif wkind == "tiny":
        w = rng.uniform(0, 3e-5, (R, Nc)).astype(F32)
    else:
        w = (rng.exponential(1.0, (R, Nc)) * (rng.uniform(size=(R, Nc)) > 0.2)).astype(F32)
    u = None
    if not perturb:
        if wkind in ("spike", "equal"):
            cdf = SR.pdf_cdf(w[:1])[0]
            u = cdf[np.round(np.linspace(0, cdf.size - 1, Nf)).astype(int)]
        else:
            u = SR.linspace(Nf)
    return t, w, u


def pdf_cases(big=True):
    """(R, Nc, Nf, wkind, tkind, perturb, seed): every shape x perturb x weight kind, with R in 1, 3, 5 and the depth
    kinds cycling; with `big`, R = 4099 once per shape and perturb (R not a multiple of the 4 rays per block)."""
    n = 0
    for Nc, Nf in PDF_SHAPES:
        for perturb in (0, 1):
            for wkind in W_KINDS:
                for tkind in T_KINDS:
                    yield (1, 3, 5)[n % 3], Nc, Nf, wkind, tkind, perturb, 1000 + n
                    n += 1
            if big:
                yield 4099, Nc, Nf, W_KINDS[n % 5], T_KINDS[n % 4], perturb, 1000 + n
                n += 1


AABB_S = (3, 33, 192, 256)


def aabb_scene(kind):
    """(voxels (V,2,3), origins (R,3), dirs (R,3), near, far) of the synthetic AABB scenes:
    * grid: a 5x5x5 grid of unit boxes (V = 125); rays along shared faces and edges (entry ties, +-0 direction components,
      origins on slab planes), through corners, tilted, axis-aligned rays whose entry / exit distances are exact integers
      so that tmin == near and tmax == far occur, and rays that miss
    * stack: 40 overlapping boxes with one bottom face and shuffled heights (the voxel list may hold any boxes): every hit
      of a ray through the bottom enters at the same distance, so the order the hit sort leaves them in decides the
      samples
    * line: 600 unit boxes in a row (V = 600) and axis rays that hit 1, 32, 33, 512 or 600 of them (more than 512: the
      overflow path) inside [near, far]."""
    if kind == "grid":
        g = np.stack(np.meshgrid(*[np.arange(5)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(F32)
        vox = np.stack([g, g + 1], 1)
        o = [(1.0, 0.5, -1.0), (1.0, 1.0, -1.0), (2.0, 2.0, -1.0), (0.5, 1.0, -1.0), (-1.0, -1.0, -1.0),
             (-1.0, 2.0, 0.5), (0.25, 0.75, -1.0), (1.5, 1.5, -1.0), (6.0, 6.0, 6.0), (0.0, 0.0, -1.0), (3.0, 0.5, 2.5)]
        d = [(0.0, 0.0, 1.0), (-0.0, 0.0, 1.0), (0.0, -0.0, 1.0), (-0.0, -0.0, 1.0), (1.0, 1.0, 1.0), (1.0, 0.0, 0.0),
             (0.3, 0.2, 1.0), (0.0, 0.0, 1.0), (1.0, 1.0, 1.0), (1.0, 1.0, 0.5), (-0.0, 1.0, -0.0)]
        return vox, np.array(o, F32), np.array(d, F32), 1.0, 4.0
    if kind == "stack":
        top = (0.5 + 0.05 * np.random.default_rng(3).permutation(40)).astype(F32)
        vox = np.stack([np.zeros((40, 3), F32), np.stack([np.ones(40, F32), np.ones(40, F32), top], 1)], 1)
        o = np.array([(0.5, 0.5, -1.0), (0.25, 0.5, -1.0), (0.5, 0.5, -1.0)], F32)
        d = np.array([(0.0, 0.0, 1.0), (0.125, -0.0, 1.0), (0.0, -0.0, 2.0)], F32)
        return vox, o, d, 1.0, 4.0
    i = np.arange(600, dtype=F32)
    vox = np.stack([np.stack([i, 0 * i, 0 * i], 1), np.stack([i + 1, 0 * i + 1, 0 * i + 1], 1)], 1)
    o = np.array([(-0.5, 0.5, 0.5)] * 6 + [(-0.5, 2.5, 0.5)], F32)
    d = np.array([(1.0, 0.0, 0.0), (1.0, -0.0, 0.0), (1.0, 0.0, -0.0), (1.0, 0.0, 0.0), (1.0, 0.0, 0.0),
                  (1.0, -0.0, -0.0), (1.0, 0.0, 0.0)], F32)
    return vox, o, d, 0.5, None


LINE_HITS = (1, 32, 33, 512)


def line_far(hits):
    """far of the line scene that admits exactly `hits` boxes (box i spans t in [i + 0.5, i + 1.5])."""
    return hits + 0.5


def aabb_cases():
    """(scene, far, S, random, seed)."""
    for S in AABB_S:
        for random in (0, 1):
            yield "grid", None, S, random, 77 + S
            yield "stack", None, S, random, 91 + S
            for hits in LINE_HITS:
                yield "line", line_far(hits), S, random, 5 * hits + S


def run_aabb_ref(scene, far, S, random, seed, fault=None):
    vox, o, d, near, far0 = aabb_scene(scene)
    far = far0 if far is None else far
    tu = SR.stratified(SR.linspace(S), near, far, False, False, R=d.shape[0])
    return SR.aabb(vox, o, d, near, far, S, SR.linspace(S), tu, random=bool(random), seed=seed, fault=fault)


# ----------------------------------------------------------------------------------------------------- oracle / goldens
def test_linspace_is_torchs():
    for n in (1, 2, 3, 31, 33, 64, 128, 192, 256, 509):
        assert np.array_equal(SR.linspace(n), torch.linspace(0, 1, n).numpy()), n


@pytest.mark.parametrize("lindisp", [False, True])
def test_stratified_equals_oracle_unperturbed(lindisp):
    R = 9
    for Nc in (3, 64, 192):
        a = SR.stratified(SR.linspace(Nc), 2.0, 6.0, lindisp, False, R=R)
        assert np.array_equal(a, O.ray_sample_interval(Nc, R, torch.tensor(2.0), torch.tensor(6.0), lindisp=lindisp).numpy())
        near = np.random.default_rng(Nc).uniform(0.2, 2, R).astype(F32)
        far = near + F32(3)
        b = O.ray_sample_interval(Nc, R, torch.from_numpy(near), torch.from_numpy(far), lindisp=lindisp).numpy()
        assert np.array_equal(SR.stratified(SR.linspace(Nc), near, far, lindisp, False), b)


def test_stratified_perturbed_stays_in_its_interval():
    t0 = SR.stratified(SR.linspace(64), 2.0, 6.0, False, False, R=50)
    t = SR.stratified(SR.linspace(64), 2.0, 6.0, False, True, seed=5, R=50)
    mids = 0.5 * (t0[:, 1:] + t0[:, :-1])
    assert (t[:, 1:] >= mids).all() and (t[:, :-1] <= mids).all() and not np.array_equal(t, t0)


def test_aabb_reproduces_the_buff_golden():
    g = load_npz("golden_lego_buff.npz")
    vox = load_npz("weights_lego_buff.npz")["voxels"].float()
    near, far = float(g["bounds"][0]), float(g["bounds"][1])
    R = g["dirs"].shape[0]
    tu = SR.stratified(SR.linspace(192), near, far, False, False, R=R)
    z, idx, hits, over = SR.aabb(vox.numpy(), g["origin"].numpy(), g["dirs"].numpy(), near, far, 192, SR.linspace(192), tu)
    assert np.array_equal(z, g["z"].numpy()) and not over
    _, idx_ref, mask = O.batch_ray_voxel_intersect(vox, g["origin"][None], g["dirs"], near, far, 192, return_indices=True)
    mask = mask.numpy()
    assert np.array_equal(idx[mask], idx_ref.numpy()[mask].astype(np.int32)) and (idx[~mask] == -1).all()


def test_sample_pdf_against_the_lego_golden():
    """The golden's t_fine is torch's SamplePDF (another summation order of the cdf): the restated samples differ from
    torch's in the last bits wherever the cdf rounds differently, and by a bucket flip only where u is undecided."""
    g, z = load_npz("golden_lego_nerf.npz"), load_npz("weights_lego_nerf.npz")
    t, w, u = g["t_coarse"].numpy(), g["coarse_weights"].numpy(), z["sample_pdf_u"].numpy()
    out, smp, uu = SR.sample_pdf(t, w, u, u.size, False, full=True)
    mids = 0.5 * (g["t_coarse"][..., 1:] + g["t_coarse"][..., :-1])
    ref = O.sample_pdf(mids, g["coarse_weights"][..., 1:-1], torch.from_numpy(u)).numpy()
    assert np.array_equal(np.sort(np.concatenate([t, ref], 1), 1), g["t_fine"].numpy())      # the oracle is torch's bits
    s64, dec, lo, hi, B = SR.pdf_truth(t, w, uu)
    differ = smp != ref
    flips = differ & ~dec
    print(f"SamplePDF vs golden: {int((out != g['t_fine'].numpy()).sum())} of {out.size} merged depths differ; "
          f"{int(differ.sum())} of {smp.size} samples, {int(flips.sum())} of them at an undecided u (max |diff| "
          f"{float(np.abs(smp - ref)[flips].max(initial=0)):.3e}), the others by at most "
          f"{float(np.abs(smp - ref)[differ & dec].max(initial=0)):.3e}")
    # decided samples: both within the float64 bound; undecided ones: both inside the span of the candidate values
    assert (np.abs(smp - s64) <= B)[dec].all() and (np.abs(ref - s64) <= B)[dec].all()
    assert ((smp >= lo - B) & (smp <= hi + B) & (ref >= lo - B) & (ref <= hi + B))[~dec].all()


# ----------------------------------------------------------------------------------------------------- edge matrix
def test_sample_pdf_within_float64_bound_and_merge_is_a_sort():
    worst, undecided, n = 0.0, 0, 0
    for R, Nc, Nf, wk, tk, perturb, seed in pdf_cases(big=False):
        t, w, u = pdf_inputs(R, Nc, Nf, wk, tk, perturb, seed)
        out, smp, uu = SR.sample_pdf(t, w, u, Nf, perturb, seed, full=True)
        assert np.array_equal(out, np.sort(np.concatenate([t, smp], 1), 1)), (R, Nc, Nf, wk, tk, perturb)
        s64, dec, lo, hi, B = SR.pdf_truth(t, w, uu)
        with np.errstate(all="ignore"):
            r = np.where(dec, np.abs(smp - s64) / B, 0.0)
        r = np.where(dec & (np.abs(smp - s64) == 0), 0.0, r)
        worst = max(worst, float(r.max()))
        assert r.max() <= 1.0, (R, Nc, Nf, wk, tk, perturb, float(r.max()))
        assert ((smp >= lo - B) & (smp <= hi + B))[~dec].all(), (R, Nc, Nf, wk, tk, perturb)
        undecided += int((~dec).sum())
        n += dec.size
    print(f"RATIO restatement-vs-float64 {worst:.3f}; {undecided} of {n} samples undecided")
    assert undecided > 0


def test_edge_matrix_reaches_its_edges():
    knots = floor = clamp_top = unsorted = 0
    for R, Nc, Nf, wk, tk, perturb, seed in pdf_cases(big=False):
        t, w, u = pdf_inputs(R, Nc, Nf, wk, tk, perturb, seed)
        _, smp, uu = SR.sample_pdf(t, w, u, Nf, perturb, seed, full=True)
        cdf = SR.pdf_cdf(w)
        knots += int((uu[..., None] == cdf[:, None, :]).any(-1).sum())
        steps = np.diff(cdf, axis=1)
        floor += int(((steps > 0) & (steps < SR.THR)).sum())
        clamp_top += int((uu >= cdf[:, -1:]).sum())
        unsorted += int((smp[:, :-1] > smp[:, 1:]).any(1).sum())
    assert knots > 100 and floor > 100 and clamp_top > 10 and unsorted > 10, (knots, floor, clamp_top, unsorted)
    hits = {h for sc, far, S, rnd, sd in aabb_cases() for h in run_aabb_ref(sc, far, S, rnd, sd)[2].tolist()}
    assert {0, 1, 32, 33, 512} <= hits, sorted(hits)


def _changes(fault):
    if fault.startswith("strat"):
        return any(not np.array_equal(SR.stratified(SR.linspace(Nc), 2.0, 6.0, lind, True, seed=3, R=R),
                                      SR.stratified(SR.linspace(Nc), 2.0, 6.0, lind, True, seed=3, R=R, fault=fault))
                   for Nc in (3, 64) for R in (1, 5) for lind in (False, True))
    if fault.startswith("pdf"):
        for R, Nc, Nf, wk, tk, perturb, seed in pdf_cases(big=False):
            t, w, u = pdf_inputs(R, Nc, Nf, wk, tk, perturb, seed)
            a = SR.sample_pdf(t, w, u, Nf, perturb, seed)
            if not np.array_equal(a.view(np.uint32), SR.sample_pdf(t, w, u, Nf, perturb, seed, fault=fault).view(np.uint32)):
                return True
        return False
    for case in aabb_cases():
        a, b = run_aabb_ref(*case), run_aabb_ref(*case, fault=fault)
        if not (np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])):
            return True
    return False


@pytest.mark.parametrize("fault", SR.FAULTS)
def test_every_fault_changes_an_edge_matrix_output(fault):
    assert _changes(fault), fault


# ----------------------------------------------------------------------------------------------------- random streams
SEEDS = (0, 1, 11, 977, 0x2545F4914F6CDD1D, 2 ** 64 - 1, 2 ** 63)
CHUNKS = (0, 1, 2, 3, 2 ** 20)
MIN_DISTANCE = 2 ** 40           # far beyond any index range of one render (R*S*2 < 2^31 per chunk)


@pytest.mark.parametrize("buff", [False, True])
def test_render_streams_are_pairwise_disjoint(buff):
    """No two consumers of one render (over its chunk seeds seed + r0) share a splitmix64 state: u01(a, i) and u01(b, j)
    coincide iff j - i == (a - b) / G mod 2^64, so every pair must lie MIN_DISTANCE apart."""
    for seed in SEEDS:
        d, a, b = SR.closest_streams(SR.render_streams(seed, CHUNKS, buff))
        assert d >= MIN_DISTANCE, (seed, a, b, d)


def test_stream_check_sees_the_shared_noise_salt():
    """The random voxel draws on the noise salt (the layout before kVoxelSalt): the same state feeds draw k's voxel and the
    noise of sample k."""
    d, a, b = SR.closest_streams(SR.render_streams(0, (0,), True, voxel_salt=SR.SALT_MAIN))
    assert d == 0 and {a, b} == {"voxel@0", "noise@0"}
