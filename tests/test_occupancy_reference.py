"""The numpy restatement of the occupancy grids (_occupancy_ref, DESIGN 4.15) against an independently written brute force:
per-cell corner loops, per-cell Chebyshev neighbourhoods, per-point scalar lookups; synthetic density fields (a sphere, two
spheres, NaN corners) on non-cubic boxes and resolutions that are not powers of two; dilation at the box faces; points on
cell and box boundaries and non-finite points; the lattice against torch.linspace."""
import itertools

import numpy as np
import pytest
import torch

import _occupancy_ref as R

f32 = np.float32


def field(kind, box, G):
    lo, hi = np.asarray(box[:3], f32), np.asarray(box[3:], f32)
    axes = [R.lattice(lo[a], hi[a], G) for a in range(3)]
    x, y, z = np.meshgrid(*axes, indexing="ij")
    if kind == "sphere":
        s = 1.0 - np.sqrt((x - 0.1) ** 2 + (y + 0.2) ** 2 + z ** 2)
    elif kind == "two":
        s = np.maximum(0.4 - np.sqrt((x - 0.6) ** 2 + y ** 2 + z ** 2), 0.3 - np.sqrt((x + 0.7) ** 2 + (y - 0.3) ** 2 + z ** 2))
    else:                                            # negative everywhere but a few NaN corners
        s = np.full(x.shape, -5.0)
        s[1, 2, 0] = np.nan
        s[-1, -1, -1] = np.nan
    return s.astype(f32) * 10.0


def brute_build(sigma, G, thr, d):
    raw = np.zeros((G, G, G), bool)
    for i, j, k in itertools.product(range(G), repeat=3):
        vals = [sigma[i + a, j + b, k + c] for a in (0, 1) for b in (0, 1) for c in (0, 1)]
        finite = [v for v in vals if not np.isnan(v)]
        raw[i, j, k] = len(finite) < 8 or max(finite) > thr
    occ = np.zeros_like(raw)
    for i, j, k in itertools.product(range(G), repeat=3):
        occ[i, j, k] = raw[max(0, i - d):i + d + 1, max(0, j - d):j + d + 1, max(0, k - d):k + d + 1].any()
    return occ


def brute_lookup(p, box, G, occ):
    out = []
    for q in np.asarray(p, f32).reshape(-1, 3):
        ev, cell = False, []
        for a in range(3):
            lo, hi = f32(box[a]), f32(box[3 + a])
            inv = f32(G / (float(hi) - float(lo)))
            with np.errstate(invalid="ignore", over="ignore"):
                c = np.floor(f32(f32(q[a] - lo) * inv))
            if not (c >= 0 and c < G):
                ev = True
                break
            cell.append(int(c))
        out.append(ev or bool(occ[tuple(cell)]))
    return np.array(out)


BOXES = [(-1.5, -1.5, -1.5, 1.5, 1.5, 1.5), (-2.0, -1.0, -0.5, 1.25, 1.5, 0.75), (-1.1, -0.3, -2.0, 0.9, 2.1, 1.3)]


@pytest.mark.parametrize("kind", ["sphere", "two", "nan"])
@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("G,d,thr", [(5, 0, 0.0), (7, 1, -3.0), (12, 2, 0.0), (6, 6, 2.5)])
def test_build_matches_brute_force(kind, box, G, d, thr):
    s = field(kind, box, G)
    bits = R.build(s, G, thr, d)
    occ = brute_build(s, G, thr, d)
    assert np.array_equal(R.unpack(bits, G), occ)
    assert bits.size == (G ** 3 + 31) // 32
    if G ** 3 % 32:
        assert bits[-1] >> (G ** 3 % 32) == 0            # the tail of the last word is clear


def test_dilation_reaches_the_faces_and_stops_there():
    G = 9
    raw = np.zeros((G, G, G), bool)
    raw[0, 4, 8] = True
    occ = R.dilate(raw, 2)
    want = np.zeros_like(raw)
    want[0:3, 2:7, 6:9] = True
    assert np.array_equal(occ, want)
    assert np.array_equal(R.dilate(raw, 0), raw)
    assert R.dilate(raw, G).all()


@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("G", [5, 12, 128])
def test_lattice_is_torch_linspace(box, G):
    for a in range(3):
        t = torch.linspace(float(f32(box[a])), float(f32(box[3 + a])), G + 1, dtype=torch.float32).numpy()
        assert np.array_equal(R.lattice(box[a], box[3 + a], G).view(np.int32), t.view(np.int32))


@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("G", [5, 12])
def test_lookup_matches_brute_force(box, G):
    rng = np.random.default_rng(G)
    s = field("two", box, G)
    bits = R.build(s, G, 0.0, 1)
    occ = R.unpack(bits, G)
    lo, hi = np.asarray(box[:3], f32), np.asarray(box[3:], f32)
    rand = (lo - 0.3 + rng.random((400, 3)) * (hi - lo + 0.6)).astype(f32)
    # every lattice plane and box face, a neighbour ulp either side, and non-finite coordinates
    edges = []
    for a in range(3):
        for v in R.lattice(lo[a], hi[a], G):
            for w in (v, np.nextafter(v, f32(-np.inf)), np.nextafter(v, f32(np.inf))):
                q = rand[len(edges) % len(rand)].copy()
                q[a] = w
                edges.append(q)
    bad = rand[:12].copy()
    for i, v in enumerate([np.nan, np.inf, -np.inf] * 4):
        bad[i, i % 3] = v
    pts = np.concatenate([rand, np.array(edges, f32), bad])
    got = R.evaluated(pts, box, G, bits)
    assert np.array_equal(got, brute_lookup(pts, box, G, occ))
    assert got[-12:].all()                                 # non-finite points are always evaluated
    assert got.any() and not got.all()


def test_all_occupied_and_all_empty():
    G, box = 4, BOXES[1]
    s = field("sphere", box, G)
    assert R.unpack(R.build(s, G, -np.inf, 0), G).all()
    assert not R.unpack(R.build(s, G, np.inf, 0), G).any()
