"""CPU oracle of the chamfer evaluation (DESIGN 4.7): the splitmix64 draws, fp32 face areas and their float64 CDF, the fp32
barycentric point formula, float64 nearest neighbours (scipy cKDTree) and the chamfer means."""
import numpy as np
from scipy.spatial import cKDTree

_F = np.float32


def u01(seed, idx):
    """nm::u01 (nm_composite.cuh) for an array of indices: splitmix64 of (seed, idx), top 24 bits as a float in [0,1)."""
    idx = np.asarray(idx, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(seed % 2 ** 64) + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(40)).astype(np.float32) * _F(1.0 / 16777216.0)


def face_areas(v, f):
    """0.5 |(v1 - v0) x (v2 - v0)| in fp32, the kernel's operation order."""
    v = np.asarray(v, np.float32)
    f = np.asarray(f, np.int64)
    e1, e2 = v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return _F(0.5) * np.sqrt((cx * cx + cy * cy) + cz * cz)


def area_cdf(v, f):
    """Inclusive float64 prefix sum of the fp32 areas."""
    return np.cumsum(face_areas(v, f).astype(np.float64))


def sample_targets(seed, n, total):
    """u * total per sample: the face is the first f with cdf[f] > that."""
    return u01(seed, 3 * np.arange(n, dtype=np.uint64)).astype(np.float64) * total


def sample_faces(v, f, seed, n):
    cdf = area_cdf(v, f)
    return np.searchsorted(cdf, sample_targets(seed, n, cdf[-1]), side="right")


def sample_points(v, f, face_idx, seed):
    """The point of every sample given its face: w0 v0 + w1 v1 + w2 v2 in fp32, left to right."""
    v = np.asarray(v, np.float32)
    f = np.asarray(f, np.int64)[np.asarray(face_idx, np.int64)]
    k = np.arange(len(face_idx), dtype=np.uint64)
    a, b = u01(seed, 3 * k + np.uint64(1)), u01(seed, 3 * k + np.uint64(2))
    r = np.sqrt(a)
    w0, w1, w2 = _F(1) - r, r * (_F(1) - b), r * b
    return (w0[:, None] * v[f[:, 0]] + w1[:, None] * v[f[:, 1]]) + w2[:, None] * v[f[:, 2]]


def nearest64(q, p):
    """float64 squared distance to the nearest point of p and one nearest index."""
    d, i = cKDTree(np.asarray(p, np.float64)).query(np.asarray(q, np.float64))
    return d * d, i


def dist64(q, p, idx):
    """float64 squared distance from each query to point idx."""
    diff = np.asarray(q, np.float64) - np.asarray(p, np.float64)[np.asarray(idx, np.int64)]
    return (diff * diff).sum(1)


def chamfer64(x, y):
    """(mean_i d2(x_i, Y), mean_j d2(y_j, X)) in float64."""
    return nearest64(x, y)[0].mean(), nearest64(y, x)[0].mean()


def create_mesh(v):
    """mesh_nerf.create_mesh's vertex normalisation in float64 (for a hand-checked case)."""
    v = np.asarray(v, np.float64)
    v = v - v.mean(0)
    return v / np.abs(v).max()
