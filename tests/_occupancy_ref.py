"""numpy restatement of the occupancy grids of empty-space skipping (nm_occupancy.cu, DESIGN 4.15): the lattice, the
corner-max build with its Chebyshev dilation and bit packing, and the fp32 point lookup, bit for bit."""
import numpy as np

f32 = np.float32


def lattice(lo, hi, G):
    """torch.linspace(lo, hi, G+1) in fp32: step = (hi - lo) / G, lo + step*i below the midpoint and hi - step*(G-i) from
    it, each one fused multiply-add (exact product in float64, one rounding: the product of two fp32 values is exact there)."""
    lo, hi = f32(lo), f32(hi)
    step = f32(f32(hi - lo) / f32(G))
    n = G + 1
    i = np.arange(n)
    low = (np.float64(step) * i.astype(np.float64) + np.float64(lo))
    high = (-np.float64(step) * (G - i).astype(np.float64) + np.float64(hi))
    return np.where(i < n // 2, low, high).astype(f32)


def inv_scale(lo, hi, G):
    """G / (hi - lo) rounded once to fp32."""
    return f32(np.float64(G) / (np.float64(f32(hi)) - np.float64(f32(lo))))


def raw_occupancy(sigma, threshold):
    """sigma (G+1,G+1,G+1) lattice values -> bool (G,G,G): max of the 8 corners > threshold, or a NaN corner."""
    s = np.asarray(sigma, f32)
    corners = [s[a:a + s.shape[0] - 1, b:b + s.shape[1] - 1, c:c + s.shape[2] - 1] for a in (0, 1) for b in (0, 1) for c in (0, 1)]
    st = np.stack(corners)
    nan = np.isnan(st).any(0)
    with np.errstate(invalid="ignore"):
        mx = np.where(np.isnan(st), -np.inf, st).max(0)
    return nan | (mx > f32(threshold))


def dilate(occ, d):
    """Chebyshev dilation by d cells, clamped at the faces: three separable 1-D max filters."""
    out = occ.copy()
    G = occ.shape[0]
    for axis in (2, 1, 0):
        cur = out
        acc = np.zeros_like(cur)
        for s in range(-d, d + 1):
            sl_dst = [slice(None)] * 3
            sl_src = [slice(None)] * 3
            lo_d, hi_d = max(0, -s), min(G, G - s)
            sl_dst[axis] = slice(lo_d, hi_d)
            sl_src[axis] = slice(lo_d + s, hi_d + s)
            acc[tuple(sl_dst)] |= cur[tuple(sl_src)]
        out = acc
    return out


def pack(occ):
    """bool (G,G,G) -> uint32 words, bit (i*G + j)*G + k."""
    flat = np.asarray(occ, bool).reshape(-1)
    n = flat.size
    w = (n + 31) // 32
    padded = np.zeros(w * 32, bool)
    padded[:n] = flat
    b = padded.reshape(w, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)
    return b.sum(1).astype(np.uint32)


def unpack(bits, G):
    bits = np.asarray(bits).view(np.uint32)
    idx = np.arange(G * G * G)
    return ((bits[idx >> 5] >> (idx & 31).astype(np.uint32)) & 1).astype(bool).reshape(G, G, G)


def build(sigma, G, threshold, d):
    return pack(dilate(raw_occupancy(sigma, threshold), d))


def evaluated(pts, box, G, bits):
    """bool (M,): the point is outside [0, G) on an axis or not finite, or its cell's bit is set.  Cell index
    floor((p - lo) * inv) as a rounded fp32 subtract and a rounded fp32 multiply."""
    p = np.asarray(pts, f32).reshape(-1, 3)
    box = np.asarray(box, f32)
    lo, hi = box[:3], box[3:]
    inv = np.array([inv_scale(lo[a], hi[a], G) for a in range(3)], f32)
    with np.errstate(invalid="ignore", over="ignore"):
        c = np.floor(((p - lo).astype(f32) * inv).astype(f32))
        inside = ((c >= 0) & (c < f32(G))).all(1)
    ci = np.where(inside[:, None], c, 0).astype(np.int64)
    cell = (ci[:, 0] * G + ci[:, 1]) * G + ci[:, 2]
    w = np.asarray(bits).view(np.uint32)
    bit = ((w[cell >> 5] >> (cell & 31).astype(np.uint32)) & 1).astype(bool)
    return ~inside | bit
