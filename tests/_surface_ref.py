"""numpy float32 restatement of the surface point filter (nm_surface_points, DESIGN 4.14) and of the PLY encodings
(nm_export_ply), written from the contract the header states:
  t = depth_raw where acc >= min_acc, else 0;  P = o + d*t per component (two roundings);
  count(r,c) = #{(a,b) in [-s,s]^2 : (dx*dx + dy*dy) + dz*dz < thr}, d = P(clamp(r+a), clamp(c+b)) - P(r,c);
  keep = count >= min_count and t > 0;  rows of the kept pixels in row-major order: P, -d, rgb, r*W + c.
Every array operation below is one fp32 rounding per element, as the kernel's -fmad=false arithmetic is."""
import math

import numpy as np

f32 = np.float32


def min_count(step, prob_threshold):
    """floor(((2s+1)^2 - 1) * prob_threshold) + 1 in python doubles: the integer form of `sum > size_samples * prob`."""
    size = 2 * step + 1
    return math.floor((size * size - 1) * prob_threshold) + 1


def gate(depth_raw, acc, min_acc):
    return np.where(np.asarray(acc, f32) >= f32(min_acc), np.asarray(depth_raw, f32), f32(0)).astype(f32)


def surface_point_map(o, d, t):
    """(H,W,3): o (3,) + d (H,W,3) * t (H,W), per component."""
    o, d, t = np.asarray(o, f32), np.asarray(d, f32), np.asarray(t, f32)
    with np.errstate(invalid="ignore", over="ignore"):
        return (o[None, None, :] + d * t[..., None]).astype(f32)


def neighbour_counts(P, s, thr):
    """(H,W) int: clamped-neighbourhood counts of the point map P (H,W,3)."""
    H, W, _ = P.shape
    rows, cols = np.arange(H), np.arange(W)
    cnt = np.zeros((H, W), np.int64)
    thr = f32(thr)
    with np.errstate(invalid="ignore", over="ignore"):
        for a in range(-s, s + 1):
            for b in range(-s, s + 1):
                Q = P[np.clip(rows + a, 0, H - 1)][:, np.clip(cols + b, 0, W - 1)]
                e = (Q - P).astype(f32)
                d2 = ((e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]).astype(f32)
                cnt += d2 < thr
    return cnt


def surface_points(o, d, depth_raw, acc, rgb, H, W, *, min_acc=1.0, step=2, dist_threshold=0.002, min_count_=15):
    """The kept rows: (points (N,3), normals (N,3), colors (N,3), pixel (N,) int32, counts (H,W), keep mask (H,W))."""
    d = np.asarray(d, f32).reshape(H, W, 3)
    t = gate(np.asarray(depth_raw, f32).reshape(H, W), np.asarray(acc, f32).reshape(H, W), min_acc)
    P = surface_point_map(o, d, t)
    cnt = neighbour_counts(P, step, dist_threshold)
    keep = (cnt >= min_count_) & (t > 0)
    idx = np.flatnonzero(keep.reshape(-1))
    col = np.asarray(rgb, f32).reshape(-1, 3)
    return (P.reshape(-1, 3)[idx], (-d).reshape(-1, 3)[idx], col[idx], idx.astype(np.int32), cnt, keep)


# ------------------------------------------------------------------------------------------------ PLY
def quantise(colors):
    """trunc(fl32(c*255)) clamped to [0, 255], NaN to 0."""
    v = (np.asarray(colors, f32) * f32(255)).astype(f32)
    out = np.zeros(v.shape, np.uint8)
    with np.errstate(invalid="ignore"):
        big, mid = v >= 255, (v > 0) & (v < 255)
    out[big] = 255
    out[mid] = v[mid].astype(np.int64).astype(np.uint8)     # a cast of a positive value truncates
    return out


def ply_bytes(points, colors, normals, binary=False):
    p, n = np.asarray(points, f32).reshape(-1, 3), np.asarray(normals, f32).reshape(-1, 3)
    q = quantise(np.asarray(colors, f32).reshape(-1, 3))
    head = ["ply", "format binary_little_endian 1.0" if binary else "format ascii 1.0", f"element vertex {len(p)}"]
    head += [f"property float {k}" for k in ("x", "y", "z", "nx", "ny", "nz")]
    head += [f"property uchar {k}" for k in ("red", "green", "blue")]
    head.append("end_header")
    out = ("\n".join(head) + "\n").encode()
    if binary:
        import struct
        return out + b"".join(struct.pack("<6f3B", *p[i].tolist(), *n[i].tolist(), *q[i].tolist()) for i in range(len(p)))
    rows = []
    for i in range(len(p)):
        vals = ["%.18g" % float(x) for x in list(p[i]) + list(n[i])] + ["%d" % int(x) for x in q[i]]
        rows.append(" ".join(vals) + "\n")
    return out + "".join(rows).encode()


def read_ply(data):
    """A small reader for what ply_bytes writes: (points, normals (N,3) float32, colours (N,3) uint8)."""
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode().split("\n")
    assert head[0] == "ply", head
    n = int(next(h for h in head if h.startswith("element vertex")).split()[2])
    names = [h.split()[2] for h in head if h.startswith("property")]
    assert names == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"], names
    body = data[end:]
    if "format binary_little_endian 1.0" in head:
        assert len(body) == 27 * n
        rec = np.frombuffer(body, dtype=[("p", "<f4", (3,)), ("n", "<f4", (3,)), ("c", "u1", (3,))], count=n)
        return rec["p"].copy(), rec["n"].copy(), rec["c"].copy()
    assert "format ascii 1.0" in head
    lines = body.decode().split("\n")
    assert lines[-1] == "" and len(lines) == n + 1
    vals = [ln.split(" ") for ln in lines[:-1]]
    assert all(len(v) == 9 for v in vals)
    a = np.array([[float(x) for x in v[:6]] for v in vals], np.float64).reshape(-1, 6)
    c = np.array([[int(x) for x in v[6:]] for v in vals], np.int64).reshape(-1, 3)
    return a[:, :3].astype(f32), a[:, 3:].astype(f32), c.astype(np.uint8)
