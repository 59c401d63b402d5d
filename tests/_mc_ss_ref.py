"""ctypes wrapper of tests/mc_ss_oracle.c, the CPU oracle of super-sampled marching cubes (test infrastructure only).
The library is compiled once per process into a temporary directory (the source tree is not written)."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def _load():
    global _lib
    if _lib is not None:
        return _lib
    d = tempfile.mkdtemp(prefix="mc_ss_oracle_")
    atexit.register(shutil.rmtree, d, True)
    so = os.path.join(d, "libmc_ss_oracle.so")
    cc = os.environ.get("CC", "gcc")
    subprocess.run([cc, "-O2", "-fPIC", "-ffp-contract=off", "-std=c99", "-Wall", "-shared", "-o", so,
                    os.path.join(_HERE, "mc_ss_oracle.c"), "-lm"], check=True, capture_output=True)
    lib = C.CDLL(so)
    lib.mc_oracle_ss.restype = C.c_int
    lib.mc_oracle_ss.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                 C.c_longlong, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    _lib = lib
    return lib


def marching_cubes_ss(volume, iso, s, xvol, yvol, zvol, x_off=0, g_nx=None, own=None, v_base=0):
    """oracle.mc.marching_cubes with super-sampled edge vertices: (verts, faces, normals).  xvol / yvol / zvol: the dense fine
    volumes of the GLOBAL grid, each refined along one axis to (n-1)(s+1)+1 samples.  Other arguments as oracle.mc."""
    lib = _load()
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    nb, ny, nz = vol.shape
    if g_nx is None:
        g_x0, g_nx, x_shift = 0, nb, int(x_off)
    else:
        g_x0, g_nx, x_shift = int(x_off), int(g_nx), 0
    p_lo, p_hi = (0, nb) if own is None else own
    fines = [np.ascontiguousarray(a, dtype=np.float32) for a in (xvol, yvol, zvol)]
    n = (g_nx, ny, nz)
    for a, f in enumerate(fines):
        want = tuple((n[b] - 1) * (s + 1) + 1 if b == a else n[b] for b in range(3))
        assert f.shape == want, f"fine volume {a}: shape {f.shape}, expected {want}"
    nv, nt = C.c_int64(0), C.c_int64(0)
    args = (vol.ctypes.data, nb, ny, nz, float(iso), g_x0, g_nx, p_lo, p_hi, x_shift, int(v_base), int(s),
            *[f.ctypes.data for f in fines])
    rc = lib.mc_oracle_ss(*args, None, None, None, C.byref(nv), C.byref(nt))
    assert rc == 0, f"mc_oracle_ss: error {rc}"
    verts = np.empty((nv.value, 3), np.float32)
    normals = np.empty((nv.value, 3), np.float32)
    faces = np.empty((nt.value, 3), np.int32)
    rc = lib.mc_oracle_ss(*args, verts.ctypes.data, normals.ctypes.data, faces.ctypes.data, C.byref(nv), C.byref(nt))
    assert rc == 0, f"mc_oracle_ss: error {rc}"
    return verts, faces, normals
