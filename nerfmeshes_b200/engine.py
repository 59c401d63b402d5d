"""Engine: one NmHandle plus the torch-tensor plumbing around it (device memory, streams).

torch is used for allocation and stream identity only; every computation is a call through the C ABI
(nerfmeshes_b200/_lib.py).  CPU tensors go through the *_host entry points (copies inside the library), CUDA
tensors through the device-pointer entry points on torch's current stream.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib as L

NET_KEYS = ("num_layers", "hidden_size", "skip_step", "num_encoding_fn_xyz", "num_encoding_fn_dir",
            "include_input_xyz", "include_input_dir", "log_sampling_xyz", "log_sampling_dir", "use_viewdirs")
NET_DEFAULTS = dict(num_layers=4, hidden_size=128, skip_step=4, num_encoding_fn_xyz=6, num_encoding_fn_dir=4,
                    include_input_xyz=True, include_input_dir=True, log_sampling_xyz=True, log_sampling_dir=True,
                    use_viewdirs=True)   # FlexibleNeRFModel.__init__ defaults, src/nerf/models.py:5-17


def net_desc(**kw) -> L.NmNetDesc:
    d = dict(NET_DEFAULTS)
    d.update({k: v for k, v in kw.items() if k in NET_KEYS})
    return L.NmNetDesc(*[int(d[k]) for k in NET_KEYS])


@dataclass
class RenderSettings:
    num_coarse: int = 64
    num_fine: int = 128
    lindisp: bool = False
    perturb: bool = False
    white_background: bool = False
    noise_std: float = 0.0
    attenuation_threshold: float = 1e-5
    precision: int = L.PREC_EXACT
    act_scale_log2: int = 0

    def to_c(self) -> L.NmRenderCfg:
        return L.NmRenderCfg(int(self.num_coarse), int(self.num_fine), int(bool(self.lindisp)), int(bool(self.perturb)),
                             int(bool(self.white_background)), float(self.noise_std), float(self.attenuation_threshold),
                             int(self.precision), int(self.act_scale_log2))


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _f32c(t, device=None) -> torch.Tensor:
    t = torch.as_tensor(t)
    if device is not None:
        t = t.to(device)
    return t.detach().to(torch.float32).contiguous()


def raster_faces(faces, device) -> torch.Tensor:
    """(F,3) int32 faces on `device` for nm_rasterize_mesh.  A wider index outside int32 would wrap to another vertex in the
    cast, so it is reported here with the message the library gives an index outside [0, V)."""
    f = torch.as_tensor(faces)
    if f.dtype != torch.int32 and f.numel() and (int(f.min()) < -2 ** 31 or int(f.max()) >= 2 ** 31):
        raise L.NmError("mesh raster: a face index lies outside [0, V) (nothing was drawn)")
    return f.to(device, torch.int32).contiguous().reshape(-1, 3)


class Engine:
    """Owns one library handle on one CUDA device."""

    # the default of render_rays / render_image's skip_empty outside training (BaseModel.build_occupancy_grid sets it)
    skip_empty = False

    def __init__(self, coarse: dict, fine: Optional[dict], settings: RenderSettings, device: int = 0):
        self.lib = L.load()
        if not torch.cuda.is_available():
            raise L.NmError("nerfmeshes_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.device = torch.device("cuda", device)
        self.settings = settings
        self.has_fine = fine is not None
        self._h = C.c_void_p()
        dc = net_desc(**coarse)
        df = net_desc(**fine) if fine is not None else None
        cfg = settings.to_c()
        self._occupancy = set()         # network slots with a grid built from their current weights
        self._occupancy_stale = set()   # network slots whose grid predates their weights (a weight load): training skipping only
        L.check(self.lib.nm_create(device, C.byref(dc), C.byref(df) if df is not None else None, C.byref(cfg),
                                   C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.nm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ configuration
    def configure(self, **kw):
        for k, v in kw.items():
            if not hasattr(self.settings, k):
                raise AttributeError(k)
            setattr(self.settings, k, v)
        cfg = self.settings.to_c()
        L.check(self.lib.nm_set_render_cfg(self._h, C.byref(cfg)))

    def load_weights(self, which: int, state: Dict[str, torch.Tensor]):
        """state: reference state-dict keys without the model prefix -> tensors.  CUDA tensors on this engine's
        device are packed on the device (nm_load_weights_dev); anything else goes through the host path."""
        items = [(k, v) for k, v in state.items() if "frequency_bands" not in k]
        on_dev = all(v.is_cuda and v.device == self.device for _, v in items)
        names, ptrs, numel, keep = [], [], [], []
        for k, v in items:
            if on_dev:
                a = v.detach().to(torch.float32).contiguous()
                ptrs.append(a.data_ptr())
                numel.append(a.numel())
            else:
                a = np.ascontiguousarray(v.detach().cpu().numpy().astype(np.float32, copy=False))
                ptrs.append(a.ctypes.data)
                numel.append(a.size)
            keep.append(a)
            names.append(k.encode())
        n = len(names)
        if which in self._occupancy:
            self._occupancy.discard(which)
            self._occupancy_stale.add(which)
        args = (self._h, which, n, (C.c_char_p * n)(*names), (C.c_void_p * n)(*ptrs), (C.c_int64 * n)(*numel))
        if on_dev:
            L.check(self.lib.nm_load_weights_dev(*args, self._stream()))
        else:
            L.check(self.lib.nm_load_weights(*args))

    def set_tables(self, coarse_s: Optional[torch.Tensor] = None, fine_u: Optional[torch.Tensor] = None):
        s = None if coarse_s is None else np.ascontiguousarray(coarse_s.detach().cpu().numpy(), dtype=np.float32)
        u = None if fine_u is None else np.ascontiguousarray(fine_u.detach().cpu().numpy(), dtype=np.float32)
        if s is not None:
            assert s.size == self.settings.num_coarse
        if u is not None:
            assert u.size == self.settings.num_fine
        L.check(self.lib.nm_set_tables(self._h, None if s is None else s.ctypes.data, None if u is None else u.ctypes.data))

    def set_tree(self, voxels: torch.Tensor):
        v = np.ascontiguousarray(voxels.detach().cpu().numpy(), dtype=np.float32)
        assert v.ndim == 3 and v.shape[1:] == (2, 3)
        L.check(self.lib.nm_set_tree(self._h, v.ctypes.data, v.shape[0]))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ------------------------------------------------------------------ hot path
    def point_mlp(self, which: int, pts: torch.Tensor, dirs: Optional[torch.Tensor], sigma_only=False) -> torch.Tensor:
        lead = pts.shape[:-1]
        host = not pts.is_cuda
        p = _f32c(pts.reshape(-1, 3))
        d = None if dirs is None else _f32c(dirs.expand_as(pts).reshape(-1, 3))
        M = p.shape[0]
        out = torch.empty((M,) if sigma_only else (M, 4), dtype=torch.float32, device=p.device)
        if M == 0:
            return out.reshape(*lead, *(() if sigma_only else (4,)))
        if host:
            L.check(self.lib.nm_point_mlp_host(self._h, which, _ptr(p), _ptr(d), M, _ptr(out), int(sigma_only)))
        else:
            L.check(self.lib.nm_point_mlp(self._h, which, _ptr(p), _ptr(d), M, _ptr(out), int(sigma_only), self._stream()))
        return out.reshape(*lead, *(() if sigma_only else (4,)))

    def sigma_grad(self, which: int, pts: torch.Tensor, want_sigma=True):
        """d raw sigma / d p of network `which` at pts (...,3) (nm_sigma_grad): (sigma (...) or None, grad (...,3)) device
        tensors.  The network's analytic density gradient in the handle's precision, independent of batch composition."""
        lead = pts.shape[:-1]
        p = _f32c(pts, self.device).reshape(-1, 3)
        M = p.shape[0]
        grad = torch.empty((M, 3), dtype=torch.float32, device=self.device)
        sigma = torch.empty((M,), dtype=torch.float32, device=self.device) if want_sigma else None
        if M:
            L.check(self.lib.nm_sigma_grad(self._h, which, _ptr(p), M, _ptr(sigma), _ptr(grad), self._stream()))
        return (None if sigma is None else sigma.reshape(lead)), grad.reshape(*lead, 3)

    def num_samples(self, buff=False):
        s = self.settings
        return s.num_coarse + (s.num_fine if (self.has_fine and not buff) else 0)

    def out_sizes(self, R, S):
        return dict(rgb=(R, 3), depth=(R,), depth_raw=(R,), acc=(R,), disp=(R,), weights=(R, S), mask_weights=(R, S),
                    t_vals=(R, S), coarse_rgb=(R, 3), coarse_acc=(R,), coarse_disp=(R,),
                    coarse_weights=(R, self.settings.num_coarse))

    def _alloc_out(self, R, S, device, want, pin=False, into=None):
        """Output tensors + the NmRenderOut pointer block.  `into`: caller-owned contiguous fp32 tensors (e.g. views of
        one gather buffer) used instead of fresh allocations."""
        sizes = self.out_sizes(R, S)
        outs = {}
        for k in want:
            if into is not None and k in into:
                t = into[k]
                assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == int(np.prod(sizes[k])) and t.device == device
                outs[k] = t
                continue
            t = torch.empty(sizes[k], dtype=torch.float32, device=device)
            if pin and device.type == "cpu":
                t = t.pin_memory()
            outs[k] = t
        block = L.NmRenderOut(*[(outs[k].data_ptr() if k in outs else None) for k in L.OUT_FIELDS])
        return outs, block

    DEFAULT_OUT = ("rgb", "depth", "depth_raw", "acc", "disp", "weights", "mask_weights")

    def render_rays(self, origins, dirs, near, far, *, training=False, buff=False, seed=0, want=None,
                    teacher_t: Optional[torch.Tensor] = None, out=None, skip_empty=None,
                    train_skip=False) -> Dict[str, torch.Tensor]:
        """NeRFModel.forward / BuFFModel.forward on a ray batch.  origins (3,), (1,3) or (R,3); dirs (R,3);
        near/far python floats / 0-dim tensors, or (R,) tensors (CUDA path only).  skip_empty: send only the samples the
        occupancy grids mark through the networks (NM_FLAG_SKIP_EMPTY, DESIGN 4.15); None = `self.skip_empty` outside
        training.  train_skip: the same in a training render (NM_FLAG_SKIP_EMPTY_TRAIN), on grids that may be stale."""
        want = tuple(want or self.DEFAULT_OUT)
        dirs_t = torch.as_tensor(dirs)
        host = not dirs_t.is_cuda
        dev = dirs_t.device if not host else torch.device("cpu")
        d = _f32c(dirs_t)
        R = d.shape[0]
        o = _f32c(origins, d.device)
        if o.numel() == 3:
            o = o.reshape(3)
            o_stride = 0
        else:
            assert o.shape == (R, 3), "origins must be (3,), (1,3) or (R,3)"
            o_stride = 3
        flags = self._flags(training, buff, skip_empty, train_skip)
        S = self.num_samples(buff)
        per_ray = isinstance(near, torch.Tensor) and near.dim() > 0 and near.shape[0] == R and near.numel() == R and R > 1
        nf = (C.c_float * 2)(0.0, 0.0)
        near_d = far_d = None
        if per_ray:
            if host:
                raise L.NmError("per-ray near/far needs CUDA tensors")
            near_d, far_d = _f32c(near, d.device), _f32c(far, d.device)
        else:
            nf = (C.c_float * 2)(float(near), float(far))
        if teacher_t is not None:
            flags |= L.FLAG_TEACHER_T
            want = tuple(k for k in want if k != "t_vals")
        outs, block = self._alloc_out(R, S, dev, want, into=out)
        if teacher_t is not None:
            tt = _f32c(teacher_t, d.device)
            assert tt.shape == (R, S) and not host
            block.t_vals = tt.data_ptr()
        if R == 0:
            return outs
        if host:
            L.check(self.lib.nm_query_host(self._h, _ptr(o), o_stride, _ptr(d), R, nf, flags, seed, C.byref(block)))
        else:
            L.check(self.lib.nm_render_rays(self._h, _ptr(o), o_stride, _ptr(d), R, None if per_ray else nf, _ptr(near_d),
                                            _ptr(far_d), flags, seed, C.byref(block), self._stream()))
        return outs

    # ------------------------------------------------------------------ training (SURVEY §8f-1)
    def _ray_args(self, origins, dirs, near, far):
        d = _f32c(torch.as_tensor(dirs))
        if not d.is_cuda:
            raise L.NmError("the backward pass takes CUDA tensors")
        R = d.shape[0]
        o = _f32c(origins, d.device)
        if o.numel() == 3:
            o, o_stride = o.reshape(3), 0
        else:
            assert o.shape == (R, 3), "origins must be (3,), (1,3) or (R,3)"
            o_stride = 3
        per_ray = isinstance(near, torch.Tensor) and near.dim() > 0 and near.numel() == R and R > 1
        if per_ray:
            return o, o_stride, d, R, None, _f32c(near, d.device), _f32c(far, d.device)
        return o, o_stride, d, R, (C.c_float * 2)(float(near), float(far)), None, None

    def zero_grad(self):
        L.check(self.lib.nm_zero_grad(self._h, self._stream()))

    def backward_rays(self, origins, dirs, near, far, d_rgb, d_coarse_rgb=None, *, training=True, buff=False, seed=0,
                      train_skip=False):
        """Accumulate dL/dtheta given dL/d rgb_map of the main (and optionally the coarse) bundle; the forward is
        re-run inside with the same flags and seed (same samples, same noise).  train_skip: empty-space skipping on the
        current grids (NM_FLAG_SKIP_EMPTY_TRAIN); the forward being differentiated must have used the same grids."""
        o, o_stride, d, R, nf, near_d, far_d = self._ray_args(origins, dirs, near, far)
        g = None if d_rgb is None else _f32c(d_rgb, d.device)
        gc = None if d_coarse_rgb is None else _f32c(d_coarse_rgb, d.device)
        assert (g is None or g.shape == (R, 3)) and (gc is None or gc.shape == (R, 3))
        flags = self._flags(training, buff, None, train_skip)
        if R:
            L.check(self.lib.nm_backward_rays(self._h, _ptr(o), o_stride, _ptr(d), R, nf, _ptr(near_d), _ptr(far_d), flags,
                                              seed, _ptr(g), _ptr(gc), self._stream()))

    def loss_backward(self, origins, dirs, near, far, target_rgb, *, training=True, buff=False, seed=0, train_skip=False):
        """The reference's training loss and its backward in one call: returns a (2,) device tensor
        [mse(coarse-or-only rgb_map, target), mse(fine rgb_map, target)] (src/models/model_nerf.py:118-126).
        train_skip: empty-space skipping on the current grids (NM_FLAG_SKIP_EMPTY_TRAIN, DESIGN 4.15)."""
        o, o_stride, d, R, nf, near_d, far_d = self._ray_args(origins, dirs, near, far)
        tgt = _f32c(target_rgb, d.device)
        assert tgt.shape == (R, 3)
        loss = torch.zeros(2, dtype=torch.float32, device=d.device)
        flags = self._flags(training, buff, None, train_skip)
        if R:
            L.check(self.lib.nm_loss_backward(self._h, _ptr(o), o_stride, _ptr(d), R, nf, _ptr(near_d), _ptr(far_d), flags,
                                              seed, _ptr(tgt), _ptr(loss), self._stream()))
        return loss

    def get_grad(self, which: int, name: str, like: torch.Tensor) -> torch.Tensor:
        out = torch.empty(like.shape, dtype=torch.float32, device=self.device)
        L.check(self.lib.nm_get_grad(self._h, which, name.encode(), _ptr(out), out.numel(), self._stream()))
        return out

    # ------------------------------------------------------------------ BuFF tree maintenance (SURVEY §8f-4)
    def _flags(self, training, buff, skip_empty=None, train_skip=False):
        """render-call flags; `voxel_random` mirrors cfg.tree.use_random_sampling (src/nerf/tree.py:280).  skip_empty None
        follows `self.skip_empty` outside training; an explicit True is passed on as asked (the library rejects it in
        training).  train_skip: NM_FLAG_SKIP_EMPTY_TRAIN, on fresh or stale grids (the library rejects it outside
        training)."""
        skip = (self.skip_empty and not training) if skip_empty is None else bool(skip_empty)
        nets = (L.NET_COARSE,) if buff or not self.has_fine else (L.NET_COARSE, L.NET_FINE)
        if skip:
            for which in nets:
                if which not in self._occupancy:
                    raise L.NmError(f"empty-space skipping: network {which} has no occupancy grid for its current weights "
                                    "(the weights changed after build_occupancy_grid, or none was built); call "
                                    "build_occupancy_grid again")
        if train_skip:
            for which in nets:
                if which not in self._occupancy and which not in self._occupancy_stale:
                    raise L.NmError(f"training-time empty-space skipping: network {which} has no occupancy grid; call "
                                    "enable_training_skip (or build_occupancy_grid) first")
        return ((L.FLAG_TRAINING if training else 0) | (L.FLAG_BUFF if buff else 0) |
                (L.FLAG_RANDOM_VOXELS if buff and getattr(self, "voxel_random", False) else 0) |
                (L.FLAG_SKIP_EMPTY if skip else 0) | (L.FLAG_SKIP_EMPTY_TRAIN if train_skip else 0))

    # ------------------------------------------------------------------ empty-space skipping (DESIGN 4.15)
    @staticmethod
    def occupancy_words(res: int) -> int:
        return (res ** 3 + 31) // 32

    @staticmethod
    def _box(box):
        b = np.ascontiguousarray(np.asarray(box, dtype=np.float32).reshape(-1))
        if b.size != 6:
            raise ValueError("an occupancy box is (lo_x, lo_y, lo_z, hi_x, hi_y, hi_z)")
        return b

    def build_occupancy(self, which: int, box, res: int = 128, threshold: float = 0.0, dilate: int = 0) -> torch.Tensor:
        """Occupancy grid of network `which` from its own density (nm_build_occupancy): res^3 cells over box (lo3, hi3); a
        cell is occupied when the max raw sigma of its 8 lattice corners is > threshold (or NaN), dilated by `dilate` cells.
        Returns the bits, ceil(res^3 / 32) words (int32 device tensor, bit (i*res + j)*res + k)."""
        b = self._box(box)
        bits = torch.empty(self.occupancy_words(res), dtype=torch.int32, device=self.device)
        self._occupancy.discard(which)
        self._occupancy_stale.discard(which)
        L.check(self.lib.nm_build_occupancy(self._h, which, b.ctypes.data, int(res), float(threshold), int(dilate), _ptr(bits),
                                            self._stream()))
        self._occupancy.add(which)
        return bits

    def set_occupancy(self, which: int, box, res: int, bits: Optional[torch.Tensor]):
        """Install caller bits (layout of build_occupancy) as network `which`'s grid; None removes it."""
        self._occupancy.discard(which)
        self._occupancy_stale.discard(which)
        if bits is None:
            L.check(self.lib.nm_set_occupancy(self._h, which, None, 0, None))
            return
        b = self._box(box)
        w = bits.to(self.device).contiguous()
        assert w.dtype in (torch.int32, torch.uint32) and w.numel() == self.occupancy_words(res), (w.dtype, w.numel())
        torch.cuda.current_stream(self.device).synchronize()
        L.check(self.lib.nm_set_occupancy(self._h, which, b.ctypes.data, int(res), _ptr(w)))
        self._occupancy.add(which)

    def occupancy_query(self, which: int, pts: torch.Tensor) -> torch.Tensor:
        """bool (...) per point (...,3): True where a skipping render evaluates the point under network `which`'s grid."""
        lead = pts.shape[:-1]
        p = _f32c(pts, self.device).reshape(-1, 3)
        out = torch.empty(p.shape[0], dtype=torch.uint8, device=self.device)
        L.check(self.lib.nm_occupancy_query(self._h, which, _ptr(p), p.shape[0], _ptr(out), self._stream()))
        return out.bool().reshape(lead)

    def skip_stats(self) -> Dict[str, int]:
        """Samples seen / evaluated per pass by skipping renders and skipping training passes since the last call
        (nm_skip_stats); resets them."""
        out = (C.c_int64 * 4)()
        L.check(self.lib.nm_skip_stats(self._h, out))
        return dict(coarse_seen=out[0], coarse_evaluated=out[1], fine_seen=out[2], fine_evaluated=out[3])

    def ray_voxel_indices(self, origins, dirs, near, far, want_z=False, seed=0):
        """(R,S) int32 voxel index of every AABB sample (-1 on rays without a hit) [, (R,S) sample distances].  With
        `voxel_random` set, `seed` must be the render call's seed for the indices to describe that call's samples."""
        o, o_stride, d, R, nf, near_d, far_d = self._ray_args(origins, dirs, near, far)
        if nf is None:
            raise L.NmError("the BuFF sampler takes scalar near/far")
        S = self.settings.num_coarse
        idx = torch.empty((R, S), dtype=torch.int32, device=d.device)
        z = torch.empty((R, S), dtype=torch.float32, device=d.device) if want_z else None
        if R:
            L.check(self.lib.nm_ray_voxel_indices_ex(self._h, _ptr(o), o_stride, _ptr(d), R, nf, self._flags(False, True) & L.FLAG_RANDOM_VOXELS,
                                                     int(seed), _ptr(z), _ptr(idx), self._stream()))
        return (idx, z) if want_z else idx

    def tree_integrate(self, idx, weights, mask_weights, memm, counter):
        """TreeSampling.ray_batch_integration on the device: updates `memm` (V,) in place."""
        idx = idx.to(torch.int32).contiguous()
        w, mw = _f32c(weights, idx.device), _f32c(mask_weights, idx.device)
        assert memm.is_cuda and memm.dtype == torch.float32 and memm.is_contiguous() and w.numel() == idx.numel() == mw.numel()
        if idx.numel() == 0:                # an empty batch (no storage to point at) changes nothing
            return
        L.check(self.lib.nm_tree_integrate(self._h, _ptr(idx), _ptr(w), _ptr(mw), idx.numel(), _ptr(memm), memm.numel(),
                                           int(counter), self._stream()))

    def debug_gemm(self, a, b, *, n_passes=3, out=None):
        """Test hook (nm_debug_gemm): D += a^T b on the backward pass's weight-gradient GEMM.  a: (K,M), b: (K,N);
        D: `out` (M,N), or a new zero tensor."""
        a, b = _f32c(a, self.device), _f32c(b, self.device)
        (K, M), N = a.shape, b.shape[1]
        assert b.shape[0] == K, (a.shape, b.shape)
        d = out if out is not None else torch.zeros((M, N), dtype=torch.float32, device=self.device)
        L.check(self.lib.nm_debug_gemm(self._h, _ptr(a), _ptr(b), M, N, K, n_passes, _ptr(d), self._stream()))
        return d

    def debug_mlp_backward(self, which: int, pts, dirs, dout):
        """Test hook (nm_debug_mlp_backward): accumulate the gradients of network `which` for per-point adjoints
        dout (M,4) = [d rgb logits, d raw sigma] at points pts (M,3) with view directions dirs (M,3) or None."""
        p = _f32c(pts, self.device).reshape(-1, 3)
        d = None if dirs is None else _f32c(dirs, self.device).reshape(-1, 3)
        g = _f32c(dout, self.device)
        M = p.shape[0]
        assert g.shape == (M, 4) and (d is None or d.shape == (M, 3)), (p.shape, g.shape)
        L.check(self.lib.nm_debug_mlp_backward(self._h, which, _ptr(p), _ptr(d), M, _ptr(g), self._stream()))

    def debug_composite_backward(self, raw, t, dirs, d_rgb, *, noise_std=0.0, seed=0, white_bg=False):
        """Test hook (nm_debug_composite_backward): the training compositor adjoint alone.  raw (R,S,4) = (sigmoid rgb,
        raw sigma), t (R,S), dirs (R,3), d_rgb (R,3) = dL/d rgb_map; `seed` is the pass's salted noise stream.  Returns
        dout (R,S,4) = [dL/d rgb logits, dL/d raw sigma]."""
        q, tt = _f32c(raw, self.device), _f32c(t, self.device)
        d, g = _f32c(dirs, self.device), _f32c(d_rgb, self.device)
        R, S = tt.shape
        assert q.shape == (R, S, 4) and d.shape == (R, 3) and g.shape == (R, 3), (q.shape, tt.shape, d.shape, g.shape)
        out = torch.empty((R, S, 4), dtype=torch.float32, device=self.device)
        L.check(self.lib.nm_debug_composite_backward(self._h, _ptr(q), _ptr(tt), _ptr(d), _ptr(g), R, S, float(noise_std),
                                                     int(seed) % 2 ** 64, int(white_bg), _ptr(out), self._stream()))
        return out

    COMPOSITE_OUT = ("rgb", "depth", "depth_raw", "acc", "disp", "weights", "mask_weights")

    def debug_composite(self, raw, t, dirs, *, noise_std=0.0, seed=0, white_bg=False, training=False, thr=1e-5, want=None):
        """Test hook (nm_debug_composite): the inference compositor alone, as a render pass calls it.  raw (R,S,4) =
        (sigmoid rgb, raw sigma), t (R,S), dirs (R,3); `seed` is the pass's salted noise stream, `thr` the mask_weights
        threshold.  Returns the maps of `want` (default all seven: rgb, depth, depth_raw, acc, disp, weights, mask_weights)."""
        q, tt, d = _f32c(raw, self.device), _f32c(t, self.device), _f32c(dirs, self.device)
        R, S = tt.shape
        assert q.shape == (R, S, 4) and d.shape == (R, 3), (q.shape, tt.shape, d.shape)
        want = tuple(want or self.COMPOSITE_OUT)
        assert set(want) <= set(self.COMPOSITE_OUT), want
        outs, block = self._alloc_out(R, S, self.device, want)
        L.check(self.lib.nm_debug_composite(self._h, _ptr(q), _ptr(tt), _ptr(d), R, S, float(noise_std), int(seed) % 2 ** 64,
                                            int(bool(white_bg)), int(bool(training)), float(thr), C.byref(block),
                                            self._stream()))
        return outs

    def debug_sample_pdf(self, t_c, w_c, u=None, *, Nf=None, perturb=False, seed=0):
        """Test hook (nm_debug_sample_pdf): the inverse-CDF resampler alone.  t_c (R,Nc) ascending coarse depths, w_c (R,Nc)
        coarse weights; u (Nf,) the deterministic positions, or None with `perturb` (drawn from the salted stream `seed`).
        Returns (R, Nc+Nf): the coarse depths and the new samples, merged in ascending order."""
        tc, wc = _f32c(t_c, self.device), _f32c(w_c, self.device)
        uu = None if u is None else _f32c(u, self.device).reshape(-1)
        Nf = int(uu.numel() if Nf is None else Nf)
        R, Nc = tc.shape
        assert wc.shape == (R, Nc) and (uu is None or uu.numel() == Nf), (tc.shape, wc.shape, None if uu is None else uu.shape)
        out = torch.empty((R, Nc + Nf), dtype=torch.float32, device=self.device)
        L.check(self.lib.nm_debug_sample_pdf(self._h, _ptr(tc), _ptr(wc), _ptr(uu), R, Nc, Nf, int(bool(perturb)),
                                             int(seed) % 2 ** 64, _ptr(out), self._stream()))
        return out

    def render_image(self, pose, H, W, focal, near, far, *, ndc=False, rows=None, training=False, buff=False, seed=0,
                     want=None, to_host=False, host_out=None, out=None, skip_empty=None) -> Dict[str, torch.Tensor]:
        """Rays generated on the device from a 3x4 / 4x4 camera-to-world pose (get_ray_bundle [+ ndc_rays]).  skip_empty:
        as in render_rays."""
        want = tuple(want or ("rgb", "depth", "acc", "disp"))
        row0, row1 = rows if rows is not None else (0, H)
        R = (row1 - row0) * W
        p = np.ascontiguousarray(torch.as_tensor(pose).detach().cpu().numpy()[:3, :4], dtype=np.float32)
        nf = (C.c_float * 2)(float(near), float(far))
        flags = self._flags(training, buff, skip_empty)
        S = self.num_samples(buff)
        if to_host:
            if host_out is not None:
                outs = host_out
                block = L.NmRenderOut(*[(outs[k].data_ptr() if k in outs else None) for k in L.OUT_FIELDS])
            else:
                outs, block = self._alloc_out(R, S, torch.device("cpu"), want, pin=True)
            L.check(self.lib.nm_render_image_host(self._h, p.ctypes.data, H, W, float(focal), int(ndc), row0, row1, nf,
                                                  flags, seed, C.byref(block)))
        else:
            outs, block = self._alloc_out(R, S, self.device, want, into=out)
            L.check(self.lib.nm_render_image(self._h, p.ctypes.data, H, W, float(focal), int(ndc), row0, row1, nf, flags,
                                             seed, C.byref(block), self._stream()))
        return outs

    def ray_bundle(self, pose, H, W, focal, *, ndc=False, ndc_near=1.0, rows=None):
        row0, row1 = rows if rows is not None else (0, H)
        p = np.ascontiguousarray(torch.as_tensor(pose).detach().cpu().numpy()[:3, :4], dtype=np.float32)
        dirs = torch.empty((row1 - row0, W, 3), dtype=torch.float32, device=self.device)
        origins = torch.empty_like(dirs) if ndc else None
        L.check(self.lib.nm_ray_bundle(self._h, p.ctypes.data, H, W, float(focal), int(ndc), float(ndc_near), row0, row1,
                                       _ptr(origins), _ptr(dirs), self._stream()))
        if not ndc:
            origins = torch.from_numpy(p[:, 3].copy()).to(self.device)
        return origins, dirs

    def ndc_rays(self, H, W, focal, near, rays_o, rays_d):
        """ndc_rays(H, W, focal, near, rays_o, rays_d) on caller-supplied rays (src/nerf/nerf_helpers.py:280-307)."""
        d = _f32c(rays_d, self.device)
        shape = d.shape
        d = d.reshape(-1, 3)
        o = _f32c(rays_o, self.device)
        if o.numel() == 3:
            o, o_stride = o.reshape(3), 0
        else:
            o = o.expand(shape).reshape(-1, 3).contiguous()
            o_stride = 3
        oo, dd = torch.empty_like(d), torch.empty_like(d)
        L.check(self.lib.nm_ndc_rays(self._h, int(H), int(W), float(focal), float(near), _ptr(o), o_stride, _ptr(d), d.shape[0],
                                     _ptr(oo), _ptr(dd), self._stream()))
        return oo.reshape(shape), dd.reshape(shape)

    def check_flags(self):
        """Synchronise the current stream and raise if a kernel of this handle flagged an error (AABB hit-list overflow,
        tensor-core pipeline watchdog)."""
        L.check(self.lib.nm_check_flags(self._h, self._stream()))

    def grid_sigma(self, lins, x0=0, x1=None, with_rgb=False, out=None):
        """extract_radiance for planes [x0,x1): lins = three 1-D fp32 tensors (torch.linspace values).  `out`: optional
        contiguous (x1-x0, n1, n2) device tensor to write the densities into (e.g. the owned planes of a halo buffer)."""
        ls = [np.ascontiguousarray(torch.as_tensor(t).detach().cpu().numpy(), dtype=np.float32) for t in lins]
        n0, n1, n2 = (a.size for a in ls)
        x1 = n0 if x1 is None else x1
        if out is not None:
            assert out.shape == (x1 - x0, n1, n2) and out.is_contiguous() and out.dtype == torch.float32 and not with_rgb
        sigma = out if out is not None else torch.empty((x1 - x0, n1, n2), dtype=torch.float32, device=self.device)
        rgb = torch.empty((x1 - x0, n1, n2, 3), dtype=torch.float32, device=self.device) if with_rgb else None
        L.check(self.lib.nm_grid_sigma(self._h, ls[0].ctypes.data, ls[1].ctypes.data, ls[2].ctypes.data, n0, n1, n2, x0,
                                       x1, _ptr(sigma), _ptr(rgb), self._stream()))
        return (sigma, rgb) if with_rgb else sigma

    def volume_stats(self, vol: torch.Tensor):
        v = _f32c(vol, self.device)
        out = (C.c_float * 3)()
        torch.cuda.current_stream(self.device).synchronize()
        L.check(self.lib.nm_volume_stats(self._h, _ptr(v), v.numel(), out))
        return float(out[0]), float(out[1]), float(out[2])

    def volume_stats_pass(self, vol: torch.Tensor, pass_no: int, out: torch.Tensor, mean: Optional[torch.Tensor] = None):
        """Asynchronous half of volume_stats for sharded volumes (nm_volume_stats_dev): out = 4 doubles on the device."""
        assert out.dtype == torch.float64 and out.numel() >= 4 and out.is_cuda and vol.is_contiguous() and vol.dtype == torch.float32
        assert mean is None or (mean.dtype == torch.float64 and mean.is_cuda)
        L.check(self.lib.nm_volume_stats_dev(self._h, _ptr(vol), vol.numel(), int(pass_no), _ptr(mean), _ptr(out), self._stream()))

    def _mesh_out(self, nv, nt, out):
        """(verts (nv,3), normals (nv,3), faces (nt,3) int32) of an emit step: fresh tensors, or the caller's `out` triple
        checked for layout and capacity."""
        if out is None:
            return (torch.empty((nv, 3), dtype=torch.float32, device=self.device),
                    torch.empty((nv, 3), dtype=torch.float32, device=self.device),
                    torch.empty((nt, 3), dtype=torch.int32, device=self.device))
        verts, normals, faces = out
        assert verts.is_contiguous() and normals.is_contiguous() and faces.is_contiguous() and faces.dtype == torch.int32
        assert verts.shape[0] >= nv and faces.shape[0] >= nt
        return verts, normals, faces

    def marching_cubes(self, vol: torch.Tensor, iso: float, x_off: int = 0):
        """skimage.measure.marching_cubes(vol, iso) on the device: (verts (V,3), faces (F,3) int32, normals (V,3)); x_off is
        added to the axis-0 coordinates of the vertices."""
        v = _f32c(vol, self.device)
        nx, ny, nz = v.shape
        counts = (C.c_int64 * 2)()
        L.check(self.lib.nm_marching_cubes_count(self._h, _ptr(v), nx, ny, nz, float(iso), counts, self._stream()))
        nv = int(counts[0])
        verts, normals, faces = self._mesh_out(nv, int(counts[1]), None)
        if nv > 0:
            L.check(self.lib.nm_marching_cubes_emit(self._h, _ptr(v), nx, ny, nz, float(iso), float(int(x_off)), _ptr(verts),
                                                    _ptr(normals), _ptr(faces), self._stream()))
        return verts, faces, normals

    def mc_count(self, vol, iso, g_x0, g_nx, p_lo, p_hi):
        """Count step of one shard (see nm_mc_count): -> (n_vertices owned, n_triangles).  Synchronises."""
        nb, ny, nz = vol.shape
        counts = (C.c_int64 * 2)()
        L.check(self.lib.nm_mc_count(self._h, _ptr(vol), nb, ny, nz, float(iso), int(g_x0), int(g_nx), int(p_lo), int(p_hi),
                                     counts, self._stream()))
        return int(counts[0]), int(counts[1])

    def mc_emit(self, vol, iso, g_x0, g_nx, p_lo, p_hi, nv, nt, v_base, out=None):
        """Emit step: vertices / normals / faces of the shard, faces offset by v_base.  `out`: optional (verts, normals,
        faces) device tensors to write into (e.g. slices of a gather buffer)."""
        nb, ny, nz = vol.shape
        verts, normals, faces = self._mesh_out(nv, nt, out)
        if nv > 0:
            L.check(self.lib.nm_mc_emit(self._h, _ptr(vol), nb, ny, nz, float(iso), int(g_x0), int(g_nx), int(p_lo), int(p_hi),
                                        int(v_base), _ptr(verts), _ptr(normals), _ptr(faces), self._stream()))
        return verts, faces, normals

    def mc_emit_ss(self, vol, iso, g_x0, g_nx, p_lo, p_hi, nv, nt, v_base, s, lins, fines, out=None):
        """Super-sampled emit step (nm_mc_emit_ss): mc_emit's arrays, with every edge vertex re-placed from `s` network
        samples along its edge.  lins: the coarse tables (g_nx, ny, nz entries), fines: the fine tables
        ((n-1)(s+1)+1 entries; mesh.super_sampling_tables)."""
        nb, ny, nz = vol.shape
        verts, normals, faces = self._mesh_out(nv, nt, out)
        want = (g_nx, ny, nz)
        tabs = [np.ascontiguousarray(torch.as_tensor(t).detach().cpu().numpy(), dtype=np.float32) for t in (*lins, *fines)]
        for a in range(3):                   # the library cannot see the host tables' lengths
            if 0 <= s and (tabs[a].size != want[a] or tabs[3 + a].size != (want[a] - 1) * (s + 1) + 1):
                raise L.NmError(f"super-sampling tables of axis {a}: {tabs[a].size} / {tabs[3 + a].size} entries, expected "
                                f"{want[a]} / {(want[a] - 1) * (s + 1) + 1}")
        L.check(self.lib.nm_mc_emit_ss(self._h, _ptr(vol), nb, ny, nz, float(iso), int(g_x0), int(g_nx), int(p_lo), int(p_hi),
                                       int(v_base), int(s), *[t.ctypes.data for t in tabs], _ptr(verts), _ptr(normals),
                                       _ptr(faces), self._stream()))
        return verts, faces, normals

    # ------------------------------------------------------------------ chamfer evaluation (DESIGN 4.7)
    def mesh_sample(self, verts, faces, n: int, seed: int, want_faces=False):
        """sample_points_from_meshes for one mesh (nm_mesh_sample): (n,3) area-weighted surface points [, (n,) int32 face
        index].  Synchronises and raises if the mesh has a face index outside [0,V) or no area."""
        v = _f32c(verts, self.device).reshape(-1, 3)
        f = torch.as_tensor(faces).to(self.device, torch.int32).contiguous().reshape(-1, 3)
        pts = torch.empty((n, 3), dtype=torch.float32, device=self.device)
        fi = torch.empty((n,), dtype=torch.int32, device=self.device) if want_faces else None
        L.check(self.lib.nm_mesh_sample(self._h, _ptr(v), v.shape[0], _ptr(f), f.shape[0], int(n), int(seed) & (2 ** 64 - 1),
                                        _ptr(pts), _ptr(fi), self._stream()))
        self.check_flags()
        return (pts, fi) if want_faces else pts

    def _nn(self, fn, q, p):
        q, p = _f32c(q, self.device).reshape(-1, 3), _f32c(p, self.device).reshape(-1, 3)
        d = torch.empty((q.shape[0],), dtype=torch.float32, device=self.device)
        i = torch.empty((q.shape[0],), dtype=torch.int32, device=self.device)
        L.check(fn(self._h, _ptr(q), q.shape[0], _ptr(p), p.shape[0], _ptr(d), _ptr(i), self._stream()))
        return d, i

    def nearest(self, q, p):
        """Exact nearest neighbour (nm_nearest): for each query of q (N,3), the squared distance to the nearest point of
        p (M,3) and its index (lowest on ties): ((N,) fp32, (N,) int32)."""
        return self._nn(self.lib.nm_nearest, q, p)

    def debug_nearest_brute(self, q, p):
        """Test hook (nm_debug_nearest_brute): nearest() by brute force, the same distance function."""
        return self._nn(self.lib.nm_debug_nearest_brute, q, p)

    def chamfer(self, x, y) -> torch.Tensor:
        """chamfer_distance without weights or normals (nm_chamfer): a (2,) float64 device tensor
        [mean_i d2(x_i, Y), mean_j d2(y_j, X)]; the loss is their sum."""
        x, y = _f32c(x, self.device).reshape(-1, 3), _f32c(y, self.device).reshape(-1, 3)
        means = torch.empty((2,), dtype=torch.float64, device=self.device)
        L.check(self.lib.nm_chamfer(self._h, _ptr(x), x.shape[0], _ptr(y), y.shape[0], _ptr(means), self._stream()))
        return means

    # ------------------------------------------------------------------ small-component removal (DESIGN 4.9)
    def mesh_components(self, verts, normals, faces, min_faces: int, want_labels=False):
        """Keep the components of the mesh with >= min_faces faces (nm_mesh_components): (verts (v,3), normals (v,3),
        faces (f,3) int32, counts, labels) with v / f the kept sizes, rows in their original order, faces re-indexed;
        counts = (kept vertices, kept faces, components with >= 1 face, kept components); labels (V,) int32 = the component
        id (smallest vertex index) of every input vertex when want_labels, else None.  Synchronises, and raises if a face
        index lies outside [0, V)."""
        v = _f32c(verts, self.device).reshape(-1, 3)
        n = _f32c(normals, self.device).reshape(-1, 3)
        f = torch.as_tensor(faces).to(self.device, torch.int32).contiguous().reshape(-1, 3)
        V, F = v.shape[0], f.shape[0]
        if n.shape[0] != V:
            raise L.NmError(f"mesh components: {n.shape[0]} normals for {V} vertices")
        vo, no = torch.empty_like(v), torch.empty_like(n)
        fo = torch.empty_like(f)
        labels = torch.empty((V,), dtype=torch.int32, device=self.device) if want_labels else None
        counts = (C.c_int64 * 4)()
        p = lambda t: _ptr(t) if t is not None and t.numel() else None
        L.check(self.lib.nm_mesh_components(self._h, p(v), p(n), V, p(f), F, int(min_faces), p(vo), p(no), p(fo), p(labels),
                                            counts, self._stream()))
        self.check_flags()
        kv, kf = int(counts[0]), int(counts[1])
        return vo[:kv], no[:kv], fo[:kf], (kv, kf, int(counts[2]), int(counts[3])), labels

    # ------------------------------------------------------------------ quadric-error decimation (DESIGN 4.11)
    def mesh_decimate(self, verts, normals, faces, target_faces: int, want_source=False):
        """Collapse edges of the mesh until at most target_faces faces remain or no collapse is legal (nm_mesh_decimate):
        (verts (v,3), normals (v,3), faces (f,3) int32, counts, source) with the surviving vertices in input order, faces
        in input order re-indexed; counts = (v, f, rounds, collapses); source (v,) int32 = the input row of every output
        vertex when want_source, else None.  Synchronises, and raises if a face index lies outside [0, V)."""
        v = _f32c(verts, self.device).reshape(-1, 3)
        n = _f32c(normals, self.device).reshape(-1, 3)
        f = torch.as_tensor(faces).to(self.device, torch.int32).contiguous().reshape(-1, 3)
        V, F = v.shape[0], f.shape[0]
        if n.shape[0] != V:
            raise L.NmError(f"mesh decimate: {n.shape[0]} normals for {V} vertices")
        vo, no = torch.empty_like(v), torch.empty_like(n)
        fo = torch.empty_like(f)
        source = torch.empty((V,), dtype=torch.int32, device=self.device) if want_source else None
        counts = (C.c_int64 * 4)()
        p = lambda t: _ptr(t) if t is not None and t.numel() else None
        L.check(self.lib.nm_mesh_decimate(self._h, p(v), p(n), V, p(f), F, int(target_faces), p(vo), p(no), p(fo), p(source),
                                          counts, self._stream()))
        self.check_flags()
        kv, kf = int(counts[0]), int(counts[1])
        return vo[:kv], no[:kv], fo[:kf], (kv, kf, int(counts[2]), int(counts[3])), (source[:kv] if want_source else None)

    # ------------------------------------------------------------------ texture bake (DESIGN 4.12)
    @staticmethod
    def texture_layout(F: int, N: int):
        """(Q cells per row, rows, W, H) of the texture atlas of F faces at N texels per triangle leg (nm_texture_layout).
        Raises for N outside [2, 64] or an atlas side above 16384."""
        out = (C.c_int64 * 4)()
        L.check(L.load().nm_texture_layout(int(F), int(N), out))
        return tuple(int(x) for x in out)

    def _texture_mesh(self, verts, normals, faces):
        v = _f32c(verts, self.device).reshape(-1, 3)
        n = _f32c(normals, self.device).reshape(-1, 3)
        f = torch.as_tensor(faces).to(self.device, torch.int32).contiguous().reshape(-1, 3)
        if n.shape[0] != v.shape[0]:
            raise L.NmError(f"texture bake: {n.shape[0]} normals for {v.shape[0]} vertices")
        return v, n, f

    def bake_texture(self, verts, normals, faces, N: int, *, mode=0, which=0, flags=0, view_disparity=0.0, near_far=(0.0, 0.0)):
        """One appearance query per texel of the atlas (nm_bake_texture): mode 0 a ray from p + view_disparity*n along -n
        rendered with `flags` and near_far, mode 1 network `which` at (p, -n).  Returns (atlas_u8 (H,W,3) uint8, atlas_f32
        (H,W,3), uv (F,3,2), vertex_rgb (V,3), counts (W, H, queries, unreferenced vertices)) device tensors.  Synchronises,
        and raises if a face index lies outside [0, V)."""
        v, n, f = self._texture_mesh(verts, normals, faces)
        V, F = v.shape[0], f.shape[0]
        _, _, W, H = self.texture_layout(F, N)
        atlas = torch.empty((H, W, 3), dtype=torch.float32, device=self.device)
        u8 = torch.empty((H, W, 3), dtype=torch.uint8, device=self.device)
        uv = torch.empty((F, 3, 2), dtype=torch.float32, device=self.device)
        rgb = torch.empty((V, 3), dtype=torch.float32, device=self.device)
        counts = (C.c_int64 * 4)()
        p = lambda t: _ptr(t) if t.numel() else None
        L.check(self.lib.nm_bake_texture(self._h, p(v), p(n), V, p(f), F, int(N), int(mode), int(which), int(flags),
                                         float(view_disparity), (C.c_float * 2)(*near_far), p(atlas), p(u8), p(uv), p(rgb),
                                         counts, self._stream()))
        self.check_flags()
        return u8, atlas, uv, rgb, tuple(int(c) for c in counts)

    def debug_texture_rays(self, verts, normals, faces, N: int, f0: int, f1: int, *, mode=0, view_disparity=0.0):
        """Test hook (nm_debug_texture_rays): the queries of faces [f0, f1), N(N+1)/2 per face: (origins (mode 0) or points
        (mode 1) (n,3), directions (n,3), atlas pixels (x, y) (n,2) int32)."""
        v, n, f = self._texture_mesh(verts, normals, faces)
        m = (int(f1) - int(f0)) * (N * (N + 1) // 2)
        a = torch.empty((max(m, 0), 3), dtype=torch.float32, device=self.device)
        d, xy = torch.empty_like(a), torch.empty((max(m, 0), 2), dtype=torch.int32, device=self.device)
        p = lambda t: _ptr(t) if t.numel() else None
        L.check(self.lib.nm_debug_texture_rays(self._h, p(v), p(n), v.shape[0], p(f), f.shape[0], int(N), int(mode),
                                               float(view_disparity), int(f0), int(f1), p(a), p(d), p(xy), self._stream()))
        return a, d, xy

    # ------------------------------------------------------------------ mesh raster (DESIGN 4.13)
    def rasterize_mesh(self, verts, faces, pose, H: int, W: int, focal: float, *, colors=None, atlas=None, N: int = 0,
                       z_near: float = 1e-3, background=(0.0, 0.0, 0.0), want=("rgb", "depth", "face")):
        """An image of the world-coordinate mesh verts (V,3) / faces (F,3) through render_image's camera (nm_rasterize_mesh):
        mode 0 with colors (V,3), mode 1 with a floating-point atlas of N texels per leg in nm_bake_texture's layout for these
        F faces (texture_layout(F, N): (H', W', 3) with W', H' its width and height; a uint8 atlas goes through
        mesh.render_mesh, which scales it by 1/255).  Returns ({"rgb": (H,W,3), "depth": (H,W) ray distance, "face": (H,W)
        int32} for the keys in `want`, (covered pixels, faces drawn, faces culled)).  Uncovered pixels hold the background,
        depth 0 and face -1.  Synchronises, and raises if a face index lies outside [0, V) or the atlas does not fit the mesh."""
        v = _f32c(verts, self.device).reshape(-1, 3)
        f = raster_faces(faces, self.device)
        p = np.ascontiguousarray(torch.as_tensor(pose).detach().cpu().numpy()[:3, :4], dtype=np.float32)
        mode = 1 if atlas is not None else 0
        col = None if colors is None else _f32c(colors, self.device).reshape(-1, 3)
        if col is not None and col.shape[0] != v.shape[0]:
            raise L.NmError(f"mesh raster: {col.shape[0]} colours for {v.shape[0]} vertices")
        tex = None
        if atlas is not None:
            a = torch.as_tensor(atlas)
            if not a.dtype.is_floating_point:
                raise L.NmError(f"mesh raster: a {a.dtype} atlas; pass colours in [0, 1] as floats (mesh.render_mesh scales a "
                                "uint8 atlas by 1/255)")
            _, _, aw, ah = self.texture_layout(f.shape[0], N)       # raises for an N the layout rejects
            if f.shape[0] and tuple(a.shape) != (ah, aw, 3):
                raise L.NmError(f"mesh raster: a {tuple(a.shape)} atlas does not fit {f.shape[0]} faces at N = {N}, which need "
                                f"({ah}, {aw}, 3): was it baked for another mesh or another N?")
            tex = _f32c(a, self.device)
        shapes = dict(rgb=((H, W, 3), torch.float32), depth=((H, W), torch.float32), face=((H, W), torch.int32))
        outs = {k: torch.empty(shapes[k][0], dtype=shapes[k][1], device=self.device) for k in want}
        bg = (C.c_float * 3)(*[float(x) for x in background])
        counts = (C.c_int64 * 3)()
        ptr = lambda t: _ptr(t) if t is not None and t.numel() else None
        L.check(self.lib.nm_rasterize_mesh(self._h, ptr(v), v.shape[0], ptr(f), f.shape[0], p.ctypes.data, int(H), int(W),
                                           float(focal), float(z_near), mode, ptr(col), ptr(tex), int(N), bg,
                                           ptr(outs.get("rgb")), ptr(outs.get("depth")), ptr(outs.get("face")), counts,
                                           self._stream()))
        self.check_flags()
        return outs, tuple(int(c) for c in counts)

    # ------------------------------------------------------------------ surface points (DESIGN 4.14)
    def surface_points(self, pose, H: int, W: int, focal: float, depth_raw, acc, rgb, *, min_acc: float = 1.0, step: int = 2,
                       dist_threshold: float = 0.002, min_count: int = 15, out=None):
        """The depth-consistent surface points of one view (nm_surface_points): depth_raw, acc (H*W) and rgb (H*W,3) are
        render_image's outputs for this pose without NDC.  `out`: optional dict of caller-owned contiguous device tensors
        "points", "normals", "colors" (H*W,3) fp32 and "pixel" (H*W,) int32 to write into.  Returns ({"points", "normals",
        "colors", "pixel"}: the first n rows of those buffers, the kept pixels in row-major order, n).  Synchronises."""
        p = np.ascontiguousarray(torch.as_tensor(pose).detach().cpu().numpy()[:3, :4], dtype=np.float32)
        n = int(H) * int(W)
        dr, ac, cl = _f32c(depth_raw, self.device).reshape(-1), _f32c(acc, self.device).reshape(-1), _f32c(rgb, self.device).reshape(-1, 3)
        if not (dr.shape[0] == ac.shape[0] == cl.shape[0] == n):
            raise L.NmError(f"surface points: depth_raw, acc and rgb must hold {H} x {W} pixels "
                            f"(got {dr.shape[0]}, {ac.shape[0]}, {cl.shape[0]})")
        shapes = dict(points=((n, 3), torch.float32), normals=((n, 3), torch.float32), colors=((n, 3), torch.float32),
                      pixel=((n,), torch.int32))
        outs = {}
        for k, (shape, dt) in shapes.items():
            t = None if out is None else out.get(k)
            if t is None:
                t = torch.empty(shape, dtype=dt, device=self.device)
            assert t.dtype == dt and t.is_contiguous() and t.device == self.device and t.shape[0] >= n, (k, t.shape)
            outs[k] = t
        count = C.c_int64()
        L.check(self.lib.nm_surface_points(self._h, p.ctypes.data, int(H), int(W), float(focal), _ptr(dr), _ptr(ac), _ptr(cl),
                                           float(min_acc), int(step), float(dist_threshold), int(min_count),
                                           _ptr(outs["points"]), _ptr(outs["normals"]), _ptr(outs["colors"]), _ptr(outs["pixel"]),
                                           C.byref(count), self._stream()))
        k = int(count.value)
        return {name: t[:k] for name, t in outs.items()}, k

    # ------------------------------------------------------------------ sparse density sweep (DESIGN 4.10)
    def _sparse_args(self, lins, block, out):
        ls = [np.ascontiguousarray(torch.as_tensor(t).detach().cpu().numpy(), dtype=np.float32) for t in lins]
        n = tuple(a.size for a in ls)
        assert out.shape == n and out.is_contiguous() and out.dtype == torch.float32 and out.device == self.device
        return ls, (self._h, *[a.ctypes.data for a in ls], *n, int(block))

    def sparse_lattice(self, lins, block, out):
        """Step 1 of the sparse sweep (nm_sparse_sweep_lattice): sigma at the lattice points (every `block`-th grid point of
        an axis, and its last) into `out` (n0,n1,n2); returns (min, max, std) over the lattice points.  Synchronises."""
        ls, args = self._sparse_args(lins, block, out)
        st = (C.c_float * 3)()
        L.check(self.lib.nm_sparse_sweep_lattice(*args, _ptr(out), st, self._stream()))
        return float(st[0]), float(st[1]), float(st[2])

    def sparse_run(self, lins, block, iso, out):
        """Steps 2-5 (nm_sparse_sweep_run) on the volume sparse_lattice wrote: seeds, rounds to the fixpoint, +-inf fill.
        Returns (lattice points, active blocks, blocks, evaluated points, rounds)."""
        ls, args = self._sparse_args(lins, block, out)
        counts = (C.c_int64 * 5)()
        L.check(self.lib.nm_sparse_sweep_run(*args, float(iso), _ptr(out), counts, self._stream()))
        return tuple(int(c) for c in counts)

    def sparse_sweep(self, lins, iso_level, block, out):
        """The sparse counterpart of grid_sigma + volume_stats + clamp_iso_level: fills `out` (n0,n1,n2) with sigma in the
        blocks of block^3 cells the iso-surface crosses (followed from block to block to a fixpoint) and +-inf elsewhere.
        The iso level is clamp_iso_level(iso_level, min, max, std) over the LATTICE points: the dense statistics do not
        exist in this mode.  Returns (iso, counts) with counts as sparse_run's."""
        from .mesh import clamp_iso_level
        mn, mx, sd = self.sparse_lattice(lins, block, out)
        iso = float(clamp_iso_level(iso_level, np.float32(mn), np.float32(mx), np.float32(sd)))
        return iso, self.sparse_run(lins, block, iso, out)

    def debug_sparse_state(self, shape, block):
        """Test hook (nm_debug_sparse_sweep_state): the last sparse_run's evaluated mask as a bool tensor of `shape` and its
        block states (nb0,nb1,nb2) int32 (bit 0: corners > iso, bit 1: active)."""
        n0, n1, n2 = shape
        W = (n2 + 31) // 32
        nb = [(n - 1 + block - 1) // block for n in shape]
        words = torch.empty((n0, n1, W), dtype=torch.int32, device=self.device)
        state = torch.empty(nb, dtype=torch.int32, device=self.device)
        L.check(self.lib.nm_debug_sparse_sweep_state(self._h, _ptr(words), _ptr(state), self._stream()))
        bits = (words[..., None] >> torch.arange(32, device=self.device, dtype=torch.int32)) & 1
        return bits.reshape(n0, n1, W * 32)[..., :n2].bool(), state

    # ------------------------------------------------------------------ introspection
    def kernel_flags(self):
        out = (C.c_int32 * 2)()
        L.check(self.lib.nm_kernel_flags(self._h, out))
        return int(out[0]), int(out[1])

    def launch_count(self) -> int:
        return int(self.lib.nm_launch_count(self._h))

    def sigma_only_points(self) -> int:
        """Points sent through a network's sigma-only program since the handle was made."""
        return int(self.lib.nm_sigma_only_points(self._h))

    def set_timing(self, on: bool):
        L.check(self.lib.nm_set_timing(self._h, int(on)))

    def mlp_time_ms(self):
        pts, n = C.c_int64(0), C.c_int64(0)
        ms = float(self.lib.nm_mlp_time_ms(self._h, C.byref(pts), C.byref(n)))
        return ms, int(pts.value), int(n.value)
