"""CPU oracle for the qway/nerfmeshes render / grid hot path.

TEST INFRASTRUCTURE ONLY.  This file restates, in plain torch-CPU fp32 ops,
the algorithm of every function SURVEY.md section 8(a) lists (a1..a14).  It is the
checker the CUDA path is compared against; nothing under `nerfmeshes_b200/`
imports it.  Allowed importers: `tests/`, `__graft_entry__.smoke()` and the
`cpu_baseline` / `--impl reference` legs of `bench.py`.

Parity pin: `tests/golden/*.npz` were produced by running the UNMODIFIED
reference (imported from /root/reference/src through tests/golden/ref_harness.py)
on its shipped checkpoints; `tests/test_oracle_golden.py` checks every function
here against those outputs (bit-exact on the machine that generated them, since
the same torch kernels are called in the same order).

All citations are relative to /root/reference/.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch


# --------------------------------------------------------------------------------------
# configuration records
# --------------------------------------------------------------------------------------
@dataclass
class NetCfg:
    """Shape of one FlexibleNeRFModel (src/nerf/models.py:5-58)."""
    num_layers: int = 8
    hidden_size: int = 256
    skip_step: int = 4
    num_encoding_fn_xyz: int = 10
    num_encoding_fn_dir: int = 4
    include_input_xyz: bool = True
    include_input_dir: bool = True
    log_sampling_xyz: bool = True
    log_sampling_dir: bool = True
    use_viewdirs: bool = True

    @property
    def dim_xyz(self):
        return 6 * self.num_encoding_fn_xyz + (3 if self.include_input_xyz else 0)

    @property
    def dim_dir(self):
        if not self.use_viewdirs:
            return 0
        return 6 * self.num_encoding_fn_dir + (3 if self.include_input_dir else 0)

    def skip_layers(self):
        """Indices i of layers_xyz[i] that take cat(x, PE(p)) (models.py:36-42,64)."""
        return [i for i in range(self.num_layers - 1)
                if i % self.skip_step == 0 and i > 0 and i != self.num_layers - 1]

    def flops_per_point(self, sigma_only=False):
        """2*in*out over the linear layers (BASELINE.md section 2)."""
        h = self.hidden_size
        f = 2 * self.dim_xyz * h
        for i in range(self.num_layers - 1):
            f += 2 * (h + (self.dim_xyz if i in self.skip_layers() else 0)) * h
        if not self.use_viewdirs:
            return f + 2 * h * 4
        f += 2 * h  # fc_alpha
        if sigma_only:
            return f
        f += 2 * h * h  # fc_feat
        f += 2 * (h + self.dim_dir) * (h // 2)
        f += 2 * (h // 2) * 3
        return f


def init_weights(cfg: NetCfg, seed: int) -> Dict[str, torch.Tensor]:
    """Random weights with torch.nn.Linear's default init, keyed like the reference state_dict
    (SURVEY Appendix A.1).  Deterministic in `seed`."""
    g = torch.Generator().manual_seed(seed)

    def lin(i, o):
        bound = 1.0 / math.sqrt(i)
        w = (torch.rand(o, i, generator=g) * 2 - 1) * bound
        b = (torch.rand(o, generator=g) * 2 - 1) * bound
        return w, b

    sd = {}
    h = cfg.hidden_size
    sd["layer1.weight"], sd["layer1.bias"] = lin(cfg.dim_xyz, h)
    for i in range(cfg.num_layers - 1):
        k = h + (cfg.dim_xyz if i in cfg.skip_layers() else 0)
        sd[f"layers_xyz.{i}.weight"], sd[f"layers_xyz.{i}.bias"] = lin(k, h)
    if cfg.use_viewdirs:
        sd["layers_dir.0.weight"], sd["layers_dir.0.bias"] = lin(h + cfg.dim_dir, h // 2)
        sd["fc_alpha.weight"], sd["fc_alpha.bias"] = lin(h, 1)
        sd["fc_rgb.weight"], sd["fc_rgb.bias"] = lin(h // 2, 3)
        sd["fc_feat.weight"], sd["fc_feat.bias"] = lin(h, h)
    else:
        sd["fc_out.weight"], sd["fc_out.bias"] = lin(h, 4)
    return sd


# --------------------------------------------------------------------------------------
# a1 / a2: ray generation
# --------------------------------------------------------------------------------------
def get_ray_bundle(height: int, width: int, focal: float, c2w: torch.Tensor):
    """src/nerf/nerf_helpers.py:226-277 (+ meshgrid_xy :184-196).

    Pixel (row r, col c) -> camera dir [(c - W/2)/f, -(r - H/2)/f, -1], L2-normalised (:267), rotated by
    c2w[:3,:3] as a broadcast-multiply-sum (:270-272).  Returns origin (3,) un-expanded and dirs (H,W,3).
    """
    cols = torch.arange(width, dtype=c2w.dtype)
    rows = torch.arange(height, dtype=c2w.dtype)
    cc = cols[None, :].expand(height, width)
    rr = rows[:, None].expand(height, width)
    cam = torch.stack([(cc - width * 0.5) / focal, -(rr - height * 0.5) / focal, -torch.ones_like(cc)], dim=-1)
    cam = cam / cam.norm(2, dim=-1)[..., None]
    dirs = torch.sum(cam[..., None, :] * c2w[:3, :3], dim=-1)
    return c2w[:3, -1], dirs


def ndc_rays(H, W, focal, near, rays_o, rays_d):
    """src/nerf/nerf_helpers.py:280-307: shift origins onto the z=-near plane, then perspective-warp."""
    t = -(near + rays_o[..., 2]) / rays_d[..., 2]
    rays_o = rays_o + t[..., None] * rays_d
    sx = -1.0 / (W / (2.0 * focal))
    sy = -1.0 / (H / (2.0 * focal))
    o0 = sx * rays_o[..., 0] / rays_o[..., 2]
    o1 = sy * rays_o[..., 1] / rays_o[..., 2]
    o2 = 1.0 + 2.0 * near / rays_o[..., 2]
    d0 = sx * (rays_d[..., 0] / rays_d[..., 2] - rays_o[..., 0] / rays_o[..., 2])
    d1 = sy * (rays_d[..., 1] / rays_d[..., 2] - rays_o[..., 1] / rays_o[..., 2])
    d2 = -2.0 * near / rays_o[..., 2]
    return torch.stack([o0, o1, o2], -1), torch.stack([d0, d1, d2], -1)


def pose_spherical(theta: float, phi: float, radius: float) -> torch.Tensor:
    """src/data/data_helpers.py:10-37 (benchmark poses; SURVEY Appendix A.4).  fp32 numpy trig like the source."""
    def trans(t):
        return np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, t], [0, 0, 0, 1]], dtype=np.float32)

    def rot_phi(p):
        return np.array([[1, 0, 0, 0], [0, np.cos(p), -np.sin(p), 0], [0, np.sin(p), np.cos(p), 0], [0, 0, 0, 1]],
                        dtype=np.float32)

    def rot_theta(th):
        return np.array([[np.cos(th), 0, -np.sin(th), 0], [0, 1, 0, 0], [np.sin(th), 0, np.cos(th), 0], [0, 0, 0, 1]],
                        dtype=np.float32)

    c2w = trans(radius)
    c2w = rot_phi(phi / 180.0 * np.pi) @ c2w
    c2w = rot_theta(theta / 180.0 * np.pi) @ c2w
    c2w = np.array([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1]]) @ c2w
    return torch.from_numpy(c2w.astype(np.float32))


# --------------------------------------------------------------------------------------
# a3 / a4: stratified sampling, points on rays
# --------------------------------------------------------------------------------------
def ray_sample_interval(count: int, ray_count: int, near, far, lindisp=False, perturb=False,
                        generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """src/nerf/modules.py:148-186.  near/far: 0-dim tensors or (R,) tensors."""
    near = torch.as_tensor(near, dtype=torch.float32)
    far = torch.as_tensor(far, dtype=torch.float32)
    s = torch.linspace(0.0, 1.0, count)[None, :]
    per_ray = near.dim() > 0 and near.shape[0] == ray_count
    if per_ray:
        near, far = near[:, None], far[:, None]
    if not lindisp:
        t = near * (1.0 - s) + far * s
    else:
        t = 1.0 / (1.0 / near * (1.0 - s) + 1.0 / far * s)
    if not per_ray:
        t = t.expand([ray_count, count])
    if perturb:
        mids = 0.5 * (t[..., 1:] + t[..., :-1])
        upper = torch.cat((mids, t[..., -1:]), dim=-1)
        lower = torch.cat((t[..., :1], mids), dim=-1)
        t = lower + (upper - lower) * torch.rand(t.shape, generator=generator)
    return t


def intervals_to_ray_points(t, ray_directions, ray_origin):
    """src/models/model_helpers.py:32-35: p = o + d * t (a separate multiply and add, no fma)."""
    return ray_origin[..., None, :] + ray_directions[..., None, :] * t[..., :, None]


# --------------------------------------------------------------------------------------
# a5 / a6: positional encoding and the MLP
# --------------------------------------------------------------------------------------
def frequency_bands(L: int, log_sampling=True) -> torch.Tensor:
    """src/nerf/modules.py:16-23."""
    if log_sampling:
        return 2.0 ** torch.linspace(0.0, L - 1, L)
    return torch.linspace(2.0 ** 0.0, 2.0 ** (L - 1), L)


def positional_encoding(x: torch.Tensor, L: int, include_input=True, log_sampling=True) -> torch.Tensor:
    """src/nerf/modules.py:26-34.  Column order (SURVEY A.2): [x, sin(x_c f_k) c-major k-minor, cos(same)]."""
    parts = [x] if include_input else []
    shp = list(x.shape)
    arg = (frequency_bands(L, log_sampling) * x[..., None].expand(*shp, L)).reshape(*shp[:-1], -1)
    return torch.cat(parts + [torch.sin(arg), torch.cos(arg)], dim=-1)


def flexible_nerf_forward(sd: Dict[str, torch.Tensor], cfg: NetCfg, pts: torch.Tensor,
                          dirs: Optional[torch.Tensor]) -> torch.Tensor:
    """src/nerf/models.py:60-80.  `layer1` has NO activation; the skip concat is [hidden | PE(p)];
    sigma (fc_alpha) is taken from the pre-feat trunk output; output is cat(sigmoid(rgb), raw sigma)."""
    F = torch.nn.functional
    xyz = positional_encoding(pts, cfg.num_encoding_fn_xyz, cfg.include_input_xyz, cfg.log_sampling_xyz)
    x = F.linear(xyz, sd["layer1.weight"], sd["layer1.bias"])
    skips = cfg.skip_layers()
    for i in range(cfg.num_layers - 1):
        if i in skips:
            x = torch.cat((x, xyz), dim=-1)
        x = F.relu(F.linear(x, sd[f"layers_xyz.{i}.weight"], sd[f"layers_xyz.{i}.bias"]))
    if cfg.use_viewdirs:
        view = positional_encoding(dirs, cfg.num_encoding_fn_dir, cfg.include_input_dir, cfg.log_sampling_dir)
        feat = F.relu(F.linear(x, sd["fc_feat.weight"], sd["fc_feat.bias"]))
        alpha = F.linear(x, sd["fc_alpha.weight"], sd["fc_alpha.bias"])
        x = torch.cat((feat, view), dim=-1)
        x = F.relu(F.linear(x, sd["layers_dir.0.weight"], sd["layers_dir.0.bias"]))
        rgb = torch.sigmoid(F.linear(x, sd["fc_rgb.weight"], sd["fc_rgb.bias"]))
        return torch.cat((rgb, alpha), dim=-1)
    out = F.linear(x, sd["fc_out.weight"], sd["fc_out.bias"])
    out[..., :3] = torch.sigmoid(out[..., :3])
    return out


# --------------------------------------------------------------------------------------
# a7: sigma -> alpha compositing
# --------------------------------------------------------------------------------------
def cumprod_exclusive(x: torch.Tensor) -> torch.Tensor:
    """src/nerf/nerf_helpers.py:199-223."""
    c = torch.roll(torch.cumprod(x, -1), 1, -1)
    c[..., 0] = 1.0
    return c


@dataclass
class Bundle:
    """src/nerf/modules.py:40-47 (OutputBundle) + the pre-threshold depth the parity tests use (SURVEY 7.3.3)."""
    rgb_map: torch.Tensor = None
    depth_map: torch.Tensor = None
    weights: torch.Tensor = None
    mask_weights: torch.Tensor = None
    acc_map: torch.Tensor = None
    disp_map: torch.Tensor = None
    depth_raw: torch.Tensor = None


def volume_render(raw: torch.Tensor, t: torch.Tensor, ray_directions: torch.Tensor, *, noise_std=0.0,
                  white_background=False, training=False, attenuation_threshold=1e-5,
                  generator: Optional[torch.Generator] = None, noise: Optional[torch.Tensor] = None) -> Bundle:
    """src/nerf/modules.py:67-121 (threshold 1e-5 from src/models/model_base.py:28-33).  `noise` (shape of raw[..., 3]),
    if given, is the sigma noise itself (already scaled), added instead of noise_std * randn: lets a test feed the
    noise stream of another implementation."""
    big = torch.tensor([1e10]).expand(t[..., :1].shape)
    dists = torch.cat((t[..., 1:] - t[..., :-1], big), dim=-1) * ray_directions[..., None, :].norm(p=2, dim=-1)
    rgb = raw[..., :3]
    if noise is None:
        noise = torch.randn(raw[..., 3].shape, generator=generator) * noise_std if noise_std > 0.0 else 0.0
    sigma = torch.nn.functional.relu(raw[..., 3] + noise)
    alpha = 1.0 - torch.exp(-sigma * dists)
    trans = cumprod_exclusive(1.0 - alpha + 1e-10)
    mask_w = (trans > attenuation_threshold).float()
    w = alpha * trans
    rgb_map = (w[..., None] * rgb).sum(dim=-2)
    acc = w.sum(dim=-1)
    depth = (w * t).sum(dim=-1)
    depth_raw = depth.clone()
    disp = 1.0 / torch.max(1e-10 * torch.ones_like(depth), depth / acc)
    disp[torch.isnan(disp)] = 0
    if not training:
        depth[acc < 1.0] = 0
    if white_background:
        rgb_map = rgb_map + (1.0 - acc[..., None])
    return Bundle(rgb_map, depth, w, mask_w, acc, disp, depth_raw)


# --------------------------------------------------------------------------------------
# a8: inverse-CDF resampling
# --------------------------------------------------------------------------------------
def sample_pdf(bins, weights, u, det=True, generator=None):
    """src/nerf/modules.py:208-248."""
    num = u.shape[-1]
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, dim=-1, keepdim=True)
    cdf = torch.cumsum(pdf, dim=-1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    if det:
        u = u.expand(list(cdf.shape[:-1]) + [num])
    else:
        u = torch.rand(list(cdf.shape[:-1]) + [num], generator=generator)
    u = u.contiguous()
    cdf = cdf.contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)
    cdf_b, cdf_a = torch.gather(cdf, -1, below), torch.gather(cdf, -1, above)
    bin_b, bin_a = torch.gather(bins, -1, below), torch.gather(bins, -1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    return bin_b + (u - cdf_b) / denom * (bin_a - bin_b)


def sample_pdf_forward(t_coarse, weights, num_fine, perturb=False, u=None, generator=None):
    """src/nerf/modules.py:197-206: mids, w[1:-1], inverse CDF, cat with the coarse t, sort."""
    if u is None:
        u = torch.linspace(0.0, 1.0, steps=num_fine)
    mids = 0.5 * (t_coarse[..., 1:] + t_coarse[..., :-1])
    z = sample_pdf(mids, weights[..., 1:-1], u, det=(perturb == 0.0), generator=generator).detach()   # modules.py:201
    out, _ = torch.sort(torch.cat((t_coarse, z), dim=-1), dim=-1)
    return out


# --------------------------------------------------------------------------------------
# a10: AABB-clipped sampling (BuFF)
# --------------------------------------------------------------------------------------
def batch_ray_voxel_intersect(voxels: torch.Tensor, origins: torch.Tensor, dirs: torch.Tensor, near, far,
                              samples_count: int, return_indices: bool = False, literal_sort: bool = False,
                              use_random_sampling: bool = False, generator: Optional[torch.Generator] = None):
    """src/nerf/tree.py:215-343: the deterministic branch (use_random_sampling False in every shipped config) and, with
    use_random_sampling=True, the random one (:280-297: multinomial over voxels weighted 1 on a hit / 1e-12 on a miss, with
    replacement, then a uniform depth inside the drawn voxel's interval; the draws come from torch's generator, so only the
    distribution is comparable with another implementation).

    voxels (V,2,3) [min,max]; origins (1,3) or (R,3); dirs (R,3).  Returns z (R,S) ascending and ray_mask (R,).
    Restated in the textbook slab form, which SURVEY D.3 verified equal to the reference's sequential
    y-then-z test (tree.py:240-262) except for NaN propagation when a direction component is exactly 0:
      per axis  lo = (bound[sign] - o) * (1/d), hi = (bound[1-sign] - o) * (1/d)   (:228-237)
      overlap   pairwise tests in the reference's x,y then (x|y),z order                   (:240-262)
      keep      tmin >= near and tmax <= far  (whole voxel interval inside the cap)        (:268)
    Rays with no hit get ray_mask False; their z rows are unspecified (the caller overwrites them,
    src/models/model_buff.py:53).  If NO ray in the batch hits, the reference returns torch.rand (:274-278);
    we return zeros (the rows are overwritten all the same).
    """
    R, V = dirs.shape[0], voxels.shape[0]
    near = torch.as_tensor(near, dtype=torch.float32)
    far = torch.as_tensor(far, dtype=torch.float32)
    inv = 1 / dirs                                           # (R,3) IEEE inf for zero components
    neg = (inv < 0)                                          # (R,3)
    vmin, vmax = voxels[:, 0, :], voxels[:, 1, :]            # (V,3)
    o = origins if origins.shape[0] == R else origins.expand(R, 3)
    b_lo = torch.where(neg[:, None, :], vmax[None], vmin[None])   # bound[sign]
    b_hi = torch.where(neg[:, None, :], vmin[None], vmax[None])   # bound[1-sign]
    tlo = (b_lo - o[:, None, :]) * inv[:, None, :]           # (R,V,3)
    thi = (b_hi - o[:, None, :]) * inv[:, None, :]
    tmin, tmax = tlo[..., 0].clone(), thi[..., 0].clone()
    mask = (tmin <= thi[..., 1]) & (tlo[..., 1] <= tmax)
    tmin = torch.where(tlo[..., 1] > tmin, tlo[..., 1], tmin)
    tmax = torch.where(thi[..., 1] < tmax, thi[..., 1], tmax)
    mask = mask & (tmin <= thi[..., 2]) & (tlo[..., 2] <= tmax)
    tmin = torch.where(tlo[..., 2] > tmin, tlo[..., 2], tmin)
    tmax = torch.where(thi[..., 2] < tmax, thi[..., 2], tmax)
    mask = mask & (tmin >= near) & (tmax <= far)
    ray_mask = mask.sum(-1) > 0
    z = torch.zeros(R, samples_count)
    if ray_mask.sum() == 0:
        return (z, torch.ones(R, samples_count, dtype=torch.long), ray_mask) if return_indices else (z, ray_mask)
    if use_random_sampling:                                       # (:280-297)
        weights = torch.ones(R, V)
        weights[~mask] = 1e-12
        samples = torch.multinomial(weights, samples_count, replacement=True, generator=generator)
        v_lo, v_hi = tmin.gather(-1, samples), tmax.gather(-1, samples)
        z = v_lo + (v_hi - v_lo) * torch.rand(v_lo.shape, generator=generator)
        z, perm = z.sort(-1)                                      # (:338-341)
        return (z, samples.gather(-1, perm), ray_mask) if return_indices else (z, ray_mask)
    # hits sorted by entry distance, compacted to the front (:299-308)
    order = tmin.sort(-1)
    tmin_s = order.values
    tmax_s = tmax.gather(-1, order.indices)
    mask_s = mask.gather(-1, order.indices)
    front = mask_s.long().sort(descending=True, stable=True)     # stable: keeps tmin order among hits
    lo = torch.where(front.values.bool(), tmin_s.gather(-1, front.indices), torch.zeros(()))
    hi = torch.where(front.values.bool(), tmax_s.gather(-1, front.indices), torch.zeros(()))
    cums = torch.cumsum(hi - lo, -1)                              # (:311-314)
    s = torch.linspace(0, 1.0, samples_count) * cums[..., -1][..., None]      # (:317-318)
    bucket = torch.searchsorted(cums, s.contiguous())            # left (:321)
    first = torch.searchsorted(bucket, bucket, right=False)     # first sample of each bucket (:324)
    z = lo.gather(-1, bucket.clamp(max=V - 1)) + (s - s.gather(-1, first))    # (:327-330)
    z, perm = z.sort(-1)                                          # (:338)
    if not return_indices:
        return z, ray_mask
    # voxel of every sample (:333-341): bucket -> position in the compacted hit list -> position in the entry-sorted
    # list -> voxel id, then reordered like the samples.  Rows of rays without a hit are meaningless (callers index
    # with ray_mask, src/models/model_buff.py:66).
    # QUIRK: the reference compacts the hit INTERVALS by boolean indexing (entry order, :307) but maps buckets to voxels
    # through the permutation of `mask.long().sort(descending=True)` (:305,:333), which torch does not promise to be
    # stable — with the CPU build used for the goldens only 21 % of the samples end up attributed to the voxel that
    # contains them.  literal_sort=True repeats that exact call (pins the oracle to the golden indices); the default
    # is the stable permutation, i.e. every sample is attributed to the voxel whose interval produced it.
    if literal_sort:
        front = mask_s.long().sort(descending=True)
    hit_pos = front.indices.gather(-1, bucket.clamp(max=V - 1))
    vox = order.indices.gather(-1, hit_pos)
    return z, vox.gather(-1, perm), ray_mask


def ray_batch_integration(memm: torch.Tensor, counter: int, indices: torch.Tensor, weights: torch.Tensor,
                          mask_weights: torch.Tensor):
    """src/nerf/tree.py:177-206 past the step gate: per-voxel mean of the sample weights that fell into it, folded into the
    running mean `memm` with 1/counter.  indices / weights / mask_weights are the rows of the rays that hit (…[mask])."""
    V = memm.shape[0]
    acc = torch.zeros(V).index_add_(0, indices.reshape(-1), weights.reshape(-1).float())
    freq = torch.zeros(V).index_add_(0, indices.reshape(-1), mask_weights.reshape(-1).float())
    m = freq > 0
    out = memm.clone()
    out[m] += (acc[m] / freq[m] - out[m]) / counter
    return out, counter + 1


# --------------------------------------------------------------------------------------
# a9 / a11 / a12: the forward orchestration
# --------------------------------------------------------------------------------------
@dataclass
class RenderCfg:
    """The cfg.nerf.* / cfg.dataset.* knobs the hot path reads (SURVEY section 5 'Config / flags')."""
    num_coarse: int = 64
    num_fine: int = 128
    lindisp: bool = False
    perturb: bool = False
    noise_std: float = 0.0
    white_background: bool = False
    attenuation_threshold: float = 1e-5


def nerf_forward(coarse_sd, fine_sd, net_c: NetCfg, net_f: Optional[NetCfg], rcfg: RenderCfg,
                 ray_origins, ray_directions, near, far, training=False, u=None, noise_c=None, noise_f=None):
    """src/models/model_nerf.py:37-78.  Returns (coarse Bundle, fine Bundle or None, t_coarse, t_fine).  noise_c / noise_f:
    explicit sigma noise of the coarse / fine compositor (volume_render's `noise`)."""
    R = ray_directions.shape[0]
    t_c = ray_sample_interval(rcfg.num_coarse, R, near, far, rcfg.lindisp, rcfg.perturb)
    p_c = intervals_to_ray_points(t_c, ray_directions, ray_origins)
    raw_c = flexible_nerf_forward(coarse_sd, net_c, p_c, ray_directions[..., None, :].expand_as(p_c))
    b_c = volume_render(raw_c, t_c, ray_directions, noise_std=rcfg.noise_std, white_background=rcfg.white_background,
                        training=training, attenuation_threshold=rcfg.attenuation_threshold, noise=noise_c)
    if fine_sd is None:
        return b_c, None, t_c, None
    t_f = sample_pdf_forward(t_c, b_c.weights, rcfg.num_fine, rcfg.perturb, u=u)
    p_f = intervals_to_ray_points(t_f, ray_directions, ray_origins)
    raw_f = flexible_nerf_forward(fine_sd, net_f, p_f, ray_directions[..., None, :].expand_as(p_f))
    b_f = volume_render(raw_f, t_f, ray_directions, noise_std=rcfg.noise_std, white_background=rcfg.white_background,
                        training=training, attenuation_threshold=rcfg.attenuation_threshold, noise=noise_f)
    return b_c, b_f, t_c, t_f


def buff_forward(sd, net: NetCfg, rcfg: RenderCfg, voxels, ray_origins, ray_directions, near, far, training=False,
                 noise=None):
    """src/models/model_buff.py:34-69 (inference part): uniform fallback samples, AABB samples, overwrite misses.
    noise: explicit sigma noise (volume_render's `noise`)."""
    R = ray_directions.shape[0]
    t_u = ray_sample_interval(rcfg.num_coarse, R, near, far, rcfg.lindisp, rcfg.perturb)
    z, mask = batch_ray_voxel_intersect(voxels, ray_origins, ray_directions, near, far, rcfg.num_coarse)
    t = torch.where(mask[:, None], z, t_u)
    p = intervals_to_ray_points(t, ray_directions, ray_origins)
    raw = flexible_nerf_forward(sd, net, p, ray_directions[..., None, :].expand_as(p))
    b = volume_render(raw, t, ray_directions, noise_std=rcfg.noise_std, white_background=rcfg.white_background,
                      training=training, attenuation_threshold=rcfg.attenuation_threshold, noise=noise)
    return b, t, mask


def sample_points(sd, net: NetCfg, points, rays):
    """src/models/model_base.py:65-73 -> FlexibleNeRFModel.forward(points, rays)."""
    return flexible_nerf_forward(sd, net, points, rays)


# --------------------------------------------------------------------------------------
# a13 / a14 / a15-rescale: dense grid sweep
# --------------------------------------------------------------------------------------
def grid_points(limit: float, res) -> torch.Tensor:
    """src/mesh_nerf.py:37-40: linspace(-limit, limit, n)^3 'ij' meshgrid flattened x-major -> (n0*n1*n2, 3)."""
    nums = (res,) * 3 if isinstance(res, int) else tuple(res)
    tiles = [torch.linspace(-limit, limit, n) for n in nums]
    return torch.stack(torch.meshgrid(*tiles, indexing="ij"), -1).view(-1, 3).float()


def extract_radiance(sd, net: NetCfg, limit: float, res, batch_size=65536) -> np.ndarray:
    """src/mesh_nerf.py:27-53: batched sample_points with dirs := positions; (res,res,res,4) numpy."""
    nums = (res,) * 3 if isinstance(res, int) else tuple(res)
    pts = grid_points(limit, res)
    out = [sample_points(sd, net, pts[i:i + batch_size], pts[i:i + batch_size]) for i in range(0, pts.shape[0], batch_size)]
    return torch.cat(out, 0).view(*nums, 4).contiguous().numpy()


def extract_iso_level(density: np.ndarray, iso_level: float) -> float:
    """src/mesh_nerf.py:56-65: clamp(iso, min+std, max-std) in numpy float32."""
    mn, mx, sd = density.min(), density.max(), density.std()
    return min(max(iso_level, mn + sd), mx - sd)


def rescale_vertices(verts_index: np.ndarray, limit: float, res: int) -> np.ndarray:
    """src/mesh_nerf.py:90 (keeps the reference's res/2 scale, SURVEY A.8)."""
    return limit * (verts_index / (res / 2.0) - 1.0)
