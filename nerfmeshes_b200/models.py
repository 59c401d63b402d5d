"""Host-side mirror of the reference's model layer for the hot path (the drop-in boundary, SURVEY section 8b).

Same names, constructor arguments, call conventions and state-dict keys as
  src/nerf/models.py:4-80          FlexibleNeRFModel
  src/nerf/modules.py:40-47        OutputBundle
  src/models/model_nerf.py:22-86   NeRFModel   (.forward -> (coarse_bundle, fine_bundle), .query, .get_model)
  src/models/model_buff.py:12-73   BuFFModel   (.forward / .query -> bundle; checkpoint['tree'])
  src/models/model_base.py:65-73   BaseModel.sample_points
but every computation is a call into libnerfmeshes_b200.so through nerfmeshes_b200.engine.Engine.  The classes are
torch.nn.Modules only so that parameters / state_dict / load_state_dict / train() / eval() behave as the reference's
callers expect (PyTorch-Lightning itself is not required).  There is no torch fallback: without an H100 the forward
raises.
"""
from __future__ import annotations

import io
import pickle
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _lib as L
from .cfgnode import CfgNode, flatten_dict, nest_dict
from .tree import Node, TreeSampling
from .engine import NET_KEYS, Engine, RenderSettings


@dataclass
class OutputBundle:
    rgb_map: torch.Tensor = None
    depth_map: torch.Tensor = None
    weights: torch.Tensor = None
    mask_weights: torch.Tensor = None
    acc_map: torch.Tensor = None
    disp_map: torch.Tensor = None
    depth_raw: torch.Tensor = None      # sum(w*t) before the eval-mode threshold (extra; parity tests use it)


class PositionalEncoding(torch.nn.Module):
    """Holder of the `frequency_bands` buffer (state-dict key parity, src/nerf/modules.py:12-24); the encoding itself
    is evaluated inside the fused kernel."""

    def __init__(self, num_encoding_functions=6, include_input=True, log_sampling=True):
        super().__init__()
        self.num_encoding_functions = num_encoding_functions
        self.include_input = include_input
        n = num_encoding_functions
        bands = 2.0 ** torch.linspace(0.0, n - 1, n) if log_sampling else torch.linspace(1.0, 2.0 ** (n - 1), n)
        self.register_buffer("frequency_bands", bands)

    def output_size(self):
        return 6 * self.num_encoding_functions + (3 if self.include_input else 0)


class FlexibleNeRFModel(torch.nn.Module):
    def __init__(self, num_layers=4, hidden_size=128, skip_step=4, num_encoding_fn_xyz=6, num_encoding_fn_dir=4,
                 include_input_xyz=True, include_input_dir=True, log_sampling_xyz=True, log_sampling_dir=True,
                 use_viewdirs=True, **kwargs):
        super().__init__()
        self.arch = dict(num_layers=num_layers, hidden_size=hidden_size, skip_step=skip_step,
                         num_encoding_fn_xyz=num_encoding_fn_xyz, num_encoding_fn_dir=num_encoding_fn_dir,
                         include_input_xyz=include_input_xyz, include_input_dir=include_input_dir,
                         log_sampling_xyz=log_sampling_xyz, log_sampling_dir=log_sampling_dir, use_viewdirs=use_viewdirs)
        self.encode_xyz = PositionalEncoding(num_encoding_fn_xyz, include_input_xyz, log_sampling_xyz)
        self.encode_dir = PositionalEncoding(num_encoding_fn_dir, include_input_dir, log_sampling_dir)
        self.dim_xyz = self.encode_xyz.output_size()
        self.dim_dir = self.encode_dir.output_size() if use_viewdirs else 0
        self.skip_step, self.num_layers, self.use_viewdirs = skip_step, num_layers, use_viewdirs
        Lin = torch.nn.Linear
        self.layer1 = Lin(self.dim_xyz, hidden_size)
        self.layers_xyz = torch.nn.ModuleList()
        for i in range(num_layers - 1):
            skip = i % skip_step == 0 and i > 0 and i != num_layers - 1
            self.layers_xyz.append(Lin(hidden_size + (self.dim_xyz if skip else 0), hidden_size))
        if use_viewdirs:
            self.layers_dir = torch.nn.ModuleList([Lin(self.dim_dir + hidden_size, hidden_size // 2)])
            self.fc_alpha = Lin(hidden_size, 1)
            self.fc_rgb = Lin(hidden_size // 2, 3)
            self.fc_feat = Lin(hidden_size, hidden_size)
        else:
            self.fc_out = Lin(hidden_size, 4)
        self._owner = None      # (parent model, slot) once bound

    def bind(self, owner, which):
        object.__setattr__(self, "_owner", (owner, which))

    def weight_version(self):
        return tuple(p._version for p in self.parameters()) + tuple(p.data_ptr() for p in self.parameters())

    def forward(self, ray_points, ray_directions=None):
        """(…,3),(…,3) -> (…,4) = [sigmoid rgb, raw sigma]  (src/nerf/models.py:60-80)."""
        if self._owner is None:
            raise L.NmError("FlexibleNeRFModel must belong to a NeRFModel/BuFFModel (it runs on that model's engine)")
        owner, which = self._owner
        return owner._engine().point_mlp(which, ray_points, ray_directions)


class _Holder(torch.nn.Module):
    pass


def _cfg_get(node, path, default=None):
    for p in path.split("."):
        if not isinstance(node, dict) or p not in node:
            return default
        node = node[p]
    return node


class _RenderGrad(torch.autograd.Function):
    """Connects the bundles' rgb maps to the networks' parameters: backward() runs nm_backward_rays (the fused
    forward is re-run with the same flags + seed, then the compositor adjoint and the layer-wise backward) and hands
    autograd one gradient per parameter — what loss.backward() yields in the reference (model_nerf.py:88-151)."""

    @staticmethod
    def forward(ctx, model, rays, seed, buff, training, train_skip, rgb, coarse_rgb, *params):
        ctx.model, ctx.rays, ctx.seed, ctx.buff, ctx.training = model, rays, seed, buff, training
        ctx.train_skip = train_skip        # the grids the forward skipped on are still installed: they change only at a step
        ctx.has_coarse = coarse_rgb is not None
        if coarse_rgb is None:
            return rgb.clone()
        return rgb.clone(), coarse_rgb.clone()

    @staticmethod
    def backward(ctx, g_rgb, g_coarse=None):
        model = ctx.model
        eng = model._engine()
        o, d, near, far = ctx.rays
        eng.zero_grad()
        eng.backward_rays(o, d, near, far, g_rgb, g_coarse if ctx.has_coarse else None, training=ctx.training,
                          buff=ctx.buff, seed=ctx.seed, train_skip=ctx.train_skip)
        grads = [eng.get_grad(which, name, p) for which, name, p in model._named_net_params()]
        return (None,) * 8 + tuple(grads)


class BaseModel(torch.nn.Module):
    """Shared part of NeRFModel / BuFFModel (src/models/model_base.py:17-73), minus the Lightning trainer hooks."""

    precision = L.PREC_EXACT
    act_scale_log2 = 0
    skip_empty = False          # eval-mode renders skip empty space (build_occupancy_grid sets it; DESIGN 4.15)

    def __init__(self, cfg, *args, **kwargs):
        super().__init__()
        self.cfg = CfgNode(nest_dict(dict(cfg), sep="."))
        self.hparams = flatten_dict(self.cfg, sep=".")
        vr = _Holder()                                   # VolumeRenderer buffers/attributes (modules.py:51-65)
        vr.train_radiance_field_noise_std = float(_cfg_get(self.cfg, "nerf.train.radiance_field_noise_std", 0.0))
        vr.val_radiance_field_noise_std = float(_cfg_get(self.cfg, "nerf.validation.radiance_field_noise_std", 0.0))
        vr.white_background = bool(_cfg_get(self.cfg, "dataset.white_background", False))
        vr.attenuation_threshold = 1e-5                  # model_base.py:28-33
        vr.register_buffer("one_e_10", torch.tensor([1e10]))
        self.volume_renderer = vr
        self._eng: Optional[Engine] = None
        self._synced = {}
        self._cuda_index = None
        self._train_skip = None          # enable_training_skip's settings and schedule state, or None (off)

    # ------------------------------------------------------------------ engine plumbing
    def _nets(self):
        raise NotImplementedError

    def _render_settings(self) -> RenderSettings:
        raise NotImplementedError

    def cuda(self, device=None):
        if isinstance(device, int):
            self._cuda_index = device
        return super().cuda(device)

    def to(self, *args, **kwargs):
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, (str, torch.device)) and torch.device(a).type == "cuda" and torch.device(a).index is not None:
                self._cuda_index = torch.device(a).index
        return super().to(*args, **kwargs)

    def _device_index(self) -> int:
        """The CUDA device the parameters live on (so `torch.cuda.set_device(rank); model.cuda()` lands on `rank`);
        CPU-resident parameters (host-buffer callers) fall back to an explicit cuda(i)/to('cuda:i'), then the current device."""
        p = next(self.parameters(), None)
        if p is not None and p.is_cuda:
            return p.device.index if p.device.index is not None else torch.cuda.current_device()
        if self._cuda_index is not None:
            return self._cuda_index
        return torch.cuda.current_device() if torch.cuda.is_available() else 0

    def _engine(self) -> Engine:
        nets = self._nets()
        dev = self._device_index()
        if self._eng is not None and self._eng.device.index != dev:
            # the module moved to another GPU after its handle was created: rebuild there (packed weights, tables, tree)
            self._eng.close()
            self._eng, self._synced = None, {}
            if hasattr(self, "_tree_version"):
                self._tree_version = None
        if self._eng is None:
            coarse = nets[0].arch
            fine = nets[1].arch if len(nets) > 1 and nets[1] is not None else None
            self._eng = Engine(coarse, fine, self._render_settings(), device=dev)
            self._after_engine_created()
        for which, net in enumerate(nets):
            if net is None:
                continue
            v = net.weight_version()
            if self._synced.get(which) != v:
                sd = {k: t for k, t in net.state_dict().items()}
                self._eng.load_weights(which, sd)
                self._synced[which] = v
        s = self._render_settings()
        if s != self._eng.settings:
            self._eng.configure(**s.__dict__)
        self._eng.skip_empty = bool(self.skip_empty) and not self.training     # training renders stay dense
        return self._eng

    def _occupancy_box(self, box, what):
        """The grid box: the caller's, else [near - mean, far - mean]^3 with mean = (near + far) / 2; NDC needs one."""
        if box is not None:
            return box
        if _cfg_get(self.cfg, "dataset.use_ndc", False):
            raise L.NmError(f"{what}: an NDC model needs an explicit box (NDC coordinates)")
        near, far = float(self.cfg.dataset.near), float(self.cfg.dataset.far)
        mean = (near + far) / 2
        return [near - mean] * 3 + [far - mean] * 3

    def _build_grids(self, res, box, threshold, dilate):
        eng = self._engine()
        return {which: eng.build_occupancy(which, box, res, threshold, dilate)
                for which, net in enumerate(self._nets()) if net is not None}

    def build_occupancy_grid(self, res: int = 128, box=None, threshold: float = -10.0, dilate: int = 2):
        """Occupancy grids of every network from its own density (Engine.build_occupancy, DESIGN 4.15), then skip_empty:
        eval-mode renders (forward, query, eval_poses, render_image_sharded, surface_points, compare_with_nerf) send only
        the samples in occupied cells, outside the box or not finite through the networks.  A ray's outputs are the dense
        render's bits whenever every sample skipped on it has raw sigma <= 0 (the defaults are chosen so that this holds
        for nearly every ray of the lego and fern scenes; DESIGN 4.15 has the numbers).  box: (lo_x, lo_y, lo_z, hi_x, hi_y,
        hi_z) in network-input coordinates; default [near - mean, far - mean]^3 with mean = (near + far) / 2 (the BuFF
        tree's root box); an NDC model needs an explicit box.  Changing the weights afterwards makes the next skipping
        render raise until the grids are built again.  Returns {slot: bits}."""
        out = self._build_grids(res, self._occupancy_box(box, "build_occupancy_grid"), threshold, dilate)
        self.skip_empty = True
        self._engine()
        return out

    def enable_training_skip(self, every: int = 16, res: int = 128, box=None, threshold: float = -10.0, dilate: int = 2):
        """Empty-space skipping in training (NM_FLAG_SKIP_EMPTY_TRAIN, DESIGN 4.15): every training-mode render (forward
        in train mode and its backward, train.training_step) sends only the samples its network's occupancy grid marks
        through the network.  The grids (parameters and default box as build_occupancy_grid) are rebuilt from the current
        weights before the first training render and then whenever the step has advanced by `every` since the last
        rebuild; the step is `global_step` when training_step is given one, else the count of training_step calls (of
        training-mode forward calls outside training_step).  A ray whose skipped samples all have a noisy pre-activation
        <= 0 trains exactly as the dense step.  Eval-mode skipping stays `skip_empty`'s (build_occupancy_grid).  Grids are
        not stored in checkpoints: a resumed run rebuilds at its first step.  Under torchrun every rank rebuilds from the
        same weights with the same deterministic build, so the ranks' grids agree.  every = 0 switches it off."""
        every = int(every)
        if every < 0:
            raise ValueError("enable_training_skip: every must be >= 0")
        if every == 0:
            self._train_skip = None
            return
        self._train_skip = dict(every=every, res=int(res), box=self._occupancy_box(box, "enable_training_skip"),
                                threshold=float(threshold), dilate=int(dilate), built=None, calls=0, in_step=False,
                                rebuilds=[])

    def _train_skip_tick(self, step=None):
        """Start of a training step: rebuild the grids when the schedule says so.  Returns whether the step skips.  Inside
        training_step (`in_step`) a forward does not tick again, so no rebuild falls between a forward and its backward."""
        ts = self._train_skip
        if ts is None or not self.training:
            return False
        if ts["in_step"] and step is None:
            return True
        if step is None:
            step = ts["calls"]
            ts["calls"] += 1
        if ts["built"] is None or step < ts["built"] or step - ts["built"] >= ts["every"]:
            self._build_grids(ts["res"], ts["box"], ts["threshold"], ts["dilate"])
            ts["built"] = step
            ts["rebuilds"].append(step)
        return True

    def _after_engine_created(self):
        pass

    def _named_net_params(self):
        """[(slot, state-dict key without prefix, parameter)] in a fixed order."""
        out = []
        for which, net in enumerate(self._nets()):
            if net is not None:
                out += [(which, name, p) for name, p in net.named_parameters()]
        return out

    def _pick_seed(self, seed):
        """Explicit seed wins; otherwise a fresh stream per training call (the reference draws new torch.rand
        jitter / noise every forward), and 0 in eval mode where nothing is random."""
        if seed is not None:
            return int(seed)
        if not self.training:
            return 0
        self._seed_counter = getattr(self, "_seed_counter", 0) + 1
        return (torch.initial_seed() * 1000003 + self._seed_counter) & 0x7FFFFFFFFFFFFFFF

    def _attach_grad(self, rays, seed, buff, rgb, coarse_rgb=None, train_skip=False):
        """Make rgb maps differentiable w.r.t. the network parameters when autograd is recording."""
        named = self._named_net_params()
        # training mode only: evaluation scripts call query() outside torch.no_grad() and expect plain tensors
        if not (self.training and torch.is_grad_enabled() and any(p.requires_grad for _, _, p in named)):
            return rgb, coarse_rgb
        if not rgb.is_cuda:
            raise L.NmError("training needs CUDA ray tensors (the backward pass has no host-buffer variant)")
        res = _RenderGrad.apply(self, rays, seed, buff, self.training, train_skip, rgb, coarse_rgb, *[p for _, _, p in named])
        return (res, None) if coarse_rgb is None else res

    def _mode_cfg(self):
        return self.cfg.nerf.train if self.training else self.cfg.nerf.validation

    # ------------------------------------------------------------------ reference surface
    def get_model(self):
        raise NotImplementedError

    def query(self, ray_batch):
        raise NotImplementedError

    def sample_points(self, points, rays=None, **kwargs):
        results = self.get_model().forward(points, rays, **kwargs)
        return results[0] if isinstance(results, tuple) else results

    def density_gradient(self, points):
        """(raw sigma (...), d sigma / d p (...,3)) at points (...,3) on the network sample_points and the grid sweep use
        (the fine one if there is one): the analytic gradient of the fused network (nm_sigma_grad, DESIGN 4.8)."""
        eng = self._engine()
        return eng.sigma_grad(self.get_model()._owner[1], points)

    @staticmethod
    def _unpack(x):
        ray_origins, ray_directions, bounds = x
        near, far = bounds
        return ray_origins, ray_directions, near, far

    # ------------------------------------------------------------------ checkpoints
    @classmethod
    def load_from_checkpoint(cls, path, map_location="cpu", **kw):
        """PyTorch-Lightning 0.9 checkpoint (SURVEY section 5 'Checkpoint / resume') without Lightning installed."""
        ck = load_lightning_checkpoint(path)
        model = cls(dict(ck["hyper_parameters"]))
        if hasattr(model, "on_load_checkpoint"):
            model.on_load_checkpoint(ck)
        model.load_state_dict(ck["state_dict"], strict=False)
        if hasattr(model, "global_step"):
            model.global_step = int(ck.get("global_step", 0))
        return model

    # ------------------------------------------------------------------ optimiser (src/models/model_base.py:150-177)
    def get_scheduler(self, optimizer):
        """Exponential decay gamma ** (step / step_size) (model_base.py:150-158)."""
        gamma = float(self.cfg.scheduler.options.gamma)
        step_size = float(self.cfg.scheduler.options.step_size)
        return torch.optim.lr_scheduler.LambdaLR(optimizer, lr_lambda=lambda step: gamma ** (step / step_size))

    def configure_optimizers(self):
        """getattr(torch.optim, cfg.optimizer.type)(parameters, lr=cfg.optimizer.lr) + a torch scheduler named by
        cfg.scheduler.type, or the exponential LambdaLR above when torch has no scheduler of that name; returned in
        Lightning's ([optimizer], [{'scheduler', 'interval': 'step', 'frequency': 1}]) shape (model_base.py:160-177)."""
        optimizer = getattr(torch.optim, self.cfg.optimizer.type)(self.parameters(), lr=float(self.cfg.optimizer.lr))
        stype = _cfg_get(self.cfg, "scheduler.type", "")
        if stype and hasattr(torch.optim.lr_scheduler, stype):
            scheduler = getattr(torch.optim.lr_scheduler, stype)(optimizer, **dict(self.cfg.scheduler.options))
        else:
            scheduler = self.get_scheduler(optimizer)
        return [optimizer], [{"scheduler": scheduler, "interval": "step", "frequency": 1}]

    def save_checkpoint(self, path, global_step=None, optimizer=None, lr_scheduler=None):
        """Write what load_from_checkpoint reads back, with the keys of a Lightning-0.9 checkpoint (SURVEY section 5
        'Checkpoint / resume'): state_dict under the reference's parameter names, hyper_parameters (the flat config),
        global_step, the on_save_checkpoint extras (BuFF: the voxel tree with its node graph, weights and counter), and
        optionally the optimiser / scheduler states for resuming."""
        ck = {"state_dict": {k: v.detach().cpu() for k, v in self.state_dict().items()},
              "hyper_parameters": dict(self.hparams),
              "global_step": int(getattr(self, "global_step", 0) if global_step is None else global_step),
              "pytorch-lightning_version": "0.9.0"}
        if optimizer is not None:
            ck["optimizer_states"] = [optimizer.state_dict()]
        if lr_scheduler is not None:
            ck["lr_schedulers"] = [lr_scheduler.state_dict()]
        if hasattr(self, "on_save_checkpoint"):
            self.on_save_checkpoint(ck)
        torch.save(ck, path)
        return ck

    @classmethod
    def from_npz(cls, cfg, weights: dict):
        """weights: {'coarse.<key>': tensor, 'fine.<key>': tensor, 'sample_pdf_u': ..., 'voxels': ...} (tests/golden)."""
        model = cls(cfg)
        nets = model._nets()
        for prefix, net in zip(("coarse.", "fine."), nets):
            if net is None:
                continue
            sd = {k[len(prefix):]: torch.as_tensor(v) for k, v in weights.items() if k.startswith(prefix)}
            net.load_state_dict(sd, strict=False)
        if "sample_pdf_u" in weights and hasattr(model, "sample_pdf"):
            model.sample_pdf.u.copy_(torch.as_tensor(weights["sample_pdf_u"]))
        if "voxels" in weights and hasattr(model, "tree"):
            model.tree.set_voxels(weights["voxels"])
        return model


class NeRFModel(BaseModel):
    def __init__(self, cfg, *args, **kwargs):
        super().__init__(cfg, *args, **kwargs)
        m = self.cfg.models
        if m.get("coarse_type", "FlexibleNeRFModel") != "FlexibleNeRFModel":
            raise L.NmError(f"models.coarse_type {m.coarse_type!r}: only FlexibleNeRFModel is on the fused path")
        self.model_coarse = FlexibleNeRFModel(**m.coarse)
        self.model_fine = None
        if "fine" in m and m.get("use_fine", False):
            self.model_fine = FlexibleNeRFModel(**m.fine)
        self.model_coarse.bind(self, L.NET_COARSE)
        if self.model_fine is not None:
            self.model_fine.bind(self, L.NET_FINE)
        sp = _Holder()                                   # SamplePDF buffer (modules.py:190-195)
        sp.num_samples = int(self.cfg.nerf.train.num_fine)
        sp.register_buffer("u", torch.linspace(0.0, 1.0, steps=sp.num_samples))
        self.sample_pdf = sp
        self.sampler = _Holder()                         # RaySampleInterval (non-persistent buffer, modules.py:154-155)
        self.sampler.count = int(self.cfg.nerf.train.num_coarse)
        self.sampler.point_intervals = torch.linspace(0.0, 1.0, self.sampler.count)[None, :]

    def _nets(self):
        return [self.model_coarse, self.model_fine]

    def get_model(self):
        return self.model_fine if self.model_fine is not None else self.model_coarse

    def _render_settings(self):
        mc = self.cfg.nerf.train if self.model_coarse.training else self.cfg.nerf.validation
        vr = self.volume_renderer
        return RenderSettings(
            num_coarse=int(self.cfg.nerf.train.num_coarse),            # sized from .train even in eval (quirk B.1)
            num_fine=int(self.cfg.nerf.train.num_fine) if self.model_fine is not None else 0,
            lindisp=bool(mc.lindisp), perturb=bool(mc.perturb), white_background=vr.white_background,
            noise_std=vr.train_radiance_field_noise_std if self.training else vr.val_radiance_field_noise_std,
            attenuation_threshold=vr.attenuation_threshold, precision=self.precision, act_scale_log2=self.act_scale_log2)

    def _after_engine_created(self):
        self._eng.set_tables(self.sampler.point_intervals[0], self.sample_pdf.u if self.model_fine is not None else None)

    def forward(self, x, seed=None):
        ray_origins, ray_directions, near, far = self._unpack(x)
        tskip = self._train_skip_tick()
        eng = self._engine()
        seed = self._pick_seed(seed)
        want = ["rgb", "depth", "depth_raw", "acc", "disp", "weights", "mask_weights"]
        if self.model_fine is not None:
            want += ["coarse_rgb", "coarse_acc", "coarse_disp", "coarse_weights"]
        o = eng.render_rays(ray_origins, ray_directions, near, far, training=self.training, seed=seed, want=want,
                            train_skip=tskip)
        o["rgb"], crgb = self._attach_grad((ray_origins, ray_directions, near, far), seed, False, o["rgb"], o.get("coarse_rgb"),
                                           tskip)
        if crgb is not None:
            o["coarse_rgb"] = crgb
        main = OutputBundle(o["rgb"], o["depth"], o["weights"], o["mask_weights"], o["acc"], o["disp"], o["depth_raw"])
        if self.model_fine is None:
            return main, None
        coarse = OutputBundle(rgb_map=o["coarse_rgb"], weights=o["coarse_weights"], acc_map=o["coarse_acc"],
                              disp_map=o["coarse_disp"])
        return coarse, main

    def query(self, ray_batch):
        coarse_bundle, fine_bundle = self.forward(ray_batch)
        return fine_bundle if fine_bundle is not None else coarse_bundle


class BuFFModel(BaseModel):
    def __init__(self, cfg, *args, **kwargs):
        super().__init__(cfg, *args, **kwargs)
        m = self.cfg.models
        self.model = FlexibleNeRFModel(**m.coarse)
        self.model.bind(self, L.NET_COARSE)
        self.tree = TreeSampling(self.cfg)
        self.global_step = 0                             # Lightning's step counter: gates the tree integration
        self.sampler = _Holder()
        self.sampler.count = int(self.cfg.nerf.train.num_coarse)
        self.sampler.point_intervals = torch.linspace(0.0, 1.0, self.sampler.count)[None, :]
        self._tree_version = None

    def _nets(self):
        return [self.model]

    def get_model(self):
        return self.model

    def _render_settings(self):
        mc = self.cfg.nerf.train if self.model.training else self.cfg.nerf.validation
        vr = self.volume_renderer
        return RenderSettings(
            num_coarse=int(self.cfg.nerf.train.num_coarse), num_fine=0, lindisp=bool(mc.lindisp), perturb=bool(mc.perturb),
            white_background=vr.white_background,
            noise_std=vr.train_radiance_field_noise_std if self.training else vr.val_radiance_field_noise_std,
            attenuation_threshold=vr.attenuation_threshold, precision=self.precision, act_scale_log2=self.act_scale_log2)

    def _after_engine_created(self):
        self._eng.set_tables(self.sampler.point_intervals[0], None)

    def _sync_tree(self, eng):
        self.tree.engine = eng
        key = (self.tree.version, tuple(self.tree.voxels.shape))
        if self._tree_version != key:
            eng.set_tree(self.tree.voxels)
            self._tree_version = key

    def forward(self, x, seed=None):
        ray_origins, ray_directions, near, far = self._unpack(x)
        seed = self._pick_seed(seed)
        if torch.as_tensor(ray_origins).dim() < 2:
            raise IndexError("BuFFModel needs ray origins of shape (1,3) or (R,3) (src/nerf/tree.py:231)")
        tskip = self._train_skip_tick()
        eng = self._engine()
        self._sync_tree(eng)
        eng.voxel_random = bool(_cfg_get(self.cfg, "tree.use_random_sampling", False))      # src/nerf/tree.py:280
        o = eng.render_rays(ray_origins, ray_directions, near, far, training=self.training, buff=True, seed=seed,
                            want=["rgb", "depth", "depth_raw", "acc", "disp", "weights", "mask_weights", "t_vals"],
                            train_skip=tskip)
        if self.training and o["rgb"].is_cuda:
            # accumulate the (detached) sample weights into the voxels (model_buff.py:65-66; tree.py:177-206)
            step_gate = int(_cfg_get(self.cfg, "tree.step_size_integration_offset", 0) or 0)
            if self.global_step >= step_gate:
                idx = eng.ray_voxel_indices(ray_origins, ray_directions, near, far, seed=seed)
                eng.check_flags()      # a truncated hit list (> 512 voxels on a ray) must not reach the tree statistics
                self.tree.ray_batch_integration(self.global_step, idx, o["weights"], o["mask_weights"])
        o["rgb"], _ = self._attach_grad((ray_origins, ray_directions, near, far), seed, True, o["rgb"], None, tskip)
        b = OutputBundle(o["rgb"], o["depth"], o["weights"], o["mask_weights"], o["acc"], o["disp"], o["depth_raw"])
        b.t_vals = o["t_vals"]
        return b

    def query(self, ray_batch):
        return self.forward(ray_batch)

    def on_save_checkpoint(self, checkpoint):
        checkpoint["tree"] = self.tree.serialize()

    def on_load_checkpoint(self, checkpoint):
        self.tree.deserialize(checkpoint["tree"])


# ---------------------------------------------------------------------------------------------------------------------
class _AttributeDict(dict):
    __getattr__ = dict.get

    def __setattr__(self, k, v):
        self[k] = v


class _CkptUnpickler(pickle.Unpickler):
    """Resolves the two foreign classes inside the shipped checkpoints without importing their packages:
    pytorch_lightning.utilities.parsing.AttributeDict and nerf.tree.Node."""

    def find_class(self, module, name):
        if name == "AttributeDict" and module.startswith("pytorch_lightning"):
            return _AttributeDict
        if name == "Node" and module in ("nerf.tree", "tree"):
            return Node
        if module.startswith("nerf.cfgnode") or (module == "nerf" and name == "CfgNode"):
            return CfgNode
        return super().find_class(module, name)


class _PickleModule:
    __name__ = "nerfmeshes_b200_ckpt_pickle"
    Unpickler = _CkptUnpickler
    load = staticmethod(lambda f, **kw: _CkptUnpickler(f, **kw).load())
    loads = staticmethod(lambda b, **kw: _CkptUnpickler(io.BytesIO(b), **kw).load())
    dump, dumps, Pickler = pickle.dump, pickle.dumps, pickle.Pickler
    HIGHEST_PROTOCOL, DEFAULT_PROTOCOL = pickle.HIGHEST_PROTOCOL, pickle.DEFAULT_PROTOCOL


def load_lightning_checkpoint(path):
    return torch.load(path, map_location="cpu", weights_only=False, pickle_module=_PickleModule)


def state_dict_to_npz(path, **tensors):
    np.savez_compressed(path, **{k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in tensors.items()})
