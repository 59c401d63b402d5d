"""Time one training step of the lego configuration (two 8x256 nets, 64+128 samples) through the fused forward +
backward: nm_loss_backward alone, and the full step with torch.optim.Adam + weight re-upload.  Run on an H100."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import nerfmeshes_b200 as nm

ARCH = dict(num_layers=8, hidden_size=256, skip_step=4, num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True,
            include_input_dir=True, log_sampling_xyz=True, log_sampling_dir=True, use_viewdirs=True)
FLOP_PER_POINT = 1186816          # BASELINE.md section 2
CFG = {"dataset.near": 2.0, "dataset.far": 6.0, "dataset.white_background": True,
       "models.coarse_type": "FlexibleNeRFModel", "models.fine_type": "FlexibleNeRFModel", "models.use_fine": True,
       **{f"models.coarse.{k}": v for k, v in ARCH.items()}, **{f"models.fine.{k}": v for k, v in ARCH.items()}}
for mode in ("train", "validation"):
    CFG.update({f"nerf.{mode}.num_coarse": 64, f"nerf.{mode}.num_fine": 128, f"nerf.{mode}.perturb": True,
                f"nerf.{mode}.lindisp": False, f"nerf.{mode}.radiance_field_noise_std": 0.2})


def main():
    R = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    model = nm.NeRFModel(CFG).cuda().train()
    g = torch.Generator().manual_seed(0)
    o = torch.tensor([0.0, 0.0, 4.0]).cuda()
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g) * 0.2 + torch.tensor([0.0, 0.0, -1.0]), dim=-1).cuda()
    target = torch.rand(R, 3, generator=g).cuda()
    eng = model._engine()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timeit(fn, n=5):
        fn(); torch.cuda.synchronize()
        ev[0].record()
        for _ in range(n):
            fn()
        ev[1].record(); torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / n

    fwd = timeit(lambda: eng.render_rays(o, d, 2.0, 6.0, training=True, seed=1, want=["rgb", "coarse_rgb"]))
    eng.zero_grad()
    bwd = timeit(lambda: eng.loss_backward(o, d, 2.0, 6.0, target, training=True, seed=1))
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)

    def step():
        opt.zero_grad(set_to_none=True)
        c, f = model.forward((o, d, (2.0, 6.0)))
        loss = torch.nn.functional.mse_loss(c.rgb_map, target) + torch.nn.functional.mse_loss(f.rgb_map, target)
        loss.backward()
        opt.step()
    t0 = time.time(); full = timeit(step, 5); wall = (time.time() - t0) / 6
    pts = R * (64 + 192)
    flops = pts * FLOP_PER_POINT * 3
    print(f"R={R}: forward {fwd:.2f} ms | loss+backward (fwd re-run inside) {bwd:.2f} ms = {R / bwd * 1e3:,.0f} rays/s, "
          f"{flops / (bwd - fwd) / 1e9:.1f} TFLOP/s fp32 over the backward part | full autograd+Adam step {full:.2f} ms "
          f"(wall {wall * 1e3:.1f} ms) = {R / full * 1e3:,.0f} rays/s")


if __name__ == "__main__":
    main()
