"""MipRunner: the reference's contrib/mipnerf runner/runner.py:13-225 on the Mip-NeRF kernels (DESIGN.md section 11).

One training step: Blender batch (ops.mip_rays; Blenders / Multicam: ops.mip_rays_multi, with per-ray loss weights) -> coarse fenceposts (ops.mip_sample) -> network -> composite with the coarse weights
(ops.mip_composite_fwd) -> resampled fenceposts (ops.mip_resample) -> network -> the loss of both levels and its gradient with respect to
every raw output in one launch (ops.mip_composite_loss_bwd) -> network backward -> LinearLog + Adam (no EMA).  With the fused fp16 model
the two forwards save into the two halves of one buffer and ONE ops.nerf_bwd covers both levels' rows (one ordered reduction: the
gradient is bit-deterministic); with the fp32 nn.Linear model torch autograd runs the chain backward."""
import os

import numpy as np
import torch

from . import ops
from .plugin import losses as L
from .utils.config import get_cfg
from .utils.registry import DATASETS, LOSSES, NETWORKS, OPTIMS, SAMPLERS, build_from_cfg


class MipRunner:
    def __init__(self, rank=0, world_size=1, process_group=None):
        if world_size > 1:
            raise NotImplementedError("MipRunner: data-parallel training is not supported for Mip-NeRF")
        self.cfg = cfg = get_cfg()
        if int(cfg.num_levels) != 2:
            raise NotImplementedError(f"MipRunner: num_levels must be 2 (coarse + fine, mip_base.py), got {cfg.num_levels}")
        if not cfg.stop_level_grad:
            raise NotImplementedError("MipRunner: stop_level_grad=False (gradients through the resampling) is not supported")
        unread = [k for k in ("near", "far") if cfg.get(k) is not None and any(
            d is not None and d.get("type") in ("Blender", "SyntheticBlender") and k not in d
            for d in (cfg.dataset.train, cfg.dataset.val, cfg.dataset.test))]
        if unread:
            # mip_base.py sets near / far at the top level, where nothing reads them: Blender then samples [0, 1] (DESIGN.md section 7)
            print(f"WARNING: config keys {', '.join(unread)} are not read: Blender takes near / far from the dataset dicts "
                  f"(defaults 0 and 1); pass them there, as mip_cfg() does", flush=True)
        self.dataset = {"train": build_from_cfg(cfg.dataset.train, DATASETS)}
        cfg.dataset_obj = self.dataset["train"]
        self.dataset["val"] = build_from_cfg(cfg.dataset.val, DATASETS) if cfg.dataset.val else None
        self.dataset["test"] = None
        self.model = build_from_cfg(cfg.model, NETWORKS)
        cfg.model_obj = self.model
        self.sampler = build_from_cfg(cfg.sampler, SAMPLERS)
        cfg.sampler_obj = self.sampler
        self.optimizer = build_from_cfg(cfg.optim, OPTIMS, params=list(self.model.parameters()))
        self.optimizer = build_from_cfg(cfg.linearlog, OPTIMS, nested_optimizer=self.optimizer)
        self.loss_func = build_from_cfg(cfg.loss, LOSSES)
        self.tot_train_steps = cfg.tot_train_steps
        self.coarse_loss_mult = float(cfg.coarse_loss_mult)
        self.using_fp16 = bool(cfg.using_fp16)
        self.disable_multiscale_loss = bool(cfg.disable_multiscale_loss)
        self.test_psnr_by_size = {}                                  # (W, H) -> mean test PSNR of that image size, set by test()
        self.chunk = 3072                                            # rays per rendered chunk (runner.py:55)
        self.start = 0
        cfg.m_training_step = 0
        self._saved = None                                           # the fused forwards' saved activations of both levels

    # ------------------------------------------------------------------------------------------ training
    def _forward_levels(self, rays, save):
        """Both levels of rays: (t (2R, S + 1), raw (2 R S, 4)) with the coarse level first.  save (fused model): the forwards save into
        the two halves of self._saved for the one backward."""
        s, m = self.sampler, self.model
        R, S = rays.shape[0], s.num_samples
        n = R * S
        t_c = s.sample(rays, 0)
        if self.using_fp16:
            raw = torch.empty((2 * n, 4), dtype=torch.float16, device=rays.device)
            saved = [None, None]
            if save:
                if n % 128:
                    raise ValueError(f"MipRunner: the fused backward needs n_rays * num_samples to be a multiple of 128, got {n}")
                half = ops.mip_workspace_bytes(n, m.degs)[0]
                if self._saved is None or self._saved.numel() < 2 * half:
                    self._saved = torch.empty(2 * half, dtype=torch.uint8, device=rays.device)
                saved = [self._saved[:half], self._saved[half:2 * half]]
            m.raw(rays, t_c, out=raw[:n], saved=saved[0])
            raw_c = raw[:n]
        else:
            raw_c = m.raw(rays, t_c)
        w = s.rays2rgb(rays, raw_c.detach(), t_c)[3]
        t_f = s.sample(rays, 1, t_c, w)
        if self.using_fp16:
            m.raw(rays, t_f, out=raw[n:], saved=saved[1])
        else:
            raw = (raw_c, m.raw(rays, t_f))
        return torch.cat([t_c, t_f]), raw

    def train_step(self, batch=None):
        """One step of runner.py:75-97; returns the loss (device scalar).  A batch of Blenders / Multicam carries the rays' lossmult, the loss
        mask of runner.py:83-85 unless disable_multiscale_loss."""
        cfg, s, m = self.cfg, self.sampler, self.model
        batch = next(self.dataset["train"]) if batch is None else batch
        rays, target = batch[:2]
        mask = batch[2] if len(batch) > 2 and not self.disable_multiscale_loss else None
        R = rays.shape[0]
        t, raw = self._forward_levels(rays, save=True)
        raw_all = raw if self.using_fp16 else torch.cat([r.detach() for r in raw])
        # fp16 gradients of a ray-mean loss would underflow: the fused path carries them scaled by R and Adam takes them back by 1 / R
        scale = float(R) if self.using_fp16 else 1.0
        _, loss, draw = ops.mip_composite_loss_bwd(raw_all, t, rays, target, mask, s.rgb_padding, s.density_bias, s.white_bkgd,
                                                   self.coarse_loss_mult, grad_scale=scale)
        adam = self.optimizer._nested_optimizer
        self.optimizer.advance_lr()
        if self.using_fp16:
            grad = ops.mip_bwd(m.params, self._saved, draw, m.degs)
            adam.n_step += 1
            st = adam.state[0]
            ops.adam_ema(m.params.data, grad, st.m, st.v, st.master, adam.lr, adam.n_step, adam.betas[0], adam.betas[1], adam.eps, 0.0,
                         grad_scale=1.0 / scale, zero_grad=False)
        else:
            n = R * s.num_samples
            torch.autograd.backward(list(raw), [draw[:n], draw[n:]])
            adam.step()
        cfg.m_training_step += 1
        return loss.sum()

    def train(self, steps=None, log_every=0):
        end = self.tot_train_steps if steps is None else self.cfg.m_training_step + steps
        while self.cfg.m_training_step < end:
            loss = self.train_step()
            i = self.cfg.m_training_step
            if log_every and i % log_every == 0:
                print(f"STEP={i} | LOSS={loss.item():.6f}", flush=True)

    # ------------------------------------------------------------------------------------------ evaluation
    @torch.no_grad()
    def render_rays(self, rays):
        """The fine level's (rgb (R, 3), distance (R,), acc (R,)) of rays, in chunks of self.chunk rays, all on the device."""
        R = rays.shape[0]
        rgb = torch.empty((R, 3), dtype=torch.float32, device=rays.device)
        dist = torch.empty(R, dtype=torch.float32, device=rays.device)
        acc = torch.empty(R, dtype=torch.float32, device=rays.device)
        for p in range(0, R, self.chunk):
            r = rays[p:p + self.chunk]
            t, raw = self._forward_levels(r, save=False)
            n = r.shape[0] * self.sampler.num_samples
            raw_f = raw[n:] if self.using_fp16 else raw[1]
            rgb[p:p + r.shape[0]], acc[p:p + r.shape[0]], dist[p:p + r.shape[0]], _ = self.sampler.rays2rgb(r, raw_f, t[r.shape[0]:], weights=False)
        return rgb, dist, acc

    @torch.no_grad()
    def render_img(self, dataset_mode="val", img_id=0):
        """runner.py:195-225 for image img_id: (img (H, W, 3), target (H, W, 3)) on the device."""
        return self._render_image(self.dataset[dataset_mode], img_id)

    def _render_image(self, ds, img_id):
        rays, target = ds.image_rays(img_id)
        rgb, _, _ = self.render_rays(rays)
        H, W = ds.image_hw(img_id)
        return rgb.reshape(H, W, 3), target.reshape(H, W, 3)

    def _save_path(self):
        return os.path.join(self.cfg.log_dir or ".", self.cfg.exp_name or "exp")

    @staticmethod
    def save_img(path, img):
        from PIL import Image
        img = img.detach().cpu().numpy() if torch.is_tensor(img) else np.asarray(img)
        Image.fromarray((img * 255 + 0.5).clip(0, 255).astype(np.uint8)).save(path)

    @torch.no_grad()
    def val_img(self, it, img_id=0):
        """runner.py:153-160: render a validation image, save img{it}.png / target{it}.png, return its mse."""
        img, tar = self.render_img("val", img_id)
        os.makedirs(self._save_path(), exist_ok=True)
        self.save_img(os.path.join(self._save_path(), f"img{it}.png"), img)
        self.save_img(os.path.join(self._save_path(), f"target{it}.png"), tar)
        return float(L.img2mse(img, tar).item())

    @torch.no_grad()
    def test(self, load_ckpt=False):
        """runner.py:108-121 + 162-179: every test view to log_dir/exp_name/test/{exp_name}_r_{i}.png and _gt_{i}.png; prints and returns
        the mean test PSNR, and the mean PSNR of every image size (the multiscale metric of Mip-NeRF) in self.test_psnr_by_size, also printed."""
        if load_ckpt:
            self.load_ckpt(self.cfg.ckpt_path)
        if self.dataset["test"] is None:
            self.dataset["test"] = build_from_cfg(self.cfg.dataset.test, DATASETS)
        ds = self.dataset["test"]
        out = os.path.join(self._save_path(), "test")
        os.makedirs(out, exist_ok=True)
        psnr, by_size = [], {}
        for i in range(ds.n_images):
            img, tar = self._render_image(ds, i)
            self.save_img(os.path.join(out, f"{self.cfg.exp_name}_r_{i}.png"), img)
            self.save_img(os.path.join(out, f"{self.cfg.exp_name}_gt_{i}.png"), tar)
            psnr.append(float(L.mse2psnr(L.img2mse(img, tar)).item()))
            by_size.setdefault((img.shape[1], img.shape[0]), []).append(psnr[-1])
        mean = sum(psnr) / len(psnr)
        self.test_psnr_by_size = {k: sum(v) / len(v) for k, v in sorted(by_size.items(), reverse=True)}
        for (w, h), p in self.test_psnr_by_size.items():
            print(f"TEST PSNR {w}x{h}===={p}", flush=True)
        print(f"TOTAL TEST PSNR===={mean}", flush=True)
        return mean

    def render(self, *a, **k):
        raise NotImplementedError("MipRunner has no video task (the reference's MipRunner has no render)")

    def extract_mesh(self, *a, **k):
        raise NotImplementedError("MipRunner: mesh extraction runs on the fused NGP kernels only")

    # ------------------------------------------------------------------------------------------ checkpoint
    def save_ckpt(self, path):
        if str(path).endswith(".pkl"):
            raise NotImplementedError("MipRunner: the .pkl interchange format is not supported; save to a .pt path")
        torch.save({"global_step": self.cfg.m_training_step, "model": self.model.state_dict(), "sampler": self.sampler.state_dict(),
                    "optimizer": self.optimizer.state_dict(), "nested_optimizer": self.optimizer._nested_optimizer.state_dict()}, path)

    def load_ckpt(self, path):
        if str(path).endswith(".pkl"):
            raise NotImplementedError("MipRunner: the .pkl interchange format is not supported; load a .pt checkpoint")
        ck = torch.load(path, map_location="cuda", weights_only=True)
        self.cfg.m_training_step = self.start = ck["global_step"]
        self.model.load_state_dict(ck["model"])
        self.sampler.load_state_dict(ck["sampler"])
        self.optimizer.load_state_dict(ck["optimizer"])
        self.optimizer._nested_optimizer.load_state_dict(ck["nested_optimizer"])


def mip_cfg(synthetic=True, **over):
    """contrib/mipnerf projects/mipnerf/configs/mip_base.py key for key, except that near = 2 / far = 6 are also passed into the dataset
    dicts (mip_base.py sets them only at the top level, where nothing reads them; DESIGN.md section 7); `synthetic` swaps the lego scene
    for the procedural stand-in (plugin/mip.py: SyntheticBlender)."""
    ds_type = "SyntheticBlender" if synthetic else "Blender"
    ds_dir = "nerf_data/nerf_synthetic/lego/"
    tot = 40001
    c = dict(
        sampler=dict(type="MipSampler"), model=dict(type="MipNerfMLP"), loss=dict(type="MSELoss"),
        optim=dict(type="Adam", lr=8e-3, eps=1e-15, betas=(0.9, 0.99)),
        dataset_type=ds_type, dataset_dir=ds_dir,
        dataset=dict(train=dict(type=ds_type, root_dir=ds_dir, batch_size=288, mode="train", near=2., far=6.),
                     val=dict(type=ds_type, root_dir=ds_dir, batch_size=4096, mode="val", preload_shuffle=False, near=2., far=6.),
                     test=dict(type=ds_type, root_dir=ds_dir, batch_size=4096, mode="test", preload_shuffle=False, near=2., far=6.)),
        exp_name="lego_sss", log_dir="./logs", tot_train_steps=tot, background_color=[0, 0, 0], hash_func="p0 ^ p1 * 19349663 ^ p2 * 83492791",
        cone_angle_constant=0.00390625, near_distance=0.2, n_rays_per_batch=4096, n_training_steps=16, target_batch_size=1 << 18, const_dt=True,
        fp16=False, white_bkgd=False, using_fp16=False, num_levels=2, num_samples=128, net_depth=8, skip_layer=4, net_width=256,
        net_depth_condition=1, net_width_condition=128, num_density_channels=1, num_rgb_channels=3, resample_padding=0.01, lindisp=False,
        ray_shape="cone", min_deg_point=0, max_deg_point=8, coarse_loss_mult=0.1, disable_multiscale_loss=False, randomized=True,
        disable_integration=False, use_viewdirs=True, deg_view=4, density_noise=0., density_bias=-1., rgb_padding=0.001, stop_level_grad=True,
        near=2., far=6., linearlog=dict(type="LinearLog", end_lr=5e-6, max_steps=tot, lr_delay_steps=2500, lr_delay_mult=0.01),
    )
    c.update(over)
    return c


def multicam_cfg(root_dir=None, synthetic=True, **over):
    """contrib/mipnerf projects/mipnerf/configs/multicam.py key for key: Blenders at 16 IPE degrees, 3072-ray batches, the fp32 network,
    120 001 steps.  root_dir: the capture's directory (default: multicam.py's own path); `synthetic` without a root_dir swaps the dataset
    for the multiscale procedural stand-in (plugin/mip.py: SyntheticMulticam)."""
    ds_type = "SyntheticMulticam" if synthetic and root_dir is None else "Blenders"
    ds_dir = root_dir if root_dir is not None else "/mnt/disk3/zhm/data/nerf_synthetic/lego/"
    tot = 120001
    c = dict(
        sampler=dict(type="MipSampler"), model=dict(type="MipNerfMLP"), loss=dict(type="MSELoss"),
        optim=dict(type="Adam", lr=5e-4, eps=1e-15, betas=(0.9, 0.99)),
        dataset_type=ds_type, dataset_dir=ds_dir,
        dataset=dict(train=dict(type=ds_type, data_dir=ds_dir, batch_size=3072, split="train", batch_type="all_images"),
                     val=dict(type=ds_type, data_dir=ds_dir, batch_size=1, split="val", batch_type="single_image"),
                     test=dict(type=ds_type, data_dir=ds_dir, batch_size=1, split="test", batch_type="single_image")),
        num_levels=2, num_samples=128, resample_padding=0.01, rgb_padding=0.001, net_depth=8, skip_layer=4, net_width=256,
        net_depth_condition=1, net_width_condition=128, num_density_channels=1, num_rgb_channels=3, ray_shape="cone", min_deg_point=0,
        max_deg_point=16, use_viewdirs=True, deg_view=4, density_noise=0., density_bias=-1.,
        exp_name="test", log_dir="./logs", tot_train_steps=tot, background_color=[0, 0, 0], hash_func="p0 ^ p1 * 19349663 ^ p2 * 83492791",
        cone_angle_constant=0.00390625, near_distance=0.2, n_rays_per_batch=4096, n_training_steps=16, target_batch_size=1 << 18, const_dt=True,
        fp16=False, white_bkgd=False, using_fp16=False, lindisp=False, coarse_loss_mult=0.1, disable_multiscale_loss=False, randomized=True,
        disable_integration=False, stop_level_grad=True, near=2., far=6.,
        linearlog=dict(type="LinearLog", end_lr=5e-6, max_steps=tot, lr_delay_steps=2500, lr_delay_mult=0.01),
    )
    c.update(over)
    return c
