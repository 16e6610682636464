"""Svox2Runner: the reference's contrib/plenoxel runner/runner_svox2.py on the Plenoxels kernels (DESIGN.md section 12).

One training step: ray ids drawn with replacement -> ops.svox_train_step (rays made from the pixel ids, forward, MSE gradient and
backward in one launch, gradients as fixed-point sums) -> sparse TV of density and colour (ops.svox_tv_grad, into the same sums) ->
ops.svox_rmsprop (reads and clears the sums).  No host synchronisation inside an epoch: the per-ray squared errors are summed on the
device, and the fixed-point overflow flag is read at the epoch's end, where the runner synchronises anyway."""
import math
import os

import numpy as np
import torch

from . import ops
from .plugin import losses as L
from .plugin.optim import PlenOptimRMSprop
from .plugin.svox2 import SparseGrid
from .utils.config import get_cfg
from .utils.registry import DATASETS, build_from_cfg

SEED = 20200823


def get_expon_lr_func(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """svox2_utils.py:532-565: log-linear decay from lr_init to lr_final over max_steps, eased in over lr_delay_steps by a sine."""
    def helper(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        if lr_delay_steps > 0:
            delay_rate = lr_delay_mult + (1 - lr_delay_mult) * np.sin(0.5 * np.pi * np.clip(step / lr_delay_steps, 0, 1))
        else:
            delay_rate = 1.0
        t = np.clip(step / max_steps, 0, 1)
        return float(delay_rate * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t))
    return helper


def tv_cells(grid_size, sparse_frac, gen):
    """_get_rand_cells (svox2_network.py:291-306), contiguous: (start, n); the cells are (start + i) mod grid_size, i < n."""
    n = max(int(sparse_frac * grid_size), 1)
    return int(torch.randint(0, grid_size, (1,), generator=gen)), n


class Svox2Runner:
    def __init__(self):
        self.cfg = cfg = get_cfg()
        self._refuse(cfg)
        # Jittor's global seed cannot be reproduced: ray ids come from a device generator and TV starts from a host one, both seeded here
        self.gen = torch.Generator(device="cuda").manual_seed(SEED)
        self.tv_gen = torch.Generator().manual_seed(SEED)
        self.exp_name = cfg.exp_name
        self.dataset = {"train": build_from_cfg(cfg.dataset.train, DATASETS)}
        cfg.dataset_obj = self.dataset["train"]
        self.dataset["val"] = build_from_cfg(cfg.dataset.val, DATASETS) if cfg.dataset.val else self.dataset["train"]
        self.dataset["test"] = None
        self.reso_list = cfg.reso_list
        ds = self.dataset["train"]
        self.model = SparseGrid(self.reso_list[0], ds.scene_radius, ds.scene_center, 1, cfg.model.basis_dim, cfg.model.basis_reso, use_z_order=True,
                                use_sphere_bound=ds.use_sphere_bound and not cfg.nosphereinit)
        cfg.model_obj = self.model
        self.optimizer = PlenOptimRMSprop(self.model.density_data, self.model.sh_data, 0, 0, 0.95, 0.95)
        self.lr_sigma_func = get_expon_lr_func(cfg.lr_sigma, cfg.lr_sigma_final, cfg.lr_sigma_delay_steps, cfg.lr_sigma_delay_mult,
                                               cfg.lr_sigma_decay_steps)
        self.lr_sh_func = get_expon_lr_func(cfg.lr_sh, cfg.lr_sh_final, cfg.lr_sh_delay_steps, cfg.lr_sh_delay_mult, cfg.lr_sh_decay_steps)
        self.save_path = os.path.join(cfg.log_dir or ".", self.exp_name or "exp")
        os.makedirs(self.save_path, exist_ok=True)
        self.ckpt_path = cfg.ckpt_path if cfg.ckpt_path else os.path.join(self.save_path, "ckpt.npz")
        self.start = 0
        if cfg.load_ckpt:
            self.load_ckpt(self.ckpt_path)
        cfg.m_training_step = 0
        self.factor = 1
        self.stats = []

    @staticmethod
    def _refuse(cfg):
        if cfg.enable_random and cfg.random_sigma_std:
            raise NotImplementedError("Svox2Runner: randomized sigma noise (enable_random with random_sigma_std > 0) is not supported")
        if cfg.model and cfg.model.get("background_nlayers", 0):
            raise NotImplementedError("Svox2Runner: the background MSI model (background_nlayers > 0) is not supported")
        if cfg.use_spheric_clip or cfg.last_sample_opaque:
            raise NotImplementedError("Svox2Runner: use_spheric_clip / last_sample_opaque (forward-facing scenes) are not supported")
        if cfg.tv_logalpha:
            raise NotImplementedError("Svox2Runner: tv_logalpha is not supported (the reference asserts it off)")
        if cfg.tv_contiguous is not None and not cfg.tv_contiguous:
            raise NotImplementedError("Svox2Runner: non-contiguous TV cells (tv_contiguous=0) are not supported")
        if (cfg.weight_decay_sh or 1.0) != 1.0 or (cfg.weight_decay_sigma or 1.0) != 1.0 or (cfg.upsample_density_add or 0.0) != 0.0:
            raise NotImplementedError("Svox2Runner: weight_decay_sh / weight_decay_sigma != 1 and upsample_density_add != 0 are not supported")

    # ------------------------------------------------------------------------------------------ training
    def train_step(self, gstep, n_rays=None, events=None):
        """One step of runner_svox2.py:172-240 at global step gstep: returns the per-ray squared errors (device).  events: None, or 4
        CUDA events recorded before the fused step, after it, after the TV and after RMSprop (tools/svox2_bench.py times the stages)."""
        args, grid, opt, ds = self.cfg, self.model, self.optimizer, self.dataset["train"]
        rec = (lambda i: events[i].record()) if events is not None else (lambda i: None)
        n = int(args.batch_size) if n_rays is None else n_rays
        if (args.lr_fg_begin_step or 0) > 0 and gstep == args.lr_fg_begin_step:
            grid.density_data.fill_(float(args.init_sigma))
        lr_sigma, lr_sh = self.lr_sigma_func(gstep), self.lr_sh_func(gstep)
        if not args.lr_decay:
            lr_sigma, lr_sh = args.lr_sigma, args.lr_sh
        rec(0)
        pix = torch.randint(0, ds.n_rays, (n,), generator=self.gen, device=ds.images.device, dtype=torch.int32)
        sqerr = ops.svox_train_step(pix, ds.w, ds.h, ds.c2w_rows, (ds.focal, ds.focal, ds.w * 0.5, ds.h * 0.5), ds.images, grid._links,
                                    grid.density_data, grid.sh_data, grid.xform(), grid.opt.as_array(), opt.grad_density, opt.grad_sh, opt.flag)
        rec(1)
        opt.update_lr(lr_sigma, lr_sh, args.rms_beta, args.rms_beta)
        G = grid._links.numel()
        if args.lambda_tv > 0.0:
            start, nc = tv_cells(G, args.tv_sparsity, self.tv_gen)
            ops.svox_tv_grad(grid._links, grid.density_data, start, nc, args.lambda_tv / nc, False, opt.grad_density, opt.flag)
        if args.lambda_tv_sh > 0.0:
            start, nc = tv_cells(G, args.tv_sh_sparsity, self.tv_gen)
            ops.svox_tv_grad(grid._links, grid.sh_data, start, nc, args.lambda_tv_sh / nc, True, opt.grad_sh, opt.flag)
        rec(2)
        opt.step()
        rec(3)
        self.cfg.m_training_step += 1
        return sqerr

    def _resample_cameras(self):
        ds = self.dataset["train"]
        return [ds.camera(i) for i in range(ds.n_images)]

    def train(self, log_every=0):
        """runner_svox2.py:71-285: epochs of epoch_size rays, an eval at the start of each, upsampling every upsamp_every steps, the last
        eval and ckpt.npz at n_iters."""
        args = self.cfg
        self.model.param_init(args)
        last_upsamp_step = args.init_iters or 0
        epoch_id, reso_id, gstep_id_base = -1, 0, 0
        ds = self.dataset["train"]
        while True:
            epoch_id += 1
            epoch_size = int(ds.epoch_size)
            batches_per_epoch = (epoch_size - 1) // args.batch_size + 1
            if epoch_id % max(self.factor, args.eval_every) == 0:
                self.eval_step(epoch_id, gstep_id_base)
            se = torch.zeros((), dtype=torch.float32, device=ds.images.device)
            for iter_id in range(batches_per_epoch):
                n = min(args.batch_size, epoch_size - iter_id * args.batch_size)
                sq = self.train_step(iter_id + gstep_id_base, n)
                se += sq.sum() / (3 * n)
                if log_every and (iter_id + 1) % log_every == 0:
                    print(f"epoch {epoch_id} step {iter_id + gstep_id_base} psnr={-10.0 * math.log10(float(sq.mean()) / 3):.2f}", flush=True)
            self.optimizer.check_overflow()
            self.stats.append(float(se) / batches_per_epoch)
            gstep_id_base += batches_per_epoch
            if gstep_id_base - last_upsamp_step >= args.upsamp_every:
                last_upsamp_step = gstep_id_base
                if reso_id < len(self.reso_list) - 1:
                    if args.tv_early_only > 0:
                        args.lambda_tv, args.lambda_tv_sh = 0.0, 0.0
                    elif args.tv_decay != 1.0:
                        args.lambda_tv *= args.tv_decay
                        args.lambda_tv_sh *= args.tv_decay
                    reso_id += 1
                    nxt = self.reso_list[reso_id]
                    z_reso = nxt if isinstance(nxt, int) else nxt[2]
                    self.model.resample(reso=nxt, sigma_thresh=args.density_thresh, weight_thresh=args.weight_thresh / z_reso, dilate=2,
                                        cameras=self._resample_cameras() if args.thresh_type == "weight" else None,
                                        max_elements=args.max_grid_elements)
                    self.optimizer = PlenOptimRMSprop(self.model.density_data, self.model.sh_data, 0, 0, 0.95, 0.95)
            if gstep_id_base >= args.n_iters:
                self.eval_step(epoch_id, gstep_id_base)
                self.model.save(self.ckpt_path)
                break

    # ------------------------------------------------------------------------------------------ evaluation
    @torch.no_grad()
    def eval_step(self, epoch_id, gstep_id_base):
        """runner_svox2.py:110-161: up to 5 (first epoch) or 20 views of the val set, PNGs under {gstep:09d}/; returns mse / psnr means."""
        ds = self.dataset["val"]
        n_eval = min(20 if epoch_id > 0 else 5, ds.n_images)
        img_ids = range(0, ds.n_images, ds.n_images // n_eval)
        out = os.path.join(self.save_path, f"{gstep_id_base:09d}")
        os.makedirs(out, exist_ok=True)
        stats = {"psnr": 0.0, "mse": 0.0}
        for img_id in img_ids:
            pred = self.model.volume_render_image(ds.camera(img_id))
            gt = ds.gt_image(img_id)
            self.save_img(os.path.join(out, f"image_pred_{img_id:04d}.png"), pred.clamp(max=1.0))
            self.save_img(os.path.join(out, f"image_test_{img_id:04d}.png"), gt)
            mse = float(((gt - pred) ** 2).mean())
            psnr = -10.0 * math.log10(mse)
            if math.isnan(psnr):
                raise FloatingPointError(f"NAN PSNR at image {img_id} (mse {mse})")
            stats["mse"] += mse
            stats["psnr"] += psnr
        stats = {k: v / len(img_ids) for k, v in stats.items()}
        print("eval stats:", stats, flush=True)
        return stats

    @staticmethod
    def save_img(path, img):
        from PIL import Image
        img = img.detach().cpu().numpy() if torch.is_tensor(img) else np.asarray(img)
        Image.fromarray((img * 255 + 0.5).clip(0, 255).astype(np.uint8)).save(path)

    @torch.no_grad()
    def render_img(self, dataset_mode="test", img_id=0):
        """runner_svox2.py:350-363: (prediction (H, W, 3), target (H, W, 3)) of image img_id, on the device."""
        ds = self.dataset[dataset_mode]
        return self.model.volume_render_image(ds.camera(img_id)), ds.gt_image(img_id)

    @torch.no_grad()
    def test(self, load_ckpt=False):
        """runner_svox2.py:288-336: every test view to {exp_name}_r_{i}.png / _gt_{i}.png under test/; prints and returns the mean PSNR."""
        if load_ckpt:
            assert os.path.exists(self.ckpt_path), "ckpt file does not exist: " + self.ckpt_path
            self.load_ckpt(self.ckpt_path)
        if self.dataset["test"] is None:
            self.dataset["test"] = build_from_cfg(self.cfg.dataset.test, DATASETS)
        out = os.path.join(self.save_path, "test")
        os.makedirs(out, exist_ok=True)
        psnr = []
        for i in range(self.dataset["test"].n_images):
            img, tar = self.render_img("test", i)
            self.save_img(os.path.join(out, f"{self.exp_name}_r_{i}.png"), img)
            self.save_img(os.path.join(out, f"{self.exp_name}_gt_{i}.png"), tar)
            psnr.append(float(L.mse2psnr(L.img2mse(img, tar))))
        mean = sum(psnr) / len(psnr)
        print(f"TOTAL TEST PSNR===={mean}", flush=True)
        return mean

    def render(self, *a, **k):
        raise NotImplementedError("Svox2Runner has no video task (the reference's Svox2Runner has none)")

    def extract_mesh(self, *a, **k):
        raise NotImplementedError("Svox2Runner: mesh extraction is not supported (the reference's Svox2Runner has none)")

    # ------------------------------------------------------------------------------------------ checkpoint
    def save_ckpt(self, path):
        self.model.save(path)

    def load_ckpt(self, path):
        self.model = SparseGrid.load(path)
        self.cfg.model_obj = self.model
        self.optimizer = PlenOptimRMSprop(self.model.density_data, self.model.sh_data, 0, 0, 0.95, 0.95)


def svox2_cfg(synthetic=False, **over):
    """contrib/plenoxel projects/svox2/configs/svox2_base.py key for key; `synthetic` swaps the lego scene for the procedural stand-in
    (plugin/svox2.py: SyntheticSvoxDataset)."""
    ds_type = "SyntheticSvoxDataset" if synthetic else "SvoxNeRFDataset"
    epoch_size, batch_size = 12800, 5000
    c = dict(
        exp_name="lego", log_dir="./logs", tot_train_steps=40000, background_color=[0, 0, 0], fp16=True, load_ckpt=False, ckpt_path=None,
        alpha_image=False, reso_list=[[256] * 3, [512] * 3], epoch_size=epoch_size, batch_size=batch_size,
        lr_basis=1e-06, lr_basis_begin_step=0, lr_basis_decay_steps=250000, lr_basis_delay_mult=0.01, lr_basis_delay_steps=0, lr_basis_final=1e-06,
        lr_color_bg=0.1, lr_color_bg_decay_steps=250000, lr_color_bg_delay_mult=0.01, lr_color_bg_delay_steps=0, lr_color_bg_final=5e-06,
        lr_decay=True, lr_fg_begin_step=0, lr_sh=0.01, lr_sh_decay_steps=250000, lr_sh_delay_mult=0.01, lr_sh_delay_steps=0, lr_sh_final=5e-06,
        lr_sigma=30.0, lr_sigma_bg=3.0, lr_sigma_bg_decay_steps=250000, lr_sigma_bg_delay_mult=0.01, lr_sigma_bg_delay_steps=0,
        lr_sigma_bg_final=0.003, lr_sigma_decay_steps=250000, lr_sigma_delay_mult=0.01, lr_sigma_delay_steps=15000, lr_sigma_final=0.05,
        lambda_tv=1e-05, lambda_tv_sh=0.001, tv_contiguous=1, tv_sh_sparsity=0.01, tv_logalpha=False, tv_sparsity=0.01, eval_every=1,
        print_every=20, init_sigma=0.1, init_sigma_bg=0.1, sigma_thresh=1e-08, step_size=0.5, stop_thresh=1e-07, background_brightness=1.0,
        random_sigma_std=0.0, random_sigma_std_background=0.0, last_sample_opaque=False, near_clip=0.0, use_spheric_clip=False, init_iters=0,
        enable_random=False, rms_beta=0.95, weight_decay_sh=1.0, weight_decay_sigma=1.0, upsamp_every=38400, tv_early_only=1, tv_decay=1.0,
        density_thresh=5.0, weight_thresh=0.256, thresh_type="weight", max_grid_elements=44000000, upsample_density_add=0.0, n_iters=128000,
        model=dict(type="SparseGrid", basis_dim=9, basis_reso=32, nosphereinit=False),
        dataset_type=ds_type, dataset_dir="data/lego",
        dataset=dict(train=dict(type=ds_type, root="data/lego", split="train", epoch_size=epoch_size * batch_size),
                     test=dict(type=ds_type, root="data/lego", split="test", epoch_size=epoch_size * batch_size)),
        loss=dict(type="MSELoss"),
    )
    c.update(over)
    return c
