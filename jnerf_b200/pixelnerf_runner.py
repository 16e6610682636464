"""PixelNeRFRunner: the reference's contrib/pixelnerf main.py (training), test_utils.py (video) on csrc/pixelnerf.cu.  DESIGN.md section 13.

One training step: 2048 shuffled rays of the reference views -> one jitter vector z (S,) for the whole batch (Render.py:22-26) -> the fused
forward (projection, gather, network) -> MSE and d(raw) in one launch, carried scaled by R so fp16 does not underflow -> the fused backward
-> Adam (ngp_adam_ema with ema_decay = 0) takes the gradient back by 1 / R."""
import os

import numpy as np
import torch

from . import ops
from .plugin import losses as L
from .plugin import pixelnerf as pn
from .utils.config import get_cfg


def pixelnerf_cfg(data_path=None, **over):
    """main.py:12-34 key for key; data_path: tiny_nerf_data.npz (main.py:16's ./tiny_nerf_data.npz by default)."""
    c = dict(data_path=data_path or "./tiny_nerf_data.npz", n_train=3, batch_size=2048, bound=(2., 6.), N_samples=(64, None), epoch=100,
             img_f_ch=512, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, seed=999, noise_std=0., pixel_aligned=False,
             encoder_weights=None, log_dir="./logs", exp_name="pixelnerf", ckpt_path=None)
    c.update(over)
    return c


class PixelNeRFRunner:
    def __init__(self, rank=0, world_size=1, process_group=None):
        if world_size > 1:
            raise NotImplementedError("PixelNeRFRunner: data-parallel training is not supported")
        self.cfg = cfg = get_cfg()
        if float(cfg.noise_std or 0) > 0:
            raise NotImplementedError("PixelNeRFRunner: noise_std > 0 (density noise) is not supported")
        if cfg.N_samples[1] is not None:
            raise NotImplementedError("PixelNeRFRunner: a fine sampling level (N_samples[1]) is not supported")
        if int(cfg.img_f_ch) != 512:
            raise NotImplementedError("PixelNeRFRunner: img_f_ch must be 512 (the encoder's channels)")
        self.device = "cuda"
        self.data = pn.TinyNerfData(cfg.data_path, cfg.n_train, self.device)
        enc_w = cfg.encoder_weights
        if isinstance(enc_w, str):
            enc_w = torch.load(enc_w, map_location="cpu", weights_only=True)
        self.encoder_label = "given resnet34 weights" if enc_w is not None else "seeded He-initialised resnet34"
        enc = pn.ImageEncoder(enc_w, seed=int(cfg.seed))
        n = self.data.n_train
        self.ref = pn.ReferenceViews(self.data.images[:n], self.data.poses[:n], self.data.focal, enc, self.device, bool(cfg.pixel_aligned))
        self.model = pn.PixelNeRF(seed=int(cfg.seed), device=self.device)
        self.S = int(cfg.N_samples[0])
        self.near, self.far = map(float, cfg.bound)
        self.gen = torch.Generator(device=self.device).manual_seed(int(cfg.seed))
        self.step = 0
        self._saved = None

    def _z(self, randomized=True):
        """Render.py:22-26: near + (far - near) (linspace(0, 1, S + 1)[:-1] + rand(S) / S), one vector for every ray."""
        S = self.S
        k = torch.rand(S, generator=self.gen, device=self.device) / S if randomized else torch.full((S,), 0.5 / S, device=self.device)
        return self.near + (self.far - self.near) * (torch.linspace(0.0, 1.0, S + 1, device=self.device)[:-1] + k)

    def _fwd(self, rays, z, saved=None):
        r = self.ref
        return ops.pixelnerf_fwd(rays, z, self.model.params, r.feats, r.cams, r.scale, r.pixel_aligned, saved=saved)

    def train_step(self, batch):
        """main.py:42-46 on one batch (R, 9); returns the loss (device scalar)."""
        cfg, m = self.cfg, self.model
        rays, target = batch[:, :6].contiguous(), batch[:, 6:9].contiguous()
        R = rays.shape[0]
        z = self._z()
        need = ops.pixelnerf_workspace_bytes(R * self.S, self.ref.feats.shape[0])[0]
        if self._saved is None or self._saved.numel() < need:
            self._saved = torch.empty(need, dtype=torch.uint8, device=self.device)
        raw = self._fwd(rays, z, self._saved)
        _, loss, draw = ops.pixelnerf_composite_loss_bwd(raw, z, rays, target, grad_scale=float(R))
        grad = ops.pixelnerf_bwd(R, self.S, m.params, self.ref.feats, self._saved, raw, draw)
        self.step += 1
        ops.adam_ema(m.params, grad, m.m, m.v, m.master, float(cfg.lr), self.step, cfg.betas[0], cfg.betas[1], float(cfg.eps), 0.0,
                     grad_scale=1.0 / R, zero_grad=False)
        return loss.sum()

    def train(self, epochs=None, steps=None, log_every=0):
        """main.py:37-49: epochs of shuffled drop_last batches; steps: stop after that many steps."""
        epochs = int(self.cfg.epoch) if epochs is None else epochs
        done = 0
        for e in range(epochs):
            for batch in self.data.batches(int(self.cfg.batch_size), self.gen):
                loss = self.train_step(batch)
                done += 1
                if log_every and self.step % log_every == 0:
                    print(f"EPOCH={e + 1} STEP={self.step} | LOSS={loss.item():.6f}", flush=True)
                if steps is not None and done >= steps:
                    return

    # ------------------------------------------------------------------------------------------ evaluation
    @torch.no_grad()
    def render_rays(self, rays, chunk=4096):
        """(rgb (R, 3), depth (R,), acc (R,)) at the mid-interval depths, in chunks of rays."""
        z = self._z(randomized=False)
        outs = []
        for p in range(0, rays.shape[0], chunk):
            r = rays[p:p + chunk].contiguous()
            outs.append(ops.pixelnerf_composite_fwd(self._fwd(r, z), z, r))
        return tuple(torch.cat(o) for o in zip(*outs))

    @torch.no_grad()
    def render_img_with_pose(self, c2w):
        """test_utils.py:41-51 as one call: the whole H x W frame (H, W, 3) of camera c2w."""
        rgb = self.render_rays(self.data.image_rays(c2w))[0]
        return rgb.reshape(self.data.H, self.data.W, 3)

    def render(self, save_path=None, r=5.0):
        """test_utils.py:27-38: 120 frames wobbling +-r degrees about reference view 0, 30 fps mp4 (OpenCV).  Returns the path."""
        try:
            import cv2
        except ImportError as e:
            raise RuntimeError("PixelNeRFRunner.render writes the video with OpenCV: install opencv-python (cv2) to use it") from e
        save_path = save_path or os.path.join(self._save_path(), "video.mp4")
        os.makedirs(os.path.dirname(os.path.abspath(save_path)), exist_ok=True)
        H, W = self.data.H, self.data.W
        writer = cv2.VideoWriter(str(save_path), cv2.VideoWriter_fourcc(*"mp4v"), 30, (W, H))
        try:
            for pose in video_poses(self.ref.c2w[0], r):
                img = (255 * self.render_img_with_pose(pose).clamp(0, 1)).byte().cpu().numpy()
                writer.write(img[..., ::-1].copy())
        finally:
            writer.release()
        return save_path

    def _save_path(self):
        return os.path.join(self.cfg.log_dir or ".", self.cfg.exp_name or "pixelnerf")

    @torch.no_grad()
    def test(self, save_dir=None):
        """Every view that is not a reference view: PNGs of the render and the target, and the mean PSNR (printed and returned)."""
        from PIL import Image
        out = save_dir or os.path.join(self._save_path(), "test")
        os.makedirs(out, exist_ok=True)
        psnr = []
        for i in range(self.data.n_train, self.data.images.shape[0]):
            img = self.render_img_with_pose(self.data.poses[i])
            tar = torch.from_numpy(self.data.images[i]).to(img.device)
            for name, a in ((f"r_{i}.png", img), (f"gt_{i}.png", tar)):
                Image.fromarray((a.clamp(0, 1).cpu().numpy() * 255 + 0.5).astype(np.uint8)).save(os.path.join(out, name))
            psnr.append(float(L.mse2psnr(L.img2mse(img, tar)).item()))
        mean = sum(psnr) / len(psnr)
        print(f"TEST PSNR ({self.encoder_label}, pixel_aligned={self.ref.pixel_aligned})===={mean}", flush=True)
        return mean

    def extract_mesh(self, *a, **k):
        raise NotImplementedError("PixelNeRFRunner: mesh extraction is not supported")

    # ------------------------------------------------------------------------------------------ checkpoint
    def save_ckpt(self, path):
        """A .pth state dict of fp32 tensors under the reference's names (what main.py:35's net.load reads)."""
        if str(path).endswith(".pkl"):
            raise NotImplementedError("PixelNeRFRunner: the .pkl interchange format is not supported; save to a .pth path")
        torch.save({k: v.cpu() for k, v in self.model.reference_state().items()}, path)

    def load_ckpt(self, path):
        if str(path).endswith(".pkl"):
            raise NotImplementedError("PixelNeRFRunner: the .pkl interchange format is not supported; load a .pth state dict")
        self.model.load_reference_state(torch.load(path, map_location="cpu", weights_only=True))


def video_poses(c2w0, r=5.0):
    """test_utils.py:9-35: the 120 camera-to-world matrices of the video around c2w0."""
    def rot_phi(phi):
        return np.array([[1, 0, 0, 0], [0, np.cos(phi), -np.sin(phi), 0], [0, np.sin(phi), np.cos(phi), 0], [0, 0, 0, 1]], dtype=np.float32)

    def rot_theta(th):
        return np.array([[np.cos(th), 0, -np.sin(th), 0], [0, 1, 0, 0], [np.sin(th), 0, np.cos(th), 0], [0, 0, 0, 1]], dtype=np.float32)
    out = []
    for th in np.linspace(-1.0, 1.0, 120, endpoint=False):
        theta = rot_theta(r * np.sin(np.pi * 2.0 * th) / 180.0 * np.pi)
        phi = rot_phi(r * np.cos(np.pi * 2.0 * th) / 180.0 * np.pi)
        out.append(theta @ phi @ np.asarray(c2w0, np.float32))
    return out
