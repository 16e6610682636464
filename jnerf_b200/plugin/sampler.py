"""DensityGridSampler (+ RaySampler, CompactedCoord, CalcRgb): mirror of
models/samplers/density_grid_sampler/{density_grid_sampler,ray_sampler,compacted_coord,calc_rgb}.py.

Differences that are visible only as speed (results are identical, see DESIGN.md):
  * the dead no-grad network pass before compaction (density_grid_sampler.py:151-158) is not run -- its output
    cannot influence compacted_coord's result because the transmittance early-out is commented out in the reference
    (compacted_coord.h:40-43);
  * the march emits rays in ray order, so "compaction" is bookkeeping only (no 117 MB memset, no copy, no host sync).
The process-global `jittor::rng` (pcg32{1337}, ops/code_ops/global_vars.py) is the `rng` attribute here."""
import math

import numpy as np
import torch

from .. import ops
from ..utils.config import get_cfg
from ..utils.registry import SAMPLERS
from .module import Module


class _CalcRgbFn(torch.autograd.Function):
    """CalcRgb.execute / .grad (DGS/calc_rgb.py:31-108)."""

    @staticmethod
    def forward(ctx, network_output, coords, numsteps, numsteps_compacted, bg, mean, cascades):
        network_output = network_output.contiguous()
        rgb = ops.composite_fwd(network_output, coords, numsteps, numsteps_compacted, bg, cascades)
        ctx.save_for_backward(network_output, coords, numsteps_compacted, rgb, mean)
        ctx.cascades = cascades
        return rgb

    @staticmethod
    def backward(ctx, grad_x):
        net, coords, ns_c, rgb, mean = ctx.saved_tensors
        dnet = ops.composite_bwd(net, coords, ns_c, grad_x.contiguous(), rgb, mean, ctx.cascades)
        return dnet, None, None, None, None, None, None


@SAMPLERS.register_module()
class DensityGridSampler(Module):
    def __init__(self, update_den_freq=16, update_block_size=5000000):
        super().__init__()
        self.cfg = get_cfg()
        self.model = self.cfg.model_obj
        self.dataset = self.cfg.dataset_obj
        self.update_den_freq = update_den_freq
        self.update_block_size = update_block_size
        self.n_rays_per_batch = self.cfg.n_rays_per_batch
        self.cone_angle_constant = self.cfg.cone_angle_constant
        self.using_fp16 = bool(self.cfg.fp16)
        self.near_distance = self.cfg.near_distance
        self.n_training_steps = self.cfg.n_training_steps
        self.target_batch_size = self.cfg.target_batch_size
        self.const_dt = bool(self.cfg.const_dt)
        self.NERF_CASCADES = 5
        self.NERF_GRIDSIZE = 128
        self.NERF_MIN_OPTICAL_THICKNESS = 0.01
        self.MAX_STEP = 1024
        self.background_color = self.cfg.background_color
        self.n_images = self.dataset.n_images
        self.image_resolutions = self.dataset.resolution
        self.aabb_range = self.dataset.aabb_range
        max_aabb_scale = 1 << (self.NERF_CASCADES - 1)
        if self.dataset.aabb_scale > max_aabb_scale:
            self.NERF_CASCADES = math.ceil(math.log2(self.dataset.aabb_scale)) + 1
        self.max_cascade = 0
        while (1 << self.max_cascade) < self.dataset.aabb_scale:
            self.max_cascade += 1
        dev = "cuda"
        G3 = self.NERF_GRIDSIZE ** 3
        self.density_grid_decay = 0.95
        self.density_n_elements = self.NERF_CASCADES * G3
        self.density_grid = torch.zeros(self.density_n_elements, dtype=torch.float32, device=dev)
        self.density_grid_tmp = torch.zeros(self.density_n_elements, dtype=torch.float32, device=dev)
        self.density_grid_bitfield = torch.zeros(self.density_n_elements // 8, dtype=torch.uint8, device=dev)
        self.density_grid_mean = torch.zeros(1, dtype=torch.float32, device=dev)
        self.density_grid_ema_step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.measured_batch_size = torch.zeros(1, dtype=torch.int32, device=dev)
        self.rng = ops.pcg32_seed(1337)                              # jittor::rng, global_vars.py:17
        self.max_samples = self.cfg.n_rays_per_batch * self.MAX_STEP  # raw sample capacity, ray_sampler.py:15,30
        self._coords_raw = torch.zeros((self.max_samples, 7), dtype=torch.float32, device=dev)
        # march workspace (per-ray chunk records, ~23 KB a ray): sized for the current ray batch with head room and re-grown when the
        # adaptive ray batch (density_grid_sampler.py:266-271) outgrows it -- that only happens at the 16-step host sync
        self._march_ws_rays = 0
        self._march_ws = None
        self._ensure_march_ws(max(2 * self.n_rays_per_batch, 8192))
        self.dp_group = None                                         # (process_group, world_size) when data parallel
        self._coords = None
        self._rays_numsteps = None
        self._rays_numsteps_compacted = None
        self._counters_compacted = None

    def _ensure_march_ws(self, n_rays):
        if n_rays > self._march_ws_rays:
            self._march_ws = None                                      # release before the larger allocation
            self._march_ws_rays = int(n_rays)
            self._march_ws = torch.empty(int(ops.lib.load().ngp_march_workspace_bytes(self._march_ws_rays)) + 16, dtype=torch.uint8, device="cuda")

    # ---- R6 + R5 -------------------------------------------------------------------------------------------
    def sample(self, img_ids, rays_o, rays_d, rgb_target=None, is_training=False, ray_index_offset=0):
        """ray_index_offset: index of rays_o[0] in the global (all-rank) ray batch -- the per-ray jitter stream is indexed by the
        global ray id so that a data-parallel shard reproduces the single-GPU samples (ray_sampler.h:30)."""
        if is_training:
            if self.cfg.m_training_step % self.update_den_freq == 0:
                self.update_density_grid()
            self._rays_numsteps, self._rays_numsteps_compacted, self._counters_compacted, self._coords = self.sample_front(
                rays_o, rays_d, self._coords_raw, ray_index_offset)
            if self.cfg.m_training_step % self.update_den_freq == self.update_den_freq - 1:
                self.update_batch_rays()
            return self._coords[:, :3], self._coords[:, 4:]
        if rays_o.shape[0] > self._march_ws_rays:
            self._ensure_march_ws(2 * rays_o.shape[0])
        coords, rays_index, rays_numsteps, counters = ops.march(
            rays_o.contiguous(), rays_d.contiguous(), self.density_grid_bitfield, self.aabb_range, self.max_samples, self.cone_angle_constant,
            self.near_distance, self.NERF_CASCADES, self.const_dt,
            ops.pcg32_advance(self.rng.copy(), ray_index_offset * 8) if ray_index_offset else self.rng, coords=self._coords_raw, workspace=self._march_ws)
        ops.pcg32_advance(self.rng)                                    # rng.advance(), ray_sampler.py:61
        self._rays_numsteps = rays_numsteps
        samples = int(counters[1].item())                              # ray_sampler.py:70 (inference only here)
        samples = min(samples, self.max_samples)
        self._coords = coords[:samples]
        self._rays_numsteps_compacted = rays_numsteps
        return self._coords[:, :3], self._coords[:, 4:]

    def sample_front(self, rays_o, rays_d, coords_raw, ray_index_offset=0):
        """Training-mode march + compaction into a caller-owned coordinate buffer, returning the step's bookkeeping
        (rays_numsteps, rays_numsteps_compacted, counters_compacted, coords) instead of keeping it on the sampler: the runner's
        software pipeline runs this for step i+1 (on a second stream) while step i still reads its own rows; sample() keeps it.
        The caller runs the occupancy-grid update and the ray-batch adaptation around it."""
        if rays_o.shape[0] > self._march_ws_rays:
            self._ensure_march_ws(2 * rays_o.shape[0])
        coords, _, rays_numsteps, _ = ops.march(rays_o.contiguous(), rays_d.contiguous(), self.density_grid_bitfield, self.aabb_range,
                                                self.max_samples, self.cone_angle_constant, self.near_distance, self.NERF_CASCADES,
                                                self.const_dt,
                                                ops.pcg32_advance(self.rng.copy(), ray_index_offset * 8) if ray_index_offset else self.rng,
                                                coords=coords_raw, workspace=self._march_ws)
        ops.pcg32_advance(self.rng)                                    # rng.advance(), ray_sampler.py:61
        cap = self.target_batch_size
        _, ns_c, cnt_c = ops.compact(coords, rays_numsteps, cap, alias=True)
        self.measured_batch_size += cnt_c[0:1]
        return rays_numsteps, ns_c, cnt_c, coords[:cap]

    @property
    def coords_compacted(self):
        """(target_batch_size, 7) NerfCoordinate rows of the last training sample() -- input of the fused network path."""
        return self._coords

    @property
    def n_samples_dev(self):
        """device uint32[1]: number of live rows in coords_compacted (may exceed the capacity; consumers clamp)."""
        return self._counters_compacted[0:1]

    # ---- R8 / R9 -------------------------------------------------------------------------------------------
    def rays2rgb(self, network_outputs, training_background_color=None, inference=False):
        assert network_outputs.shape[0] == self._coords.shape[0]
        if inference:
            return ops.composite_infer(network_outputs.contiguous(), self._coords, self._rays_numsteps, self.NERF_CASCADES)
        bg = training_background_color
        if bg is None:
            bg = torch.tensor(self.background_color, dtype=torch.float32, device="cuda").expand(self._rays_numsteps.shape[0], 3).contiguous()
        return _CalcRgbFn.apply(network_outputs, self._coords, self._rays_numsteps, self._rays_numsteps_compacted, bg.contiguous(),
                                self.density_grid_mean, self.NERF_CASCADES)

    # ---- R10 -----------------------------------------------------------------------------------------------
    def update_density_grid_nerf(self, decay, n_uniform, n_nonuniform):
        if self.cfg.m_training_step == 0:
            self.density_grid.zero_()
            if getattr(self.dataset, "frame_cameras", False):
                # frames with their own cameras: every image's own signed frustum, whatever its size, principal point and lens
                ops.grid_mark_untrained_cams(self.density_grid, self.dataset.frame_extents, self.dataset.transforms_gpu)
            else:
                # through a lens the images see further out than a pinhole of the same focal length: the dataset's effective focal lengths
                focal = getattr(self.dataset, "focal_eff", None)
                ops.grid_mark_untrained(self.density_grid, self.dataset.focal_lengths if focal is None else focal, self.dataset.transforms_gpu,
                                        self.image_resolutions)
        self.density_grid_tmp.zero_()
        parts_p, parts_i = [], []
        for n, thresh in ((n_uniform, -0.01), (n_nonuniform, self.NERF_MIN_OPTICAL_THICKNESS)):
            if n == 0:
                continue                                               # zero-sized jt.code op: body (and rng.advance) not run -- SURVEY H5
            p, i = ops.grid_generate_samples(n, self.rng, self.density_grid_ema_step, self.aabb_range, self.density_grid, self.max_cascade + 1, thresh)
            ops.pcg32_advance(self.rng)                                # generate_grid_samples_nerf_nonuniform.py:44
            parts_p.append(p)
            parts_i.append(i)
        pos = torch.cat(parts_p) if len(parts_p) > 1 else parts_p[0]
        idx = torch.cat(parts_i) if len(parts_i) > 1 else parts_i[0]
        with torch.no_grad():
            bs = self.update_block_size
            res = [self.model.density(pos[i:i + bs]) for i in range(0, pos.shape[0], bs)]
            mlp_out = (torch.cat(res, 0) if len(res) > 1 else res[0]).reshape(-1).contiguous()
        ops.grid_splat(idx, mlp_out, self.density_grid_tmp)
        ops.grid_ema(self.density_grid, self.density_grid_tmp, decay)
        self.density_grid_ema_step += 1
        ops.grid_update_bitfield(self.density_grid, self.density_grid_mean, self.density_grid_bitfield, self.NERF_CASCADES)

    def update_density_grid(self):
        G3 = self.NERF_GRIDSIZE ** 3
        n_cascades = self.max_cascade + 1
        # note: the reference computes alpha = decay ** (n_training_steps/16) but its ema op uses the constructor's 0.95
        if self.cfg.m_training_step < 256:
            self.update_density_grid_nerf(self.density_grid_decay, G3 * n_cascades, 0)
        else:
            self.update_density_grid_nerf(self.density_grid_decay, G3 * n_cascades // 4, G3 * n_cascades // 4)

    def update_batch_rays(self, measured_total=None):
        """measured_total: the (global) sample count of the 16 steps when the caller has read the counter back itself (the runner's
        software pipeline does, on its side stream, so that the host does not wait for the step in flight)."""
        from .. import dp
        W = 1
        if measured_total is not None:
            W = self.dp_group[1] if self.dp_group is not None else 1
            self.n_rays_per_batch = max(dp.adapt_rays_per_batch(self.n_rays_per_batch * W, measured_total / 16, self.target_batch_size * W) // W, 1)
            self.dataset.batch_size = self.n_rays_per_batch
            return
        if self.dp_group is not None:
            # data parallel: the GLOBAL ray batch adapts to the GLOBAL sample budget, exactly as one GPU training on the global batch
            # would (same rounding to 128 rays), and every rank takes 1/W of it -- adapting each rank's shard on its own rounds to
            # 128 rays PER RANK and the two runs part ways at the first adaptation (tools/dp_check.py)
            W = self.dp_group[1]
            dp.global_sum_count(self.measured_batch_size, self.dp_group[0], W)
        measured = self.measured_batch_size.item() / 16                # the one host sync per 16 steps (density_grid_sampler.py:266-271)
        self.n_rays_per_batch = max(dp.adapt_rays_per_batch(self.n_rays_per_batch * W, measured, self.target_batch_size * W) // W, 1)
        self.measured_batch_size.zero_()
        self.dataset.batch_size = self.n_rays_per_batch

    def state_dict(self, *args, **kwargs):
        return {"density_grid": self.density_grid, "density_grid_bitfield": self.density_grid_bitfield, "density_grid_mean": self.density_grid_mean,
                "density_grid_ema_step": self.density_grid_ema_step, "n_rays_per_batch": self.n_rays_per_batch,
                "rng": torch.from_numpy(self.rng.astype(np.int64))}

    def load_state_dict(self, sd, *args, **kwargs):
        for k in ("density_grid", "density_grid_bitfield", "density_grid_mean", "density_grid_ema_step"):
            getattr(self, k).copy_(sd[k])
        # the two entries below are not jt.Vars in the reference and hence absent from its params.pkl (utils/ckpt_compat.py)
        if "n_rays_per_batch" in sd:
            self.n_rays_per_batch = int(sd["n_rays_per_batch"])
            self.dataset.batch_size = self.n_rays_per_batch
        if "rng" in sd:
            self.rng = sd["rng"].cpu().numpy().astype(np.uint64)
