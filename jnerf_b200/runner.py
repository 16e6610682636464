"""Thin training / evaluation driver: the caller of the hot path, mirroring runner/runner.py:14-264 step for step
(SURVEY.md section 3.1).  `train_step` is the fast path: no autograd graph, no host sync (except the
reference's own batch-size adaptation every 16 steps), one C-ABI call per stage:

    [grid update /16] -> raygen -> march -> (compaction bookkeeping) -> fused network fwd ->
    fused composite + Huber + composite bwd -> fused network bwd -> [NCCL all-reduce] -> fused Adam+EMA

The steps are software-pipelined: raygen + march of step i+1 are enqueued on a second stream as soon as step i starts, and run beside
its network kernels and Adam+EMA sweep (`_train_step_pipe`; NGP_PIPELINE=0 restores the strictly sequential step).  Both schedules run
the same pieces: `_batch` (background colours + ray batch), the sampler's march, `_net_pass` (network forward, composite + loss + its
backward, network backward) and the optimizer tail.

`train_step_autograd` runs the same step through the per-operator plugin classes and torch autograd, exactly as
JNeRF's Runner.train does with Jittor; tests check that both give the same parameters."""
import contextlib
import os

import numpy as np
import torch

from . import dp, ops
from .plugin import losses as L
from .utils.config import get_cfg
from .utils.registry import DATASETS, LOSSES, NETWORKS, OPTIMS, SAMPLERS, build_from_cfg


class Runner:
    def __init__(self, rank=0, world_size=1, process_group=None):
        self.cfg = get_cfg()
        cfg = self.cfg
        self.rank, self.world_size, self.pg = rank, world_size, process_group
        self.dataset = {"train": build_from_cfg(cfg.dataset.train, DATASETS)}
        cfg.dataset_obj = self.dataset["train"]
        self.dataset["val"] = build_from_cfg(cfg.dataset.val, DATASETS) if cfg.dataset.val else self.dataset["train"]
        self.dataset["test"] = None
        self.model = build_from_cfg(cfg.model, NETWORKS)
        cfg.model_obj = self.model
        self.sampler = build_from_cfg(cfg.sampler, SAMPLERS)
        cfg.sampler_obj = self.sampler
        if world_size > 1:
            self.sampler.dp_group = (process_group, world_size)
        params = list(self.model.parameters())
        self.optimizer = build_from_cfg(cfg.optim, OPTIMS, params=params)
        self.optimizer = build_from_cfg(cfg.expdecay, OPTIMS, nested_optimizer=self.optimizer)
        self.ema_optimizer = build_from_cfg(cfg.ema, OPTIMS, params=params)
        self.ema_optimizer.attach(self.optimizer)
        self.loss_func = build_from_cfg(cfg.loss, LOSSES)
        self.background_color = cfg.background_color
        self.tot_train_steps = cfg.tot_train_steps
        self.n_rays_per_batch = cfg.n_rays_per_batch
        self.W, self.H = self.dataset["train"].resolution
        self.start = 0
        cfg.m_training_step = 0
        self.val_freq = 4096
        self.fast = bool(getattr(self.model, "fused", False))
        # the march / network / composite renderers drive the fused NGP kernels or a model with its own inference forward (infer)
        self._can_infer = self.fast or hasattr(self.model, "infer")
        # state the evaluation / checkpoint code reads on EVERY kind of model (fused or the nn.Linear fallback)
        self._table_work, self._pending_epoch = None, None
        self._host_stage = None
        self._render_ws = None                                       # workspace of the whole-frame renderer (render_rays)
        self._pipe = None                                            # march of step i+1 beside step i (software pipeline over steps)
        self._st = {id(s.p): s for s in self.optimizer._nested_optimizer.state}
        if world_size > 1 and not self.fast:
            raise ValueError("data-parallel training needs the fused model (fp16=True, use_fully=True): the per-operator autograd step "
                             "shards the ray batch but has no gradient exchange, the replicas would silently diverge")
        if self.fast:
            self._init_fast_path()
        self._bg_gen = torch.Generator(device="cuda").manual_seed(int(cfg.seed or 1) + 7)

    # ------------------------------------------------------------------------------------------ fast path
    def _init_fast_path(self):
        dev = "cuda"
        m = self.model
        cap = self.sampler.target_batch_size
        self.grid_grad = torch.zeros(m.pos_encoder.m_grid.numel(), dtype=torch.float16, device=dev)
        n_w = m.density_mlp.con_weights.numel() + m.rgb_mlp.con_weights.numel()
        # [dW density | dW colour | measured-sample counter]: one flat fp32 buffer = one small all-reduce
        self.w_grad = torch.zeros(n_w + 8, dtype=torch.float32, device=dev)
        self.dwd = self.w_grad[:m.density_mlp.con_weights.numel()]
        self.dwr = self.w_grad[m.density_mlp.con_weights.numel():n_w]
        self.net_out = torch.zeros((cap, 4), dtype=torch.float16, device=dev)
        self.enc = torch.empty((cap, 32), dtype=torch.float16, device=dev)
        self.dnet = torch.zeros((cap, 4), dtype=torch.float16, device=dev)
        self.last_loss = None
        self.last_rgb = None
        # One GPU: the backward leaves its gradients in caller-owned scratch (fixed-point table gradient, per-CTA weight-gradient slots)
        # and ONE sweep turns them into the optimizer step of all three tensors (ops.train_sweep, same bits as the backward's own
        # reduction + three adam_ema sweeps, about 80 MB less traffic a step).  Only with the library's own network_bwd: a stand-in
        # operator layer keeps the per-tensor calls.  Data parallelism exchanges the fp16 table gradient and keeps them too.
        self._fx = self._w_part = None
        if self.world_size == 1 and ops.network_bwd is ops._network_bwd:
            self._fx, self._w_part = ops.network_bwd_scratch(m.pos_encoder.levels, device=dev)
        # Software pipeline over steps (default): nothing the march reads is written by the network kernels -- rays, jitter and the
        # occupancy bitfield only -- so the "front" of step i+1 (background colours, ray generation, march, compaction) is enqueued
        # on a second stream while step i's network kernels / Adam+EMA sweep still run.  The sweep is HBM-bound and the march is
        # latency-bound: side by side they share the SMs instead of queueing.  The front of step i+1 may start as soon as step i does
        # (`at` = "front"): starting it after step i's forward or backward was measured slower on the H100 (DESIGN.md section 5).
        if os.environ.get("NGP_PIPELINE", "1") == "1":
            # both coordinate buffers are allocated (and zero-filled) HERE, on the constructor's stream: a fill enqueued lazily from inside
            # a step would land on the main stream behind that step's kernels and wipe what the side stream's march had just written
            raw = self.sampler._coords_raw
            self._pipe = dict(stream=torch.cuda.Stream(), coords=[torch.zeros_like(raw), torch.zeros_like(raw)], made=0, pending=None, at="front",
                              mid=torch.cuda.Event(), back_done=[torch.cuda.Event(), torch.cuda.Event()], prefetched=0, aux=torch.cuda.Stream(),
                              aux_done=torch.cuda.Event(), main=None)
        if self.world_size > 1:
            self._init_sharded_table()

    def _init_sharded_table(self):
        """Sharded optimizer for the hash table (dp.py header): this rank owns slice [lo, hi) of the padded table.
        Exchange mode (env NGP_DP_EXCHANGE = auto | p2p | nccl):
          p2p  -- ONE kernel per step over NVLink peer memory (ngp_dp_exchange_step): pull-reduce the peers' gradient slices,
                  Adam+EMA on the slice, push the fp16 slice into every peer's table, all-reduce + update the MLP weights;
          nccl -- reduce-scatter -> Adam+EMA on the slice -> async all-gather, + all-reduce of the MLP weight gradients.
        Either way the table of the next step is awaited only after the march (which does not read it)."""
        import os
        g = self.model.pos_encoder.m_grid
        m = self.model
        n, W = g.numel(), self.world_size
        mode = os.environ.get("NGP_DP_EXCHANGE", "auto")
        assert mode in ("auto", "p2p", "nccl")
        self.dp_mode = "p2p" if mode == "p2p" or (mode == "auto" and dp.peer_exchange_available(W)) else "nccl"
        P = dp.padded_len(n, W)
        nd, nr = m.density_mlp.con_weights.numel(), m.rgb_mlp.con_weights.numel()
        if self.dp_mode == "p2p":
            try:
                self._arena = dp.PeerArena(n, nd + nr, W, self.rank, self.pg)
            except RuntimeError as e:                                  # raised on EVERY rank when any mapping failed
                if mode == "p2p":
                    raise
                if self.rank == 0:
                    print(f"[jnerf_b200] peer-memory exchange unavailable ({e}); using the NCCL exchange", flush=True)
                self.dp_mode = "nccl"
        if self.dp_mode == "p2p":
            self._table, self._table_grad, self.w_grad = self._arena.table, self._arena.table_grad, self._arena.w_grad
            self.dwd, self.dwr = self.w_grad[:nd], self.w_grad[nd:nd + nr]
            self._peers = {k: self._arena.peers(k) for k in ("table", "table_grad", "w_grad", "flags")}
            # the two MLP weight tensors and their optimizer state become views of flat buffers (one sweep inside the kernel)
            self._w_param = torch.cat([m.density_mlp.con_weights.data.reshape(-1), m.rgb_mlp.con_weights.data.reshape(-1)]).contiguous()
            m.density_mlp.con_weights.data = self._w_param[:nd].view_as(m.density_mlp.con_weights.data)
            m.rgb_mlp.con_weights.data = self._w_param[nd:].view_as(m.rgb_mlp.con_weights.data)
            std, str_ = self._st[id(m.density_mlp.con_weights)], self._st[id(m.rgb_mlp.con_weights)]
            self._w_m, self._w_v = torch.cat([std.m, str_.m]), torch.cat([std.v, str_.v])
            self._w_master = torch.cat([std.master, str_.master])
            for st, lo_, hi_ in ((std, 0, nd), (str_, nd, nd + nr)):
                st.m, st.v, st.master = self._w_m[lo_:hi_], self._w_v[lo_:hi_], self._w_master[lo_:hi_]
            self._epoch, self._pending_epoch = 0, None
        else:
            self._table = torch.zeros(P, dtype=g.dtype, device=g.device)
            self._table_grad = torch.zeros(P, dtype=self.grid_grad.dtype, device=g.device)
        self._table[:n].copy_(g.data.reshape(-1))
        g.data = self._table[:n]                                   # the live parameter is a view of the padded table
        self.grid_grad = self._table_grad[:n]
        self._lo, self._hi = dp.slice_bounds(P, W, self.rank)
        self._slice_grad = torch.empty(self._hi - self._lo, dtype=self.grid_grad.dtype, device=g.device)
        self._slice_param = self._table[self._lo:self._hi].clone()
        st = self._st[id(g)]
        master = torch.zeros(P, dtype=torch.float32, device=g.device)
        master[:n].copy_(st.master)
        st.master = master[self._lo:self._hi].clone()
        st.m = torch.zeros(self._hi - self._lo, dtype=torch.float32, device=g.device)
        st.v = torch.zeros_like(st.m)

    def _table_ready(self, zero_on=None):
        """Make the current stream wait for the in-flight all-gather of the updated table (no-op on one GPU).
        zero_on: (stream, event) -- clear the gradient buffers on that stream instead of the current one and record the event; the
        caller waits for it before its backward.  The 25 MB memset then runs beside the network forward (which does not touch the
        gradients) instead of in front of it."""
        if self._table_work is not None:
            self._table_work.wait()
            self._table_work = None
        if getattr(self, "_pending_epoch", None) is not None:
            ops.dp_exchange_wait(self.world_size, self._arena.flags, self._pending_epoch)
            self._pending_epoch = None
            # peers no longer read the gradients: clear table + MLP gradients in one memset
            if zero_on is None:
                self._arena.grads.zero_()
                return False
            stream, ev = zero_on
            ev.record(torch.cuda.current_stream())                   # behind the wait kernel
            stream.wait_event(ev)
            with torch.cuda.stream(stream):
                self._arena.grads.zero_()
                ev.record(stream)
            return True
        return False

    def _gather_table_state(self):
        """Full-length (m, v, master) of the hash table for checkpoints: all-gather of the per-rank slices."""
        g = self.model.pos_encoder.m_grid
        st, n = self._st[id(g)], g.numel()
        out = []
        for t in (st.m, st.v, st.master):
            full = torch.empty(self._table.numel(), dtype=torch.float32, device=g.device)
            dp.all_gather_slices(full, t, self.pg, self.world_size)
            out.append(full[:n].clone())
        return out

    def _scatter_table_state(self, m, v, master):
        g = self.model.pos_encoder.m_grid
        st, n = self._st[id(g)], g.numel()
        for dst, src in ((st.m, m), (st.v, v), (st.master, master)):
            full = torch.zeros(self._table.numel(), dtype=torch.float32, device=g.device)
            full[:n].copy_(src.reshape(-1))
            dst.copy_(full[self._lo:self._hi])

    def next_batch(self):
        """Global pixel batch of this step (identical on every rank), sharded contiguously by rank (SURVEY 8e)."""
        ds = self.dataset["train"]
        n = self.sampler.n_rays_per_batch                       # per-rank rays; the global batch is world_size x n (weak scaling)
        pix = ds.next_pixels(n * self.world_size)
        if self.world_size > 1:
            pix = pix[self.rank * n:(self.rank + 1) * n]
        img_ids, rays_o, rays_d = ds.rays_for(pix)
        return img_ids, rays_o, rays_d, ds.rgba_for(pix)

    def _batch(self, batch):
        """(img_ids, rays_o, rays_d, bg, target) of this rank's rays of the step: the next device-generated pixel batch (batch None)
        or a fed (img_ids, rays_o, rays_d, rgba) batch.  The background colours are drawn for the global batch and this rank takes its
        rows, so the generator stays in step across ranks (runner.py:66)."""
        ds, W = self.dataset["train"], self.world_size
        if batch is None:
            R = self.sampler.n_rays_per_batch                        # per-rank rays; the global batch is W x R (weak scaling)
            pix = ds.next_pixels(R * W)
            bg = torch.rand((R * W, 3), device="cuda", generator=self._bg_gen)
            if W > 1:
                lo, hi = dp.shard_range(R, self.rank)
                pix, bg = pix[lo:hi], bg[lo:hi]
            bg = bg.contiguous()
            img_ids, rays_o, rays_d, target = ops.prepare_batch(pix.contiguous(), ds.W, ds.H, ds.transforms_gpu, ds.focal_lengths,
                                                                ds.principal, ds.image_data, bg)    # dataset.py:172-188 + runner.py:68
            return img_ids, rays_o, rays_d, bg, target
        img_ids, rays_o, rays_d, rgba = batch
        R = rays_o.shape[0]
        bg = torch.rand((R * W, 3), device="cuda", generator=self._bg_gen)
        if W > 1:
            bg = bg[self.rank * R:(self.rank + 1) * R]
        bg = bg.contiguous()
        return img_ids, rays_o, rays_d, bg, ops.blend_target(rgba.contiguous(), bg)                # runner.py:68

    # ------------------------------------------------------------------------------------------ software pipeline over steps
    def _front(self, step, batch, prefetch):
        """The part of training step `step` that does not read a network parameter: background colours, ray generation + target
        lookup (or the blend of a fed batch), march, compaction.  prefetch=True runs it on the side stream, behind the start of the
        step in flight; otherwise on the current stream (first step, and every step that starts with an occupancy-grid update: the
        update evaluates the density network, so it needs the finished optimizer sweep)."""
        P, s = self._pipe, self.sampler
        slot = P["made"] & 1
        main = P["main"] if P["main"] is not None else torch.cuda.current_stream()
        side = P["stream"]
        if prefetch:
            side.wait_event(P["mid"])                                # recorded on the main stream at the start of the step in flight
        # the step that read this slot's coordinate rows two fronts ago must be through (it is, unless the host runs far ahead)
        (side if prefetch else main).wait_event(P["back_done"][slot])
        with (torch.cuda.stream(side) if prefetch else contextlib.nullcontext()):
            rng_before = s.rng.copy()
            if step % s.update_den_freq == 0:
                assert not prefetch
                self._table_ready()                                  # the update evaluates the density network on the exchanged table
                s.update_density_grid()
            img_ids, rays_o, rays_d, bg, target = self._batch(batch)
            numsteps, ns_c, cnt_c, coords = s.sample_front(rays_o, rays_d, P["coords"][slot],
                                                           ray_index_offset=dp.shard_range(rays_o.shape[0], self.rank)[0])
            done = torch.cuda.Event()
            done.record(side if prefetch else main)
        P["made"] += 1
        P["prefetched"] += int(prefetch)
        return dict(step=step, src=batch, slot=slot, bg=bg, target=target, numsteps=numsteps, ns_c=ns_c, cnt_c=cnt_c, coords=coords, done=done,
                    rng_before=rng_before, rays=(img_ids, rays_o, rays_d), side=prefetch)

    def _adapt_ray_batch(self, F):
        """DensityGridSampler.update_batch_rays (density_grid_sampler.py:266-271) without stalling the pipeline: the 16-step sample
        counter is read back on the SIDE stream (all-reduced there first under data parallelism), behind the last march that added
        to it -- the host waits for that march only, not for the network kernels of the step it has just enqueued, and keeps its
        lead over the device (a `.item()` on the main stream drained the queue every 16 steps: the device then idled while the host
        enqueued the next step from scratch)."""
        P, s = self._pipe, self.sampler
        side = P["stream"]
        if P.get("count_host") is None:
            P["count_host"], P["count_ev"] = torch.zeros(1, dtype=torch.int32).pin_memory(), torch.cuda.Event()
        side.wait_event(F["done"])
        with torch.cuda.stream(side):
            if self.world_size > 1:
                dp.global_sum_count(s.measured_batch_size, self.pg, self.world_size)
            P["count_host"].copy_(s.measured_batch_size, non_blocking=True)
            s.measured_batch_size.zero_()
            P["count_ev"].record(side)
        P["count_ev"].synchronize()
        P["main"].wait_event(P["count_ev"])                          # the next front (a grid-update step: main stream) adds to the counter
        s.update_batch_rays(measured_total=int(P["count_host"][0]))

    def _sync_front(self):
        """Evaluation and checkpoint code shares the march workspace with a prefetched front: order the current stream behind it."""
        P = self._pipe
        if P is not None and P["pending"] is not None:
            torch.cuda.current_stream().wait_event(P["pending"]["done"])

    def _train_step_pipe(self, batch=None, next_batch=None):
        cfg, s, P = self.cfg, self.sampler, self._pipe
        i = cfg.m_training_step
        main = P["main"] = torch.cuda.current_stream()
        F, P["pending"] = P["pending"], None
        if F is not None and (F["step"] != i or F["src"] is not batch):
            main.wait_event(F["done"])                               # it may still be marching: the workspace is shared with the new front
            F = None                                                 # the caller changed course (other batch, other step): drop it
        if F is None:
            F = self._front(i, batch, prefetch=False)
        elif F["side"]:
            main.wait_event(F["done"])
        P["mid"].record(main)                                        # the next front may start with this step
        # (the sampler is an nn.Module: plain attribute assignment goes through Module.__setattr__, ~2 us apiece)
        s.__dict__.update(_rays_numsteps=F["numsteps"], _rays_numsteps_compacted=F["ns_c"], _counters_compacted=F["cnt_c"], _coords=F["coords"])
        # data parallel: the exchange of step i-1 has delivered the table; its gradient buffers are cleared beside the forward
        rgb, loss = self._net_pass(F["bg"], F["target"], zero_on=(P["aux"], P["aux_done"]))
        self._optimizer_tail()
        P["back_done"][F["slot"]].record(main)
        self.last_loss, self.last_rgb = loss, rgb
        cfg.m_training_step = i + 1
        self._pipe_last = F                                          # keeps the front's tensors alive until the next step replaces them
        if i % s.update_den_freq == s.update_den_freq - 1:
            self._adapt_ray_batch(F)                                 # after this step's march, before the next front, as in sample()
        # the front of step i+1, unless that step opens with an occupancy-grid update (needs the sweep above) or the caller feeds
        # batches and has not said which one comes next
        if (i + 1) % s.update_den_freq != 0 and (batch is None or next_batch is not None):
            P["pending"] = self._front(i + 1, next_batch if batch is not None else None, prefetch=True)
        return loss

    def train_step(self, batch=None, next_batch=None):
        if self._pipe is not None:
            return self._train_step_pipe(batch, next_batch)
        cfg, s = self.cfg, self.sampler
        i = cfg.m_training_step
        img_ids, rays_o, rays_d, bg, target = self._batch(batch)
        if i % s.update_den_freq == 0:
            self._table_ready()                                      # the occupancy-grid update evaluates the density network
        s.sample(img_ids, rays_o, rays_d, is_training=True,          # grid update /16, march, bookkeeping, ray-batch adaptation /16
                 ray_index_offset=dp.shard_range(rays_o.shape[0], self.rank)[0])
        rgb, loss = self._net_pass(bg, target)
        self._optimizer_tail()
        self.last_loss, self.last_rgb = loss, rgb
        cfg.m_training_step = i + 1
        return loss

    # ------------------------------------------------------------------------------------------ host-fed batches
    def train_step_host(self, batch, next_batch=None):
        """One training step on a ray batch that lives in PINNED HOST memory -- (img_ids int32 (R,), rays_o (R,3), rays_d (R,3),
        rgba (R,4) f32), what the reference's dataset yields (dataset.py:172-188).  The batch is copied on a side stream into one of
        two device staging slots; passing `next_batch` starts the copy of the following step's batch before this step's kernels are
        enqueued, so that the copy runs under them.  The mean loss goes back to the host on the side stream as well: the returned
        pinned 1-element tensor holds it once that stream has caught up (read it a step later, or synchronise)."""
        st = self._host_stage
        if st is None:
            st = self._host_stage = dict(stream=torch.cuda.Stream(), slots=[None, None], ready=[torch.cuda.Event(), torch.cuda.Event()],
                                         free=[torch.cuda.Event(), torch.cuda.Event()], staged=[None, None], dev=[None, None], k=0,
                                         loss_host=torch.zeros(1, dtype=torch.float32).pin_memory(), done=torch.cuda.Event())
            for e in st["free"]:
                e.record()
        main = torch.cuda.current_stream()

        def put(b, slot):
            R = b[1].shape[0]
            if st["slots"][slot] is None or st["slots"][slot][1].shape[0] < R:
                cap = max(2 * R, 4096)
                st["slots"][slot] = (torch.empty(cap, dtype=torch.int32, device="cuda"), torch.empty((cap, 3), device="cuda"),
                                     torch.empty((cap, 3), device="cuda"), torch.empty((cap, 4), device="cuda"))
            with torch.cuda.stream(st["stream"]):
                st["stream"].wait_event(st["free"][slot])              # the step that read this slot has finished with it
                for dst, src in zip(st["slots"][slot], b):
                    dst[:R].copy_(src, non_blocking=True)
                st["ready"][slot].record()
            st["staged"][slot] = (b, R)
            st["dev"][slot] = tuple(t[:R] for t in st["slots"][slot])

        slot = st["k"] % 2
        if st["staged"][slot] is None or st["staged"][slot][0] is not batch:
            put(batch, slot)
        if next_batch is not None:
            put(next_batch, 1 - slot)
        main.wait_event(st["ready"][slot])
        dev, nxt = st["dev"][slot], None
        if next_batch is not None and self._pipe is not None:
            nxt = st["dev"][1 - slot]                                # its front (blend, march) is enqueued under this step's kernels
            self._pipe["stream"].wait_event(st["ready"][1 - slot])
        loss = self.train_step(dev, nxt)
        st["free"][slot].record(main)
        st["staged"][slot] = None
        st["k"] += 1
        st["done"].record(main)
        with torch.cuda.stream(st["stream"]):
            st["stream"].wait_event(st["done"])
            loss.record_stream(st["stream"])
            st["loss_host"].copy_(loss.mean().reshape(1), non_blocking=True)
        return st["loss_host"]

    def net_forward(self, coords, n_dev):
        """Fused hash encode + SH + both MLPs on the sampler's coordinate rows -> self.net_out (+ self.enc)."""
        m = self.model
        ops.network_fwd(coords, m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights,
                        n_dev=n_dev, out=self.net_out, enc=self.enc)

    def _net_pass(self, bg, target, zero_on=None):
        """Network forward, composite + Huber loss + composite backward, network backward on the rows of the sampler's last march ->
        (rgb, loss); the gradients are left for the optimizer tail.  zero_on: as in _table_ready."""
        s = self.sampler
        coords, n_dev = s.coords_compacted, s.n_samples_dev
        zeroing = self._table_ready(zero_on)
        self.net_forward(coords, n_dev)
        # local loss_scale is 128/R_local (calc_rgb.h:100-101): the all-reduced sum is W x the global-batch gradient, and the exchange
        # applies 1 / W to it
        rgb, loss, _ = ops.composite_loss_bwd(self.net_out, coords, s._rays_numsteps, s._rays_numsteps_compacted, bg, target, s.density_grid_mean,
                                              delta=self.loss_func.delta, cascades=s.NERF_CASCADES, dnet=self.dnet,
                                              reg_scale=float(self.world_size))
        if zeroing:
            torch.cuda.current_stream().wait_event(zero_on[1])
        self.net_backward(coords, n_dev)
        return rgb, loss

    def net_backward(self, coords, n_dev):
        """self.dnet -> gradients of the hash table (self.grid_grad) and of both weight vectors (self.dwd, self.dwr)."""
        m = self.model
        if self._fx is not None:                                     # into the scratch the next sweep reads and clears
            ops.network_bwd_fx(coords, self.enc, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights, self.dnet,
                               self._fx, self._w_part, n_dev=n_dev)
            self._bwd_rows = coords.shape[0]                         # the sweep reads as many weight-gradient slots as this fills
            return
        ops.network_bwd(coords, self.enc, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights, self.dnet,
                        self.grid_grad, self.dwd, self.dwr, n_dev=n_dev)

    def _optimizer_tail(self):
        """One optimizer step of the host-state training steps: ExpDecay's learning rate, Adam's and the EMA's step counters, then
        _optimizer_step."""
        lr = self.optimizer.advance_lr()
        adam = self.optimizer._nested_optimizer
        adam.n_step += 1
        self.ema_optimizer.steps += 1
        self._optimizer_step(lr, adam.n_step)

    def _optimizer_step(self, lr, n_step):
        """Gradient exchange + fused Adam/EMA sweep(s) (optims/adam.py + ema.py; runner.py:75-76)."""
        m = self.model
        adam = self.optimizer._nested_optimizer
        hyper = (lr, n_step, adam.betas[0], adam.betas[1], adam.eps, self.ema_optimizer.decay)
        if self._fx is not None:
            st = [self._st[id(p)] for p in (m.pos_encoder.m_grid, m.density_mlp.con_weights, m.rgb_mlp.con_weights)]
            ops.train_sweep(m.pos_encoder.m_grid.data, (st[0].m, st[0].v, st[0].master), self._fx, self._w_part, self._bwd_rows,
                            m.density_mlp.con_weights.data, (st[1].m, st[1].v, st[1].master), m.rgb_mlp.con_weights.data,
                            (st[2].m, st[2].v, st[2].master), *hyper)
            return
        if self.world_size > 1 and self.dp_mode == "p2p":
            st = self._st[id(m.pos_encoder.m_grid)]
            self._epoch += 1
            ops.dp_exchange_step(self.world_size, self.rank, self._hi - self._lo, self._w_param.numel(), self._peers["table"],
                                 self._peers["table_grad"], self._peers["w_grad"], self._peers["flags"], self._epoch, st.m, st.v, st.master,
                                 self._w_param, self._w_m, self._w_v, self._w_master, *hyper, grad_scale=1.0 / self.world_size)
            self._pending_epoch = self._epoch
            return
        if self.world_size > 1:
            # hash table: reduce-scatter -> Adam+EMA on this rank's slice -> async all-gather (waited for in the NEXT step, after the march)
            dp.reduce_scatter_sum(self._slice_grad, self._table_grad, self.pg, self.world_size, self.rank)
            scale = dp.allreduce_grads((self.w_grad,), self.pg, self.world_size)
            st = self._st[id(m.pos_encoder.m_grid)]
            ops.adam_ema(self._slice_param, self._slice_grad, st.m, st.v, st.master, *hyper, grad_scale=scale, zero_grad=False)
            self._table_work = dp.all_gather_slices(self._table, self._slice_param, self.pg, self.world_size, async_op=True)
            self._table_grad.zero_()
            tensors = ((m.density_mlp.con_weights, self.dwd), (m.rgb_mlp.con_weights, self.dwr))
        else:
            scale = 1.0
            tensors = ((m.pos_encoder.m_grid, self.grid_grad), (m.density_mlp.con_weights, self.dwd), (m.rgb_mlp.con_weights, self.dwr))
        for p, g in tensors:
            st = self._st[id(p)]
            ops.adam_ema(p.data, g, st.m, st.v, st.master, *hyper, grad_scale=scale, zero_grad=True)

    # --------------------------------------------------------------------- per-operator path (as the reference wires it)
    def train_step_autograd(self, batch=None):
        cfg = self.cfg
        i = cfg.m_training_step
        img_ids, rays_o, rays_d, rgba = self.next_batch() if batch is None else batch
        bg = torch.rand((rays_o.shape[0], 3), device="cuda", generator=self._bg_gen)
        target = (rgba[:, :3] * rgba[:, 3:] + bg * (1 - rgba[:, 3:])).detach()
        pos, dir_ = self.sampler.sample(img_ids, rays_o, rays_d, is_training=True)
        network_outputs = self.model(pos, dir_)
        rgb = self.sampler.rays2rgb(network_outputs, bg)
        loss = self.loss_func(rgb, target)
        self.optimizer.step(loss)
        self.ema_optimizer.ema_step()
        cfg.m_training_step = i + 1
        return loss.sum(-1)

    def train(self, steps=None, log_every=0):
        end = self.tot_train_steps if steps is None else self.cfg.m_training_step + steps
        step_fn = self.train_step if self.fast else self.train_step_autograd
        while self.cfg.m_training_step < end:
            loss = step_fn()
            i = self.cfg.m_training_step
            if log_every and i % log_every == 0 and self.rank == 0:
                print(f"STEP={i} | LOSS={loss.mean().item():.6f} | rays/batch={self.sampler.n_rays_per_batch}", flush=True)

    # ------------------------------------------------------------------------------------------ evaluation
    @torch.no_grad()
    def render_img(self, dataset_mode="train", img_id=0):
        """runner.py:197-236: tile the image in n_rays_per_batch chunks; returns (img HxWx3, target HxWx3)."""
        self._table_ready()
        self._sync_front()
        ds = self.dataset[dataset_mode]
        W, H = ds.resolution
        rays_o, rays_d = ds.generate_rays_total_test(img_id)
        tile = self.cfg.n_rays_per_batch
        img = torch.empty((H * W, 3), device="cuda")
        alpha = torch.empty((H * W, 1), device="cuda")
        ids = torch.zeros(tile, dtype=torch.int32, device="cuda")
        s, m = self.sampler, self.model
        for p in range(0, H * W, tile):
            e = min(p + tile, H * W)
            o, d = rays_o[p:e], rays_d[p:e]
            if e - p < tile:
                o = torch.cat([o, torch.ones((tile - (e - p), 3), device="cuda")])
                d = torch.cat([d, torch.ones((tile - (e - p), 3), device="cuda")])
            s.sample(ids, o.contiguous(), d.contiguous())
            coords = s._coords
            if self.fast:
                out, _ = ops.network_fwd(coords.contiguous(), m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights,
                                         m.rgb_mlp.con_weights, save_enc=False) if coords.shape[0] else (torch.empty((0, 4), dtype=torch.float16, device="cuda"), None)
            else:
                out = m(coords[:, :3], coords[:, 4:])
            rgb, a = s.rays2rgb(out, inference=True)
            img[p:e], alpha[p:e] = rgb[:e - p], a[:e - p]
        bgc = torch.tensor(self.background_color, dtype=torch.float32, device="cuda")
        img = img + bgc * (1 - alpha)
        return img.reshape(H, W, 3), self._target_img(ds, img_id)

    def _target_img(self, ds, img_id):
        """Image img_id of split ds as (H, W, 3), with the background colour blended in (runner.py:68)."""
        W, H = ds.resolution
        bgc = torch.tensor(self.background_color, dtype=torch.float32, device="cuda")
        tar = ds.rgba_for(torch.arange(H * W, device="cuda", dtype=torch.int32) + int(img_id) * H * W)
        return (tar[:, :3] * tar[:, 3:] + bgc * (1 - tar[:, 3:])).reshape(H, W, 3)

    def _infer_tiles(self, rays_o, rays_d):
        """(rgb (R,3) without background, alpha (R,1)) of the rays through march -> fused network -> inference composite, in tiles of
        n_rays_per_batch rays (the last one as short as the rays leave it); one rng.advance() per tile.  The march's device-side
        counter bounds the network kernel: nothing is read back."""
        s = self.sampler
        tile = self.cfg.n_rays_per_batch
        rgb = torch.empty((rays_o.shape[0], 3), device=rays_o.device)
        alpha = torch.empty((rays_o.shape[0], 1), device=rays_o.device)
        if getattr(self, "_infer_net_out", None) is None:
            self._infer_net_out = torch.empty((s.max_samples, 4), dtype=torch.float16, device="cuda")
        s._ensure_march_ws(tile)
        for p in range(0, rays_o.shape[0], tile):
            coords, _, numsteps, counters = ops.march(
                rays_o[p:p + tile].contiguous(), rays_d[p:p + tile].contiguous(), s.density_grid_bitfield, s.aabb_range, s.max_samples,
                s.cone_angle_constant, s.near_distance, s.NERF_CASCADES, s.const_dt, s.rng, coords=s._coords_raw, workspace=s._march_ws)
            ops.pcg32_advance(s.rng)                                   # rng.advance(), ray_sampler.py:61
            self._net_infer(coords, counters[1:2], self._infer_net_out)
            rgb[p:p + tile], alpha[p:p + tile] = ops.composite_infer(self._infer_net_out, coords, numsteps, s.NERF_CASCADES)
        return rgb, alpha

    def _net_infer(self, rows, n_dev, out):
        """Inference forward of the model on (N,7) coordinate rows into out (N,4), bounded by the device row count n_dev."""
        m = self.model
        if self.fast:
            ops.network_fwd(rows, m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights, n_dev=n_dev,
                            save_enc=False, out=out)
        else:
            m.infer(rows, n_dev, out)

    @torch.no_grad()
    def render_img_nosync(self, dataset_mode="train", img_id=0):
        """N3 (SURVEY 8f): the image of render_img without the reference tiler's host round trips (runner.py:206-228 reads the
        sample count back with .item() and copies every tile to the host; 157 tiles per 800x800 image).  The march's device-side
        counter bounds the fused network kernel (n_dev), ngp_composite_infer writes into the image buffer, nothing is read back
        before the caller uses the result.  Same kernels, same RNG consumption, same pixels as render_img."""
        assert self._can_infer, "render_img_nosync needs the fused NGP model or a model with an inference forward (infer)"
        self._table_ready()
        self._sync_front()
        ds = self.dataset[dataset_mode]
        W, H = ds.resolution
        rays_o, rays_d = ds.generate_rays_total_test(img_id)
        tile = self.cfg.n_rays_per_batch
        n_pix = H * W
        n_pad = (n_pix + tile - 1) // tile * tile
        if n_pad > n_pix:                                              # the reference pads the last tile with ones (runner.py:213-217)
            fill = torch.ones((n_pad - n_pix, 3), device="cuda")
            rays_o, rays_d = torch.cat([rays_o, fill]), torch.cat([rays_d, fill])
        img, alpha = self._infer_tiles(rays_o, rays_d)
        bgc = torch.tensor(self.background_color, dtype=torch.float32, device="cuda")
        img = img[:n_pix] + bgc * (1 - alpha[:n_pix])
        return img.reshape(H, W, 3), self._target_img(ds, img_id)

    # ------------------------------------------------------------------------------------------ rendering (runner.py:86-121, 162-264)
    @torch.no_grad()
    def render_rays(self, rays_o, rays_d, min_transmittance=1e-4):
        """Whole-frame renderer (ops.render_rays): every ray at once in rounds, each ray dropped after the first sample that brings its
        transmittance below min_transmittance (0: never, and then every ray composites the samples render_img_nosync gives it).  The
        jitter and the sampler rng advance exactly as render_img_nosync's n_rays_per_batch tiles would have them.
        Returns (rgb (R,3) without background, alpha (R,1), n_samples (R,), rounds).
        The renderer's workspace (per-ray state, and 144 MB of round rows and network outputs at the default capacity) is kept for the
        next frame; render() and test() release it when they finish, and release_render_workspace() does so at any time."""
        assert self._can_infer, "render_rays needs the fused NGP model or a model with an inference forward (infer)"
        self._table_ready()
        self._sync_front()
        s, m = self.sampler, self.model
        R, tile = rays_o.shape[0], int(self.cfg.n_rays_per_batch)
        self._render_ws = ops.render_workspace(R, self._render_ws)
        args = (rays_o.contiguous(), rays_d.contiguous(), s.density_grid_bitfield, s.aabb_range, s.cone_angle_constant, s.near_distance,
                s.NERF_CASCADES, s.const_dt, s.rng)
        if self.fast:
            out = ops.render_rays(*args, m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights, m.rgb_mlp.con_weights, tile,
                                  min_transmittance=min_transmittance, workspace=self._render_ws)
        else:
            out = ops.render_rays(*args, None, None, None, None, tile, min_transmittance=min_transmittance, workspace=self._render_ws,
                                  net=m.infer)
        ops.pcg32_advance(s.rng, ((R + tile - 1) // tile) << 32)       # one rng.advance() per tile (ray_sampler.py:61)
        return out

    def release_render_workspace(self):
        """Free the whole-frame renderer's workspace (the next render_rays allocates a new one), e.g. before training on."""
        self._render_ws = None

    def _render_frame(self, rays_o, rays_d, W, H, min_transmittance):
        """(img (H,W,3) with the background blended in unless alpha_image, alpha (H,W,1), n_samples (H,W), rounds)"""
        rgb, alpha, n, rounds = self.render_rays(rays_o, rays_d, min_transmittance)
        if not getattr(self.cfg, "alpha_image", False):
            rgb = rgb + torch.tensor(self.background_color, dtype=torch.float32, device=rgb.device) * (1 - alpha)
        return rgb.reshape(H, W, 3), alpha.reshape(H, W, 1), n.reshape(H, W), rounds

    def pose_rays(self, pose):
        """generate_rays_with_pose (dataset.py:236-253): the rays of every pixel, row-major, of a camera at `pose` (3x4 or 4x4 NeRF
        camera-to-world) with the train split's image-0 intrinsics and its true [W, H] (DESIGN.md section 7)."""
        from .plugin.dataset import matrix_nerf2ngp
        ds = self.dataset["train"]
        W, H = ds.resolution
        xf = matrix_nerf2ngp(np.asarray(pose, np.float32)[:3, :4], ds.scale, ds.offset, getattr(ds, "correct_pose", (1, -1, -1)))
        dev = ds.transforms_gpu.device
        xforms = torch.from_numpy(np.ascontiguousarray(xf.T).reshape(1, 12)).to(dev)   # one-entry table, column-major like transforms_gpu
        pix = torch.arange(H * W, dtype=torch.int32, device=dev)
        _, o, d = ops.raygen(pix, W, H, xforms, ds.focal_lengths[:1].contiguous(), ds.principal[:1].contiguous())
        return o, d

    @torch.no_grad()
    def render_img_with_pose(self, pose, min_transmittance=1e-4):
        """runner.py:238-264 on the whole-frame renderer: the (H, W, 3) image of a camera at `pose`, background blended in unless
        alpha_image is set."""
        W, H = self.dataset["train"].resolution
        o, d = self.pose_rays(pose)
        return self._render_frame(o, d, W, H, min_transmittance)[0]

    def _save_path(self):
        return os.path.join(self.cfg.log_dir or ".", self.cfg.exp_name or "exp")

    @staticmethod
    def save_img(path, img, alpha=None):
        """runner.py:180-188: an (H, W, 3) image in [0, 1] (+ (H, W, 1) alpha: RGBA) as an 8-bit PNG."""
        from PIL import Image
        img = img.detach().cpu().numpy() if torch.is_tensor(img) else np.asarray(img)
        if alpha is not None:
            alpha = alpha.detach().cpu().numpy() if torch.is_tensor(alpha) else np.asarray(alpha)
            img = np.concatenate([img, alpha], axis=-1)
        Image.fromarray((img * 255 + 0.5).clip(0, 255).astype(np.uint8)).save(path)

    @torch.no_grad()
    def render(self, save_path=None, load_ckpt=False, min_transmittance=1e-4):
        """runner.py:101-121: the 80-frame spherical camera path (utils/camera_path.py) as an mp4 (OpenCV, mp4v, 28 fps), by default
        log_dir/exp_name/demo.mp4.  Returns the path."""
        try:
            import cv2
        except ImportError as e:
            raise RuntimeError("Runner.render writes the video with OpenCV: install opencv-python (cv2) to use it") from e
        from .utils.camera_path import path_spherical
        if load_ckpt:
            self.load_ckpt(self.cfg.ckpt_path)
        if not save_path:
            save_path = os.path.join(self._save_path(), "demo.mp4")
        elif not str(save_path).endswith(".mp4"):
            raise ValueError(f"Runner.render: the video path must end in .mp4, got {save_path}")
        os.makedirs(os.path.dirname(os.path.abspath(save_path)), exist_ok=True)
        W, H = self.dataset["train"].resolution
        writer = cv2.VideoWriter(str(save_path), cv2.VideoWriter_fourcc(*"mp4v"), 28, (W, H))
        try:
            for pose in path_spherical():
                img = self.render_img_with_pose(pose, min_transmittance)
                u8 = (img.cpu().numpy() * 255 + 0.5).clip(0, 255).astype(np.uint8)
                writer.write(np.ascontiguousarray(u8[..., ::-1]))    # OpenCV takes BGR: the file shows the true colours (DESIGN.md section 7)
        finally:
            writer.release()
            self.release_render_workspace()
        return save_path

    @torch.no_grad()
    def render_test(self, save_img=True, save_path=None, min_transmittance=1e-4):
        """runner.py:162-178: every view of the test split on the whole-frame renderer; saves {exp_name}_r_{i}.png (RGBA when
        alpha_image is set) and, when the split has images, {exp_name}_gt_{i}.png; returns the per-view mse against the target with the
        background blended in (an empty list for a split without images, as the reference computes no PSNR then)."""
        ds = self.dataset["test"]
        save_path = self._save_path() if save_path is None else save_path
        if save_img:
            os.makedirs(save_path, exist_ok=True)
        exp = self.cfg.exp_name
        W, H = ds.resolution
        have_img = getattr(ds, "have_img", True)
        mse = []
        for i in range(ds.n_images):
            o, d = ds.generate_rays_total_test(i)
            img, alpha, _, _ = self._render_frame(o, d, W, H, min_transmittance)
            if save_img:
                self.save_img(os.path.join(save_path, f"{exp}_r_{i}.png"), img, alpha if getattr(self.cfg, "alpha_image", False) else None)
            if not have_img:                                          # runner.py:173: no target, no gt image, no mse
                continue
            tar = self._target_img(ds, i)
            if save_img:
                self.save_img(os.path.join(save_path, f"{exp}_gt_{i}.png"), tar)
            mse.append(float(L.img2mse(img, tar).item()))
        return mse

    @torch.no_grad()
    def test(self, load_ckpt=False, min_transmittance=1e-4):
        """runner.py:86-99: render the test split into log_dir/exp_name/test and print the mean test PSNR, which is returned (None for
        a split without images, as the reference prints none then).  Releases the renderer's workspace when done."""
        if load_ckpt:
            self.load_ckpt(self.cfg.ckpt_path)
        if self.dataset["test"] is None:
            self.dataset["test"] = build_from_cfg(self.cfg.dataset.test, DATASETS)
        try:
            mse = self.render_test(save_path=os.path.join(self._save_path(), "test"), min_transmittance=min_transmittance)
        finally:
            self.release_render_workspace()
        if not getattr(self.dataset["test"], "have_img", True):
            return None
        psnr = sum(float(L.mse2psnr(torch.tensor(v)).item()) for v in mse) / len(mse)
        print(f"TOTAL TEST PSNR===={psnr}", flush=True)
        return psnr

    @torch.no_grad()
    def extract_mesh(self, out_dir, resolution=512, mcube_smooth=False):
        """tools/extract_mesh.py of the reference on the device: the density lattice of the unit cube (:42-70), marching cubes at 0.5
        (:78) in the PLY frame (:80-84) -> out_dir/mesh-origin.ply, the largest edge-connected component (:92-97), area-weighted vertex
        normals (:106), one colour ray per vertex through the march / network / inference-composite kernels (:108-135) ->
        out_dir/mesh-color.ply.  The colour ray starts 0.2 outside the vertex and runs along the unit normal into the object (towards
        higher density), in model space (DESIGN.md section 7).  mcube_smooth (:74-78): the lattice is smoothed (ops.mesh_smooth, method
        auto) and marched at 0 instead, which removes the terraces of the integer density field; the result then also holds the
        smoothing's info under "smooth".  Returns the arrays, the counts and the device time of each stage."""
        import os
        from .utils.ply import write_ply
        if not self.fast:
            raise NotImplementedError(f"extract_mesh: mesh extraction runs on the fused NGPNetworks kernels; {type(self.model).__name__} "
                                      "(fp16 / use_fully off, or another model) has no density lattice kernel")
        self._table_ready()
        self._sync_front()
        N = int(resolution)
        if not 2 <= N <= 1024:
            raise ValueError(f"extract_mesh: resolution {N} is outside [2, 1024]")
        os.makedirs(out_dir, exist_ok=True)
        m = self.model
        names = ("density_lattice",) + (("smooth",) if mcube_smooth else ()) + ("marching_cubes", "write_origin", "component_normals", "colour")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
        stamps = iter(ev)                                             # one event after each stage, in the order of `names`
        next(stamps).record()
        field = ops.density_lattice(N, m.pos_encoder.m_grid, m.pos_encoder.levels, m.density_mlp.con_weights)
        next(stamps).record()
        smooth = None
        if mcube_smooth:
            field, smooth = ops.mesh_smooth(field)
            next(stamps).record()
        verts0, tris0 = ops.marching_cubes(field, 0.0 if mcube_smooth else 0.5)
        next(stamps).record()
        del field
        v0_host, t0_host = verts0.cpu().numpy(), tris0.cpu().numpy()
        write_ply(os.path.join(out_dir, "mesh-origin.ply"), v0_host, t0_host)
        next(stamps).record()
        verts, tris = ops.mesh_largest_component(verts0, tris0)
        normals = ops.mesh_vertex_normals(verts, tris)
        next(stamps).record()
        # back to model space (x/y swapped again); the ray runs against the outward normal, into the object
        perm = torch.tensor([1, 0, 2], device=verts.device)
        v_model, n_model = verts[:, perm], normals[:, perm]
        zero = (n_model == 0).all(dim=1, keepdim=True)                 # a vertex whose triangles all have zero area: any direction
        dirs = torch.where(zero, torch.tensor([0.0, 0.0, -1.0], device=verts.device), -n_model).contiguous()
        origins = (v_model - 0.2 * dirs).contiguous()
        rgb, alpha = self._infer_tiles(origins, dirs)                 # same kernels and RNG consumption per tile as render_img_nosync
        next(stamps).record()
        # :136-137 in float64, as numpy promotes the reference's integer background colour
        img = rgb.cpu().numpy().astype(np.float64) + np.asarray(self.background_color, np.float64) * (1 - alpha.cpu().numpy().astype(np.float64))
        colors = (img * 255 + 0.5).clip(0, 255).astype(np.uint8)
        v_host, t_host = verts.cpu().numpy(), tris.cpu().numpy()
        write_ply(os.path.join(out_dir, "mesh-color.ply"), v_host, t_host, colors)
        torch.cuda.synchronize()
        times = {k: round(ev[i].elapsed_time(ev[i + 1]), 3) for i, k in enumerate(names)}
        res = dict(vertices=v_host, triangles=t_host, normals=normals.cpu().numpy(), colors=colors, origins=origins.cpu().numpy(),
                   dirs=dirs.cpu().numpy(), n_verts_origin=int(v0_host.shape[0]), n_tris_origin=int(t0_host.shape[0]),
                   n_verts=int(v_host.shape[0]), n_tris=int(t_host.shape[0]), stage_ms=times)
        if mcube_smooth:
            res["smooth"] = smooth
        return res

    @torch.no_grad()
    def psnr(self, dataset_mode="val", max_images=None):
        """mean over images of -10 log10(mse) (runner.py:86-99, mse_loss.py:6-7)."""
        ds = self.dataset[dataset_mode]
        n = ds.n_images if max_images is None else min(max_images, ds.n_images)
        tot = 0.0
        for k in range(n):
            img, tar = self.render_img(dataset_mode, k)
            tot += float(L.mse2psnr(L.img2mse(img, tar)).item())
        return tot / n

    # ------------------------------------------------------------------------------------------ checkpoint (N4)
    def save_ckpt(self, path):
        """Every rank must call this when world_size > 1 (the table's optimizer state is gathered); rank 0 writes the file."""
        adam = self.optimizer._nested_optimizer
        self._table_ready()
        nested = adam.state_dict()
        if self.world_size > 1:
            k = [id(s.p) for s in adam.state].index(id(self.model.pos_encoder.m_grid))
            full = self._gather_table_state()
            for key, t in zip(("m", "v", "master"), full):
                nested[key] = list(nested[key])
                nested[key][k] = t
            if self.rank != 0:
                return
        sampler_state = self.sampler.state_dict()
        if self._pipe is not None and self._pipe["pending"] is not None:
            # a prefetched front has drawn the next step's jitter already: the checkpoint holds the stream position of global_step
            sampler_state["rng"] = torch.from_numpy(self._pipe["pending"]["rng_before"].astype(np.int64))
        ck = {"global_step": self.cfg.m_training_step, "model": self.model.state_dict(), "sampler": sampler_state,
              "optimizer": self.optimizer.state_dict(), "nested_optimizer": nested, "ema_optimizer": self.ema_optimizer.state_dict()}
        if str(path).endswith(".pkl") and not hasattr(getattr(self.model, "density_mlp", None), "con_weights"):
            raise NotImplementedError(f"the .pkl interchange format is written for the fused-MLP parameter layout (con_weights) of "
                                      f"NGPNetworks; save {type(self.model).__name__} to a .pt path")
        if str(path).endswith(".pkl"):
            # the reference's params.pkl wire format (runner/runner.py:123-131), readable by its load_ckpt (:133-151)
            from .utils import ckpt_compat as cc
            dec = self.optimizer
            ref = cc.native_to_reference(
                ck, adam_hyper=dict(lr=adam.lr, eps=adam.eps, betas=tuple(adam.betas)),
                expdecay_hyper=dict(base_lr=dec.base_lr, decay_start=dec.decay_start, decay_interval=dec.decay_interval, decay_base=dec.decay_base,
                                    decay_end=dec.decay_end),
                param_dtype=np.float16 if self.model.pos_encoder.m_grid.dtype == torch.float16 else np.float32)
            cc.write_reference_ckpt(ref, path)
            return
        torch.save(ck, path)

    def load_ckpt(self, path):
        self._table_ready()                                          # an exchange of the previous step may still be writing the table
        if self._pipe is not None:
            self._sync_front()
            self._pipe["pending"] = None                             # marched against the occupancy grid that is about to be replaced
        if self.world_size > 1:
            import torch.distributed as dist
            dist.barrier(group=self.pg)                              # no peer may still push into this rank's table while it is overwritten
        if str(path).endswith(".pkl") and not hasattr(getattr(self.model, "density_mlp", None), "con_weights"):
            raise NotImplementedError("the .pkl interchange format carries the fused-MLP parameter layout; load a .pt checkpoint instead")
        if str(path).endswith(".pkl"):
            from .utils import ckpt_compat as cc
            ck = cc.load_native_from_reference_file(path, self.model.pos_encoder.m_grid.numel(), "cuda",
                                                    {k: v.dtype for k, v in self.model.state_dict().items()})
        else:
            ck = torch.load(path, map_location="cuda", weights_only=True)      # tensors, numbers, lists and dicts only
        self.cfg.m_training_step = self.start = ck["global_step"]
        self.model.load_state_dict(ck["model"])
        self.sampler.load_state_dict(ck["sampler"])
        self.optimizer.load_state_dict(ck["optimizer"])
        nested = ck["nested_optimizer"]
        if self.world_size > 1:
            adam = self.optimizer._nested_optimizer
            k = [id(s.p) for s in adam.state].index(id(self.model.pos_encoder.m_grid))
            self._scatter_table_state(nested["m"][k], nested["v"][k], nested["master"][k])
            st = self._st[id(self.model.pos_encoder.m_grid)]
            nested = dict(nested, **{key: [t if j != k else getattr(st, key) for j, t in enumerate(nested[key])] for key in ("m", "v", "master")})
            self._slice_param.copy_(self._table[self._lo:self._hi])
        self.optimizer._nested_optimizer.load_state_dict(nested)
        self.ema_optimizer.load_state_dict(ck["ema_optimizer"])


def lego_cfg(fp16=True, synthetic=True, **over):
    """projects/ngp/configs/ngp_base.py key for key, + fp16 (BASELINE config #2) and the synthetic stand-in dataset."""
    ds_type = "SyntheticNerfDataset" if synthetic else "NerfDataset"
    c = dict(
        sampler=dict(type="DensityGridSampler", update_den_freq=16),
        encoder=dict(pos_encoder=dict(type="HashEncoder"), dir_encoder=dict(type="SHEncoder")),
        model=dict(type="NGPNetworks", use_fully=True),
        loss=dict(type="HuberLoss", delta=0.1),
        optim=dict(type="Adam", lr=1e-1, eps=1e-15, betas=(0.9, 0.99)),
        ema=dict(type="EMA", decay=0.95),
        expdecay=dict(type="ExpDecay", decay_start=20_000, decay_interval=10_000, decay_base=0.33, decay_end=None),
        dataset=dict(train=dict(type=ds_type, root_dir="data/lego", batch_size=4096, mode="train"),
                     val=dict(type=ds_type, root_dir="data/lego", batch_size=4096, mode="val", preload_shuffle=False),
                     test=dict(type=ds_type, root_dir="data/lego", batch_size=4096, mode="test", preload_shuffle=False)),
        exp_name="lego", log_dir="./logs", tot_train_steps=40000, background_color=[0, 0, 0],
        hash_func="p0 ^ p1 * 19349663 ^ p2 * 83492791", cone_angle_constant=0.00390625, near_distance=0.2, n_rays_per_batch=4096,
        n_training_steps=16, target_batch_size=1 << 18, const_dt=True, load_ckpt=False, ckpt_path=None, alpha_image=False, fp16=fp16,
    )
    c.update(over)
    return c


def fox_cfg(fp16=True, synthetic=True, **over):
    """projects/ngp/configs/ngp_fox.py key for key (BASELINE config #3: aabb_scale 4 from the capture's transforms, cone stepping
    `const_dt=False`, fp16, no validation split); `synthetic` swaps data/fox for the procedural stand-in with the capture's
    resolution, intrinsics, camera arc and aabb_scale (plugin/dataset.py: SyntheticNerfDataset(style="fox"))."""
    c = lego_cfg(fp16=fp16, synthetic=synthetic)
    ds_type = "SyntheticNerfDataset" if synthetic else "NerfDataset"
    extra = dict(style="fox") if synthetic else {}
    c.update(dataset=dict(train=dict(type=ds_type, root_dir="data/fox", batch_size=4096, mode="train", **extra),
                          test=dict(type=ds_type, root_dir="data/fox", batch_size=4096, mode="test", preload_shuffle=False, **extra)),
             exp_name="fox", const_dt=False)
    c.update(over)
    return c


def nerf_cfg(fp16=True, synthetic=True, **over):
    """projects/nerf/configs/nerf_base.py key for key (vanilla NeRF: FrequencyEncoder(10) / FrequencyEncoder(4), OriginNeRFNetworks, Adam
    lr 1e-2, 512 rays a batch, 200 000 steps); `synthetic` swaps data/lego for the procedural stand-in."""
    ds_type = "SyntheticNerfDataset" if synthetic else "NerfDataset"
    c = dict(
        sampler=dict(type="DensityGridSampler", update_den_freq=16),
        encoder=dict(pos_encoder=dict(type="FrequencyEncoder", multires=10), dir_encoder=dict(type="FrequencyEncoder", multires=4)),
        model=dict(type="OriginNeRFNetworks"),
        loss=dict(type="HuberLoss", delta=0.1),
        optim=dict(type="Adam", lr=1e-2, eps=1e-15, betas=(0.9, 0.99)),
        ema=dict(type="EMA", decay=0.95),
        expdecay=dict(type="ExpDecay", decay_start=20_000, decay_interval=10_000, decay_base=0.33, decay_end=None),
        dataset_type=ds_type, dataset_dir="data/lego",
        dataset=dict(train=dict(type=ds_type, root_dir="data/lego", batch_size=512, mode="train"),
                     val=dict(type=ds_type, root_dir="data/lego", batch_size=512, mode="val", preload_shuffle=False),
                     test=dict(type=ds_type, root_dir="data/lego", batch_size=512, mode="test", preload_shuffle=False)),
        exp_name="lego", log_dir="./logs", tot_train_steps=200000, background_color=[0, 0, 0], cone_angle_constant=0.00390625,
        near_distance=0.2, n_rays_per_batch=512, n_training_steps=16, target_batch_size=1 << 18, const_dt=True, fp16=fp16,
    )
    c.update(over)
    return c
