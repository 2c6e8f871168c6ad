"""Online map training on the fused kernels.

API-compatible with the reference `Mapper` (utils/mapper.py:33 of PRBonn/PIN_SLAM): same
constructor, pool attributes, `process_frame`, `get_batch`, `mapping`, `sdf`, `sdf_batch`,
`get_numerical_gradient`, `dynamic_filter`, `determine_used_pose`, `transform_data_pool`.
One training iteration (reference: ~590 ATen ops + ~32 host syncs, mapper.py:623-822) is

    batch draw          torch.randint + pool gathers (same RNG calls as the reference)
    K1  query_sdf       all bs + 6*ceil(bs/10) rows in ONE launch (training side effects on the
                        first bs rows only), kNN ids / weights saved
    loss heads          BCE-with-logits + Eikonal (numerical gradient) -> d loss / d sdf per row
    K2  train_backward  decoder activations recomputed, feature-gradient scatter + decoder grads
    K3  adam_step x2    neural-point features, decoder parameters (fresh Adam state per call,
                        like the reference's per-frame setup_optimizer)

With torch.distributed initialised (one process per GPU, NCCL over NVLink) every rank trains on its
own sub-batch of its pool shard and the gradients are summed with ONE all-reduce per iteration
(certainty increments / timestamps are reduced once per mapping() call); map, decoder and Adam
state stay replicated and bit-identical across ranks.
"""

import torch

from .. import ops


class DataSampler:
    """Per-ray training samples (reference: utils/data_sampler.py:18-260): the measured end point,
    `surface_sample_n` Gaussian samples around it, `free_front_n` uniform samples in front and
    `free_behind_n` behind; label = signed distance along the ray (positive in front)."""

    FUSED = True  # CUDA inputs: the arithmetic runs in pinb200_ray_samples (the RNG draws stay torch calls)

    def __init__(self, config):
        self.config = config
        self.dev = config.device

    def sample(self, points, normals, sem_labels, colors):
        c = self.config
        dev = points.device
        n = points.shape[0]
        ns, nf, nb = c.surface_sample_n, c.free_front_n, c.free_behind_n
        total = 1 + ns + nf + nb
        sigma = c.surface_sample_range_m
        if self.FUSED and points.is_cuda and points.dtype == torch.float32 and normals is None and n > 0:
            # the reference's RNG draws (same generator, order and sizes), everything else in one kernel
            z_surf = torch.randn(n * ns, 1, device=dev)
            u_front = torch.rand(n * nf, 1, device=dev)
            u_behind = torch.rand(n * nb, 1, device=dev)
            coord, label, weight, color_label = ops.ray_samples(
                points.contiguous(), None if colors is None else colors.contiguous(), z_surf, u_front, u_behind, ns, nf, nb,
                sigma, c.free_sample_begin_ratio, c.free_sample_end_dist_m, c.max_range, c.dist_weight_on,
                c.dist_weight_scale, c.behind_dropoff_on)
            return coord, label, None, None, color_label, weight
        dist = torch.linalg.norm(points, dim=1, keepdim=True)  # [n,1]
        # same RNG draws, in the same order, as the reference sampler
        disp_surf = torch.randn(n * ns, 1, device=dev) * sigma
        d_f = dist.repeat(nf, 1)
        front_hi = 1.0 - 2.0 * sigma / d_f
        ratio_front = torch.rand(n * nf, 1, device=dev) * (front_hi - c.free_sample_begin_ratio) + c.free_sample_begin_ratio
        d_b = dist.repeat(nb, 1)
        behind_lo = 1.0 + 2.0 * sigma / d_b
        ratio_behind = torch.rand(n * nb, 1, device=dev) * (c.free_sample_end_dist_m / d_b + 1.0 - behind_lo) + behind_lo
        ratio = torch.cat((torch.ones_like(dist), disp_surf / dist.repeat(ns, 1) + 1.0, ratio_front, ratio_behind), 0)
        disp = torch.cat((torch.zeros_like(dist), disp_surf, (ratio_front - 1.0) * d_f, (ratio_behind - 1.0) * d_b), 0)
        d_all = dist.repeat(total, 1)
        coord = points.repeat(total, 1) * ratio
        weight = torch.ones_like(d_all)
        n_surf = n * (ns + 1)
        if c.dist_weight_on:
            weight[:n_surf] = 1 + c.dist_weight_scale * 0.5 - (d_all[:n_surf] / c.max_range) * c.dist_weight_scale
        if c.behind_dropoff_on:
            lo, hi = 0.2 * c.free_sample_end_dist_m, c.free_sample_end_dist_m
            weight = weight * (torch.clamp((hi - disp) / (hi - lo), 0.0, 1.0) * 0.8 + 0.2)
        weight[n_surf:] *= -1.0  # sign marks free-space samples
        # ray-major order: all samples of ray 0, then ray 1, ...
        by_ray = lambda t_, w: t_.reshape(total, n, w).transpose(0, 1).reshape(-1, w)  # noqa: E731
        coord = by_ray(coord, 3)
        label = -by_ray(disp, 1).squeeze(1)
        weight = by_ray(weight, 1).squeeze(1)
        normal_label = None if normals is None else by_ray(normals.repeat(total, 1), 3)
        color_label = None
        if colors is not None:
            cc = colors.shape[1]
            color_all = torch.cat((colors, colors.repeat(ns, 1), torch.zeros(n * (nf + nb), cc, device=dev)), 0)
            color_label = by_ray(color_all, cc)
        return coord, label, normal_label, None, color_label, weight


def allreduce_gradients(red):
    """Per-iteration exchange step of data-parallel map training (one process per GPU): ONE all-reduce (sum) over
    the contiguous buffer [feature grads | decoder grads | colour-feature grads | colour-decoder grads].  The loss
    heads already scaled d loss/d sdf by 1/world, so the sum is the global-batch mean gradient; every rank then
    applies the identical Adam step, keeping map features, decoder and optimiser state bit-identical."""
    import torch.distributed as dist

    dist.all_reduce(red, op=dist.ReduceOp.SUM)


def allreduce_map_statistics(cert_at_start, certainties, ts_update):
    """Once per mapping() call: the per-point certainty increments of all ranks are summed and the last-update
    timestamps max-reduced.  Neither feeds back into the training iterations (the reference only reads them
    between frames), so they do not need a collective per iteration."""
    import torch.distributed as dist

    delta = certainties - cert_at_start
    dist.all_reduce(delta, op=dist.ReduceOp.SUM)
    torch.add(cert_at_start, delta, out=certainties)
    dist.all_reduce(ts_update, op=dist.ReduceOp.MAX)


def _transform(points, pose):
    p = pose.to(points)
    return points @ p[:3, :3].T + p[:3, 3]


class _PoolArena:
    """Fixed-capacity storage behind the replay-pool tensors (SURVEY.md section 8 row f2).  The reference grows the
    pool with `torch.cat` and filters it with boolean masks: six multi-million-row reallocations per frame.  Here the
    public pool attributes of `Mapper` are views `[:count]` of one of two arenas: appending copies the new samples in
    place, the window filter compacts from the active arena into the other one (pinb200_pool_filter) and swaps."""

    FIELDS = (("coord", 3, torch.float32), ("gcoord", 3, torch.float32), ("label", 0, torch.float32),
              ("weight", 0, torch.float32), ("ts", 0, torch.int32))

    def __init__(self, device, color_channels: int, capacity_hint: int = 0):
        self.device, self.cc, self.hint = device, int(color_channels), int(capacity_hint)
        self.bufs, self.cap, self.count, self.cur = [None, None], 0, 0, 0
        self.scratch = self.counts = None

    def _alloc(self, cap):
        d = {n: torch.empty((cap, w) if w else (cap,), dtype=dt, device=self.device) for n, w, dt in self.FIELDS}
        d["color"] = torch.empty((cap, self.cc), dtype=torch.float32, device=self.device) if self.cc else None
        return d

    def reserve(self, need):
        if need <= self.cap and self.bufs[0] is not None:
            return
        # sized once for the configured pool capacity (config.pool_capacity samples + one frame of new samples: 36-48
        # bytes per sample, 1.5 GB for the 2e7-sample KITTI pool) so that a run never re-allocates: a cudaMalloc of a
        # few hundred MB costs ~25 ms, more than a whole frame
        cap = max(int(need * 1.5), 1 << 20, self.hint)
        old = self.bufs[self.cur]
        self.bufs = [self._alloc(cap), self._alloc(cap)]
        if old is not None and self.count:
            for n, t in old.items():
                if t is not None:
                    self.bufs[0][n][: self.count].copy_(t[: self.count])
        self.cap, self.cur = cap, 0

    def view(self, name):
        t = self.bufs[self.cur][name]
        return None if t is None else t[: self.count]

    def owns(self, name, t):
        b = None if self.bufs[self.cur] is None else self.bufs[self.cur][name]
        return b is not None and t is not None and t.data_ptr() == b.data_ptr() and t.shape[0] == self.count

    def load(self, tensors: dict):
        """Adopt pool tensors that were assigned from outside (tests, checkpoints, transform_data_pool)."""
        n = tensors["label"].shape[0]
        self.count = 0
        self.reserve(n)
        for name, t in tensors.items():
            if t is not None and self.bufs[self.cur][name] is not None:
                self.bufs[self.cur][name][:n].copy_(t)
        self.count = n

    def append(self, new: dict):
        n = new["label"].shape[0]
        self.reserve(self.count + n)
        for name, t in new.items():
            if t is not None and self.bufs[self.cur][name] is not None:
                self.bufs[self.cur][name][self.count: self.count + n].copy_(t)
        self.count += n

    def filter_window(self, origin64, radius2, n_tail):
        """Order-preserving compaction into the other arena; returns (kept, kept among the last n_tail) as ints."""
        lib = ops._lib.load()
        n = self.count
        need = int(lib.pinb200_pool_filter_scratch(max(n, 1)))
        if self.scratch is None or self.scratch.numel() < need:
            self.scratch = torch.empty((need,), dtype=torch.int32, device=self.device)
            self.counts = torch.empty((2,), dtype=torch.int64, device=self.device)
        a, b = self.bufs[self.cur], self.bufs[1 - self.cur]
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        rc = lib.pinb200_pool_filter(p(a["coord"]), p(a["gcoord"]), p(a["label"]), p(a["weight"]), p(a["ts"]), p(a["color"]),
                                     self.cc, n, int(n_tail), origin64.data_ptr(), float(radius2), p(b["coord"]),
                                     p(b["gcoord"]), p(b["label"]), p(b["weight"]), p(b["ts"]), p(b["color"]),
                                     self.scratch.data_ptr(), self.counts.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream)
        ops._lib.check(rc, "pinb200_pool_filter")
        ops._count(3)
        kept, tail = (int(v) for v in self.counts.tolist())  # the one host sync of the filter
        self.cur, self.count = 1 - self.cur, kept
        return kept, tail


class Mapper:
    def __init__(self, config, dataset, neural_points, decoders: dict):
        self.config = config
        self.silence = config.silence
        self.dataset = dataset
        self.neural_points = neural_points
        self.sdf_mlp = decoders["sdf"]
        self.sem_mlp = decoders.get("semantic")
        self.color_mlp = decoders.get("color")
        self.device = config.device
        self.dtype = config.dtype
        self.used_poses = None
        self.require_gradient = False
        self.total_iter = 0
        self.sdf_scale = config.logistic_gaussian_ratio * config.sigma_sigmoid_m
        self.sampler = DataSampler(config)
        self.ray_sample_count = 1 + config.surface_sample_n + config.free_behind_n + config.free_front_n
        self.new_idx = None
        self.ba_done_flag = False
        self.adaptive_iter_offset = 0
        self.static_mask = None
        self.cur_sample_count = 0
        self.pool_sample_count = 0
        self.last_losses = None
        self._work = {}
        self._batch = {}
        self.fused_allreduce = True  # data-parallel training: NCCL all-reduce issued by the library (one host call)
        self.init_pool()

    # ------------------------------------------------------------------ pool
    def init_pool(self):
        dev, dt = self.device, self.dtype
        self.coord_pool = torch.empty((0, 3), device=dev, dtype=dt)
        self.global_coord_pool = torch.empty((0, 3), device=dev, dtype=dt)
        self.sdf_label_pool = torch.empty((0,), device=dev, dtype=dt)
        self.color_pool = torch.empty((0, self.config.color_channel), device=dev, dtype=dt)
        self.sem_label_pool = None
        self.normal_label_pool = None
        self.weight_pool = torch.empty((0,), device=dev, dtype=dt)
        self.time_pool = torch.empty((0,), device=dev, dtype=torch.int32)

    def free_pool(self):
        self.coord_pool = self.weight_pool = self.sdf_label_pool = self.time_pool = None
        self.sem_label_pool = self.color_pool = self.normal_label_pool = None

    def determine_used_pose(self):
        cur = self.dataset.processed_frame
        src = None
        if getattr(self.config, "pgo_on", False):
            src = self.dataset.pgo_poses
        elif self.config.track_on:
            src = self.dataset.odom_poses
        elif self.dataset.gt_pose_provided:
            src = self.dataset.gt_poses
        if src is not None:
            self.used_poses = torch.as_tensor(src[: cur + 1], device=self.device, dtype=torch.float64)

    def transform_data_pool(self, pose_diff_torch):
        g = self.global_coord_pool
        if g.is_cuda and g.dtype == torch.float32 and g.is_contiguous():
            ops.frame_transform(g, self.time_pool.contiguous(), pose_diff_torch)  # in place, one streaming kernel
            return
        tf = pose_diff_torch[self.time_pool.long()].to(g)
        self.global_coord_pool = (tf[:, :3, :3] @ g.unsqueeze(-1)).squeeze(-1) + tf[:, :3, 3]

    # ------------------------------------------------------------------ per-frame preparation
    def dynamic_filter(self, points_torch, type_2_on: bool = True):
        """Static mask of a frame from the map's SDF and stability (reference: mapper.py:99-137)."""
        cfg = self.config
        o = self.neural_points.query_sdf(points_torch.contiguous(), self.sdf_mlp, need_grad=type_2_on)
        uncertain = o["certainty"] < cfg.dynamic_certainty_thre
        static = uncertain | (o["sdf"] < cfg.dynamic_sdf_ratio_thre * cfg.voxel_size_m)
        if type_2_on:
            static = static & ((o["grad"].norm(dim=-1) > cfg.dynamic_min_grad_norm_thre) | uncertain)
        return static

    def process_frame(self, point_cloud_torch, frame_label_torch, cur_pose_torch, frame_id: int,
                      filter_dynamic: bool = False):
        """Sample the frame, grow the map, append to the replay pool (reference: mapper.py:162-449)."""
        cfg = self.config
        origin = cur_pose_torch[:3, 3]
        orient = cur_pose_torch[:3, :3]
        pts = point_cloud_torch[:, :3]
        self.static_mask = torch.ones(pts.shape[0], dtype=torch.bool, device=self.device)
        if filter_dynamic:
            self.neural_points.reset_local_map(origin, orient, frame_id)
            self.static_mask = self.dynamic_filter(_transform(pts, cur_pose_torch))
            pts = pts[self.static_mask]
        colors = None
        if cfg.color_on:
            colors = point_cloud_torch[:, 3:]
            if filter_dynamic:
                colors = colors[self.static_mask]
        self.dataset.static_mask = self.static_mask

        coord, label, normal_label, _, color_label, weight = self.sampler.sample(pts, None, None, colors)
        stamps = torch.full((coord.shape[0],), frame_id, dtype=torch.int32, device=self.device)
        self.cur_sample_count = label.shape[0]
        self.pool_sample_count = self.sdf_label_pool.shape[0]

        if cfg.from_sample_points:
            if cfg.from_all_samples:
                grow_pts = coord
            else:
                near = torch.abs(label) < cfg.surface_sample_range_m * cfg.map_surface_ratio
                grow_pts = _transform(coord[near], cur_pose_torch)
        else:
            grow_pts = _transform(pts, cur_pose_torch)
        if cfg.prune_map_on and ((frame_id + 1) % cfg.prune_freq_frame == 0):
            if self.neural_points.prune_map(cfg.max_prune_certainty):
                self.neural_points.recreate_hash(None, None, True, True, frame_id)
        self.cur_new_point_ratio = self.neural_points.update(grow_pts, origin, orient, frame_id)
        self.neural_points.record_memory(verbose=(not self.silence))

        self.determine_used_pose()
        on_gpu = coord.is_cuda
        if on_gpu:
            # fixed-capacity arenas behind the pool tensors (no per-frame reallocation), pinb200_pool_filter below
            P = self.__dict__.get("_pool")
            cc = 0 if color_label is None else color_label.shape[1]
            if P is None or P.cc != cc:
                P = self._pool = _PoolArena(self.device, cc, min(int(cfg.pool_capacity), 30_000_000) + 2_000_000)
            cur = {"coord": self.coord_pool, "gcoord": self.global_coord_pool, "label": self.sdf_label_pool,
                   "weight": self.weight_pool, "ts": self.time_pool, "color": self.color_pool if cc else None}
            if not all(P.owns(k, v) for k, v in cur.items() if v is not None and (k != "color" or cc)):
                P.load(cur)
            P.append({"coord": coord, "gcoord": _transform(coord, cur_pose_torch), "label": label, "weight": weight,
                      "ts": stamps, "color": color_label})
            self._bind_pool(P)
            if self.ba_done_flag:
                tf = self.used_poses[self.time_pool.long()].to(self.coord_pool)
                self.global_coord_pool.copy_((tf[:, :3, :3] @ self.coord_pool.unsqueeze(-1)).squeeze(-1) + tf[:, :3, 3])
                self.ba_done_flag = False
        else:
            self.coord_pool = torch.cat((self.coord_pool, coord), 0)
            self.weight_pool = torch.cat((self.weight_pool, weight), 0)
            self.sdf_label_pool = torch.cat((self.sdf_label_pool, label), 0)
            self.time_pool = torch.cat((self.time_pool, stamps), 0)
            self.color_pool = torch.cat((self.color_pool, color_label), 0) if color_label is not None else None
            if self.ba_done_flag:
                tf = self.used_poses[self.time_pool.long()].to(self.coord_pool)
                self.global_coord_pool = (tf[:, :3, :3] @ self.coord_pool.unsqueeze(-1)).squeeze(-1) + tf[:, :3, 3]
                self.ba_done_flag = False
            else:
                self.global_coord_pool = torch.cat((self.global_coord_pool, _transform(coord, cur_pose_torch)), 0)

        if (frame_id + 1) % cfg.pool_filter_freq == 0 and on_gpu:
            kept, tail = P.filter_window(origin.to(torch.float64).contiguous(), cfg.window_radius**2, self.cur_sample_count)
            self._bind_pool(P)
            self.cur_sample_count, self.pool_sample_count = tail, kept
            if kept > cfg.pool_capacity:  # rare: random down-sampling of an over-full window (mapper.py:418-424)
                drop = torch.randint(0, kept, (kept - cfg.pool_capacity,), device=self.device)
                keep = torch.ones(kept, dtype=torch.bool, device=self.device)
                keep[drop] = False
                tens = {"coord": self.coord_pool[keep], "gcoord": self.global_coord_pool[keep],
                        "label": self.sdf_label_pool[keep], "weight": self.weight_pool[keep], "ts": self.time_pool[keep],
                        "color": self.color_pool[keep] if P.cc else None}
                self.cur_sample_count = int(keep[-self.cur_sample_count:].sum().item())
                P.load(tens)
                self._bind_pool(P)
                self.pool_sample_count = P.count
        elif (frame_id + 1) % cfg.pool_filter_freq == 0:
            keep = ((self.global_coord_pool - origin) ** 2).sum(-1) < cfg.window_radius**2
            alive = torch.nonzero(keep).squeeze(-1)
            if alive.shape[0] > cfg.pool_capacity:
                drop = torch.randint(0, alive.shape[0], (alive.shape[0] - cfg.pool_capacity,), device=self.device)
                keep[alive[drop]] = False
            self.coord_pool = self.coord_pool[keep]
            self.global_coord_pool = self.global_coord_pool[keep]
            self.sdf_label_pool = self.sdf_label_pool[keep]
            self.weight_pool = self.weight_pool[keep]
            self.time_pool = self.time_pool[keep]
            if self.color_pool is not None:
                self.color_pool = self.color_pool[keep]
            self.cur_sample_count = int(keep[-self.cur_sample_count:].sum().item())
            self.pool_sample_count = int(keep.sum().item())
        else:
            self.cur_sample_count = coord.shape[0]
            self.pool_sample_count = self.coord_pool.shape[0]

        if cfg.bs_new_sample > 0:
            fresh = self.global_coord_pool[-self.cur_sample_count:]
            fresh_label = self.sdf_label_pool[-self.cur_sample_count:]
            self.neural_points.set_search_neighborhood(num_nei_cells=1, search_alpha=0.0)
            certainty = self.neural_points.query_certainty(fresh.contiguous())
            self.neural_points.set_search_neighborhood(num_nei_cells=cfg.num_nei_cells, search_alpha=cfg.search_alpha)
            self.new_idx = torch.where((certainty < cfg.new_certainty_thre) &
                                       (torch.abs(fresh_label) < cfg.surface_sample_range_m * 3.0))[0]
            self.new_idx += self.pool_sample_count - self.cur_sample_count
            self.adaptive_iter_offset = 0
            if cfg.adaptive_iters:
                ratio = self.new_idx.shape[0] / max(1, self.cur_sample_count)
                if ratio < cfg.new_sample_ratio_less:
                    self.adaptive_iter_offset = -5
                elif ratio > cfg.new_sample_ratio_more:
                    self.adaptive_iter_offset = 5
                    if frame_id > cfg.freeze_after_frame and ratio > cfg.new_sample_ratio_restart:
                        self.adaptive_iter_offset = 10

    def _bind_pool(self, P):
        self.coord_pool, self.global_coord_pool = P.view("coord"), P.view("gcoord")
        self.sdf_label_pool, self.weight_pool, self.time_pool = P.view("label"), P.view("weight"), P.view("ts")
        self.color_pool = P.view("color") if P.cc else None

    # ------------------------------------------------------------------ batches
    def draw_batch_index(self, bs=None):
        """The batch draw of the reference (mapper.py:452-480): same torch.randint calls, same RNG stream."""
        cfg = self.config
        bs = cfg.bs if bs is None else bs
        lose = getattr(self.dataset, "lose_track", False) or getattr(self.dataset, "stop_status", False)
        if cfg.bs_new_sample > 0 and self.new_idx is not None and not lose and self.new_idx.shape[0] > 0:
            n_new = min(self.new_idx.shape[0], cfg.bs_new_sample)
            hist = torch.randint(0, self.pool_sample_count, (bs - n_new,), device=self.device)
            pick = torch.randint(0, self.new_idx.shape[0], (n_new,), device=self.device)
            return torch.cat((hist, self.new_idx[pick]), dim=0)
        return torch.randint(0, self.pool_sample_count, (bs,), device=self.device)

    def get_batch(self, global_coord=False, bs=None):
        """Reference-compatible batch tuple (mapper.py:452-503)."""
        index = self.draw_batch_index(bs)
        coord = (self.global_coord_pool if global_coord else self.coord_pool)[index, :]
        has_color = self.color_pool is not None and self.color_pool.shape[0] == self.sdf_label_pool.shape[0]
        color = self.color_pool[index] if has_color else None
        return coord, self.sdf_label_pool[index], self.time_pool[index], None, None, color, self.weight_pool[index]

    # ------------------------------------------------------------------ queries
    def sdf(self, x, get_std=False, min_nn_count=1, accumulate_stability=False):
        o = self.neural_points.query_sdf(x.contiguous(), self.sdf_mlp, need_grad=False,
                                         training_mode=accumulate_stability)
        return o["sdf"], (o["sdf_std"] if (get_std and not self.config.weighted_first) else None), \
            o["nn_count"] >= min_nn_count

    def sdf_batch(self, x, bs, get_std=False, min_nn_count=1, accumulate_stability=False):
        return self.sdf(x, get_std, min_nn_count, accumulate_stability)  # one launch covers any batch size

    def get_numerical_gradient(self, x, sdf_x=None, eps=0.02, two_side=True):
        e = torch.eye(3, device=x.device, dtype=x.dtype) * eps
        n = x.shape[0]
        if two_side:
            s = self.sdf(torch.cat([x + e[0], x - e[0], x + e[1], x - e[1], x + e[2], x - e[2]], 0))[0]
            return torch.stack([(s[0:n] - s[n:2 * n]), (s[2 * n:3 * n] - s[3 * n:4 * n]),
                                (s[4 * n:5 * n] - s[5 * n:])], 1) / (2 * eps)
        s = self.sdf(torch.cat([x + e[0], x + e[1], x + e[2]], 0))[0]
        return torch.stack([s[0:n] - sdf_x, s[n:2 * n] - sdf_x, s[2 * n:] - sdf_x], 1) / eps

    # ------------------------------------------------------------------ training
    def _decoder_trainable(self):
        return any(p.requires_grad for p in self.sdf_mlp.parameters())

    def mapping(self, iter_count):
        """Reference: utils/mapper.py:600-844."""
        cfg = self.config
        if not (cfg.main_loss_type == "bce" and cfg.numerical_grad and cfg.opt_adam):
            raise NotImplementedError("the CUDA mapper supports the reference defaults: bce loss, numerical Eikonal, Adam")
        iter_count = max(1, iter_count + self.adaptive_iter_offset)
        npm = self.neural_points
        feat = npm.local_geo_features.data
        dev = feat.device
        dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()
        world = torch.distributed.get_world_size() if dist_on else 1
        train_dec = self._decoder_trainable()
        flat = self.sdf_mlp.flat_parameters()  # decoder weights live in (and are views of) this vector
        n_dec = flat.numel()
        m_rows = npm.local_count()
        color_on = bool(cfg.color_on and cfg.weight_i > 0 and self.color_mlp is not None and self.color_pool is not None
                        and self.color_pool.shape[0] > 0)
        cfeat = npm.local_color_features.data if color_on else None
        cflat = self.color_mlp.flat_parameters() if color_on else None
        n_cf = cfeat.numel() if color_on else 0
        n_cd = cflat.numel() if color_on else 0
        train_cdec = color_on and any(p.requires_grad for p in self.color_mlp.parameters())
        # ONE zero-filled arena: [feature grads | decoder grads | colour-feature grads | colour-decoder grads]
        # (the data-parallel reduction buffer `red`), then the Adam moments of the same four blocks, then the
        # loss accumulators
        n_red = feat.numel() + n_dec + n_cf + n_cd
        arena = torch.zeros(3 * n_red + 4, device=dev, dtype=torch.float32)
        red, m_all, v_all = arena[:n_red], arena[n_red: 2 * n_red], arena[2 * n_red: 3 * n_red]
        o0, o1, o2 = feat.numel(), feat.numel() + n_dec, feat.numel() + n_dec + n_cf
        gfeat, mf, vf = (b[:o0].view_as(feat) for b in (red, m_all, v_all))
        gdec, md, vd = (b[o0:o1] for b in (red, m_all, v_all))
        gcfeat = gcdec = mcf = vcf = mcd = vcd = closs = None
        if color_on:
            gcfeat, mcf, vcf = (b[o1:o2].view_as(cfeat) for b in (red, m_all, v_all))
            gcdec, mcd, vcd = (b[o2:n_red] for b in (red, m_all, v_all))
            closs = arena[3 * n_red + 2: 3 * n_red + 3]
        losses = arena[3 * n_red: 3 * n_red + 2]
        cert_at_start = npm.local_point_certainties.clone() if dist_on else None
        dec_step = cfg.gradient_decimation
        eik_on = cfg.ekional_loss_on and cfg.weight_e > 0
        eps_num = cfg.voxel_size_m * cfg.num_grad_step_ratio
        shifts = None
        out = self._work
        stock_batches = (type(self).get_batch is Mapper.get_batch and "get_batch" not in self.__dict__
                         and not self.ba_done_flag)
        if stock_batches and not color_on:
            # the loop from ONE host call (two per iteration when the gradients are all-reduced in between): the
            # batch indices are drawn up front -- same torch.randint calls in the same order as the reference,
            # nothing else consumes the RNG in between
            index = torch.stack([self.draw_batch_index() for _ in range(iter_count)])
            kw = dict(nn_k=cfg.query_nn_k, weighted_first=cfg.weighted_first, coord_pool=self.global_coord_pool,
                      label_pool=self.sdf_label_pool, ts_pool=self.time_pool, weight_pool=self.weight_pool,
                      decimation=dec_step if eik_on else 0, eik_eps=eps_num, sigma=self.sdf_scale,
                      weight_e=cfg.weight_e, loss_weight_on=cfg.loss_weight_on, lr=cfg.lr, beta1=0.9, beta2=0.99,
                      eps=cfg.adam_eps, weight_decay=cfg.weight_decay, train_decoder=train_dec, feat=feat,
                      dec_flat=flat, grad_feat=gfeat, grad_dec=gdec, m_feat=mf, v_feat=vf, m_dec=md, v_dec=vd,
                      losses=losses, work=out)
            mh, dh = npm.map_handle(True), self.sdf_mlp.handle()
            if not dist_on:
                ops.map_iterations(mh, dh, iter_count, index=index, first_step=1, **kw)
            elif torch.distributed.get_backend() == "nccl" and self.fused_allreduce:
                # data parallel, still ONE host call: the library enqueues the NCCL all-reduce of `red` on the
                # kernel stream between the backward and the Adam kernels of every iteration
                comm = ops.NcclComm.get(dev)
                ops.map_iterations(mh, dh, iter_count, index=index, first_step=1, grad_scale=1.0 / world,
                                   nccl_comm=comm, reduce_buf=red, **kw)
            else:
                for it in range(iter_count):
                    ops.map_iterations(mh, dh, 1, index=index[it:it + 1], first_step=it + 1, stages=1,
                                       grad_scale=1.0 / world, **kw)
                    allreduce_gradients(red)
                    ops.map_iterations(mh, dh, 1, index=index[it:it + 1], first_step=it + 1, stages=2, **kw)
            self.total_iter += iter_count
            iter_count = 0
        for it in range(iter_count):
            fused_batch = stock_batches
            if fused_batch:
                # one launch: pool gathers + the 6 shifted numerical-gradient copies of every dec_step-th sample
                index = self.draw_batch_index()
                has_color = color_on and self.color_pool.shape[0] == self.sdf_label_pool.shape[0]
                rows, label, ts, weight, color_label, ne = ops.assemble_batch(
                    self.global_coord_pool, self.sdf_label_pool, self.time_pool, self.weight_pool,
                    self.color_pool if has_color else None, index, dec_step if eik_on else 0, eps_num, self._batch)
                n = index.shape[0]
            else:
                coord, label, ts, _, _, color_label, weight = self.get_batch(global_coord=not self.ba_done_flag)
                if self.ba_done_flag:
                    tf = self.used_poses[ts.long()].to(coord)
                    coord = (tf[:, :3, :3] @ coord.unsqueeze(-1)).squeeze(-1) + tf[:, :3, 3]
                n = coord.shape[0]
                if eik_on:
                    if shifts is None:
                        e = eps_num
                        shifts = torch.tensor([[e, 0, 0], [-e, 0, 0], [0, e, 0], [0, -e, 0], [0, 0, e], [0, 0, -e]],
                                              device=dev, dtype=torch.float32).unsqueeze(1)
                    sub = coord[::dec_step]
                    ne = sub.shape[0]
                    rows = torch.cat((coord, (sub.unsqueeze(0) + shifts).reshape(-1, 3)), 0)
                else:
                    ne = 0
                    rows = coord.contiguous()
            o = ops.query_sdf(npm.map_handle(True), self.sdf_mlp.handle(), rows, nn_k=cfg.query_nn_k,
                              weighted_first=cfg.weighted_first, training_mode=True, training_rows=n, need_grad=False,
                              query_ts=ts.contiguous(), save_knn=True, out=out,
                              color_dec=self.color_mlp.handle(sigmoid_out=True) if color_on else None)
            dl = out.get("dl")
            if dl is None or dl.shape[0] != rows.shape[0]:
                dl = out["dl"] = torch.empty(rows.shape[0], device=dev)
            ops.mapping_loss(o["sdf"], label.contiguous(), weight.contiguous(), n, ne, self.sdf_scale,
                             cfg.loss_weight_on, cfg.weight_e if eik_on else 0.0, eps_num, dl, losses,
                             grad_scale=1.0 / world)
            ops.train_backward(npm.map_handle(True), self.sdf_mlp.handle(), feat, rows, o["knn_idx"], o["knn_weight"],
                               dl, cfg.weighted_first, gfeat, gdec)
            if color_on:  # colour head: L1 on surface samples (mapper.py:804-812), its own backward through K2
                label_c, weight_c = label.contiguous(), weight.contiguous()
                n_surf = (label_c.abs() < cfg.surface_sample_range_m).sum().float().reshape(1)
                dlc = torch.empty((n, self.color_mlp.out_dim), device=dev)
                ops.color_loss(o["color"][:n], color_label.contiguous(), label_c, weight_c, cfg.surface_sample_range_m,
                               cfg.loss_weight_on, cfg.weight_i, n_surf, dlc, closs, grad_scale=1.0 / world)
                ops.train_backward(npm.map_handle(True), self.color_mlp.handle(sigmoid_out=True), cfeat, rows[:n],
                                   o["knn_idx"][:n], o["knn_weight"][:n], dlc, cfg.weighted_first, gcfeat, gcdec)
            if dist_on:
                allreduce_gradients(red)
            if train_dec:
                ops.adam_step(flat, gdec, md, vd, cfg.lr, 0.9, 0.99, cfg.adam_eps, 0.0, it + 1)
            else:
                gdec.zero_()
            ops.adam_step(feat, gfeat, mf, vf, cfg.lr, 0.9, 0.99, cfg.adam_eps, cfg.weight_decay, it + 1)
            if color_on:
                if train_cdec:
                    ops.adam_step(cflat, gcdec, mcd, vcd, cfg.lr, 0.9, 0.99, cfg.adam_eps, 0.0, it + 1)
                else:
                    gcdec.zero_()
                ops.adam_step(cfeat, gcfeat, mcf, vcf, cfg.lr, 0.9, 0.99, cfg.adam_eps, cfg.weight_decay, it + 1)
            self.total_iter += 1
        if dist_on:
            allreduce_map_statistics(cert_at_start, npm.local_point_certainties, npm.local_point_ts_update)
        self.last_losses = losses
        npm.assign_local_to_global()

    def allreduce_floats(self):
        """Size of the per-iteration data-parallel exchange (feature + decoder [+ colour] gradient blocks)."""
        n = self.neural_points.local_geo_features.numel() + self.sdf_mlp.flat_parameters().numel()
        if self.config.color_on and self.color_mlp is not None:
            n += self.neural_points.local_color_features.numel() + self.color_mlp.flat_parameters().numel()
        return n

    def bundle_adjustment(self, iter_count, window_size: int = 50, use_lie_group: bool = False):
        raise NotImplementedError("local bundle adjustment (pypose) is outside the CUDA hot path (SURVEY.md section 2 #4)")
