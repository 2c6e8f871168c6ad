"""Drop-in `NeuralPoints` for PIN-SLAM backed by the sm_90a kernels.

Keeps the Python surface of the reference class (model/neural_points.py:29 of
PRBonn/PIN_SLAM: constructor, tensor attribute names, method names, argument
meaning, return tuples) so that `pin_slam.py` and the reference's tracker /
mapper / mesher / GUI code run against it unchanged, and adds the fused entry
points the CUDA tracker / mapper use:

    query_sdf(...)        one launch: voxel-hash kNN + IDW + decoder (+ d/dx)   [K1]
    map_handle(...)       the plain-C view of the map handed to the kernels

Differences in storage (values identical to the reference):
  * `buffer_pt_index` and `global2local` are int32 (the reference uses int64):
    half the footprint of the 5e7-slot table, and what the kernels read directly;
  * there is no CPU path: the map lives on a CUDA device and every query runs a
    kernel from libpinb200.so (a missing library raises, nothing falls back).

Map maintenance: voxel down-sampling, map growth (`update`, into fixed-capacity
arenas), the local-map reset and the loop-closure point transform run as kernels
(SURVEY.md section 8 f1 / f4); prune / rehash are host-orchestrated PyTorch.  The RNG
stream is consumed exactly like the reference (randn for the new feature rows even
when feature_std == 0).
"""
import sys

import torch
import torch.nn as nn

from .. import ops

_PRIMES = (73856093, 19349669, 83492791)


def _quat_rotate_passive(quat, v):
    """Rotate v into the frame of the (unit) quaternion wxyz -- conjugate rotation."""
    w = quat[..., :1]
    u = -quat[..., 1:]
    t = 2.0 * torch.linalg.cross(u, v)
    return v + w * t + torch.linalg.cross(u, t)


def _put_last(table: torch.Tensor, slots: torch.Tensor, vals: torch.Tensor) -> None:
    """table[slots] = vals with sequential semantics: where a slot repeats, the last write wins.  A plain index_put
    with duplicate indices leaves the winner unspecified (on the CPU it depends on the thread count)."""
    slots = slots.long()
    pos = torch.arange(slots.numel(), device=slots.device)
    last = torch.full(table.shape, -1, dtype=torch.int64, device=slots.device)
    last.scatter_reduce_(0, slots, pos, reduce="amax")
    keep = last[slots] == pos
    table[slots[keep]] = vals[keep]


def voxel_down_sample(points: torch.Tensor, voxel_size: float) -> torch.Tensor:
    """Index of the point closest to each occupied voxel's centre.

    Same selection rule and output order as the reference helper
    (utils/tools.py:583-626): voxel key x + y*v + z*v^2 over the offset grid,
    centre distance quantised to 1000 levels, ties broken by the smaller index,
    result ordered by ascending voxel key.  CUDA tensors go through pinb200_voxel_downsample (a lock-free hash set
    instead of torch.unique over the whole frame: section 8 row f1); the torch formulation below is the CPU form
    the golden fixtures pin."""
    if points.is_cuda:
        return ops.voxel_downsample(points, voxel_size)
    grid = torch.floor(points / voxel_size)
    centre = (grid + 0.5) * voxel_size
    dist = ((points - centre) ** 2).sum(dim=1) ** 0.5
    q = (dist / dist.max() * 999).long()
    origin = torch.floor(points.min(dim=0)[0] / voxel_size).long()
    g = grid.long() - origin
    v = g.max()
    key = g[:, 0] + g[:, 1] * v + g[:, 2] * v * v
    uniq, inv = torch.unique(key, return_inverse=True)
    n = points.shape[0]
    packed = q * n + torch.arange(n, device=points.device)  # lexicographic (quantised distance, index)
    best = torch.full((uniq.shape[0],), torch.iinfo(torch.int64).max, dtype=torch.int64, device=points.device)
    best.scatter_reduce_(0, inv, packed, reduce="amin", include_self=True)
    return best % n


def voxel_down_sample_min_value(points: torch.Tensor, voxel_size: float, value: torch.Tensor) -> torch.Tensor:
    """Index of the point with the smallest `value` in each occupied voxel, `value` quantised to 1000 levels of its
    maximum and ties broken by the smaller index -- the selection rule of the reference helper
    (utils/tools.py:629-668 voxel_down_sample_min_value_torch), result ordered by ascending voxel key."""
    if points.is_cuda:
        return ops.voxel_downsample(points, voxel_size, value)
    origin = torch.floor(points.min(dim=0)[0] / voxel_size).long()
    g = torch.floor(points / voxel_size).long() - origin
    v = g.max()
    key = g[:, 0] + g[:, 1] * v + g[:, 2] * v * v
    uniq, inv = torch.unique(key, return_inverse=True)
    n = points.shape[0]
    q = (value / value.max() * 999).long()
    packed = q * n + torch.arange(n, device=points.device)  # lexicographic (quantised value, index)
    best = torch.full((uniq.shape[0],), torch.iinfo(torch.int64).max, dtype=torch.int64, device=points.device)
    best.scatter_reduce_(0, inv, packed, reduce="amin", include_self=True)
    return best % n


class _MapArena:
    """Fixed-capacity storage behind the global map tensors (SURVEY.md section 8 row f1).  The reference grows seven
    tensors with torch.cat every frame; here `NeuralPoints.neural_points`, `.point_orientations`, `.point_ts_create`,
    `.point_ts_update`, `.point_certainties`, `.geo_features` (+ pad row) and `.color_features` are views `[:count]` of
    these buffers and pinb200_map_grow appends in place.  Tensors assigned from outside (pruning, rehash, loop
    closure, checkpoints, tests) are adopted on the next update."""

    NAMES = ("neural_points", "point_orientations", "point_ts_create", "point_ts_update", "point_certainties")

    def __init__(self):
        self.buf, self.cap = None, 0

    def owns(self, npm):
        if self.buf is None:
            return False
        for name in self.NAMES + ("geo_features",):
            if getattr(npm, name).data_ptr() != self.buf[name].data_ptr():
                return False
        return npm.color_features is None or npm.color_features.data_ptr() == self.buf["color_features"].data_ptr()

    def reserve(self, npm, rows):
        if self.owns(npm) and rows <= self.cap:
            return
        n, dev = npm.count(), npm.neural_points.device
        cap = max(int(rows * 1.5) + 4096, 1 << 16)
        new = {"neural_points": torch.empty((cap, 3), dtype=torch.float32, device=dev),
               "point_orientations": torch.empty((cap, 4), dtype=torch.float32, device=dev),
               "point_ts_create": torch.empty((cap,), dtype=torch.int32, device=dev),
               "point_ts_update": torch.empty((cap,), dtype=torch.int32, device=dev),
               "point_certainties": torch.empty((cap,), dtype=torch.float32, device=dev),
               "geo_features": torch.empty((cap + 1, npm.geo_features.shape[1]), dtype=torch.float32, device=dev),
               "color_features": None if npm.color_features is None else
               torch.empty((cap + 1, npm.color_features.shape[1]), dtype=torch.float32, device=dev)}
        for name in self.NAMES:
            new[name][:n].copy_(getattr(npm, name))
        new["geo_features"][: n + 1].copy_(npm.geo_features)
        if npm.color_features is not None:
            new["color_features"][: n + 1].copy_(npm.color_features)
        self.buf, self.cap = new, cap
        self.bind(npm, n)

    def bind(self, npm, n):
        for name in self.NAMES:
            setattr(npm, name, self.buf[name][:n])
        npm.geo_features = self.buf["geo_features"][: n + 1]
        if self.buf["color_features"] is not None:
            npm.color_features = self.buf["color_features"][: n + 1]


class NeuralPoints(nn.Module):
    STRICT_REFERENCE_G2L = True  # reproduce the reference's global2local fill value (see reset_local_map)

    def __init__(self, config) -> None:
        super().__init__()
        self.config = config
        self.silence = config.silence
        self.geo_feature_dim = config.feature_dim
        self.geo_feature_std = config.feature_std
        self.color_feature_dim = config.feature_dim
        self.color_feature_std = config.feature_std
        if getattr(config, "pos_encoding_band", 0) > 0 or getattr(config, "layer_norm_on", False):
            raise NotImplementedError("pin_slam_b200: positional encoding / feature layer-norm are not supported")
        self.mean_grid_sampling = False
        self.device = config.device
        self.dtype = config.dtype
        self.idx_dtype = torch.int32
        self.resolution = config.voxel_size_m
        self.buffer_size = int(config.buffer_size)
        self.temporal_local_map_on = True
        self.local_map_radius = self.config.local_map_radius
        self.diff_travel_dist_local = self.config.local_map_radius * self.config.local_map_travel_dist_ratio
        self.diff_ts_local = self.config.diff_ts_local
        self.reboot_ts = 0
        self.local_orientation = torch.eye(3, device=self.device)
        self.cur_ts = 0
        self.max_ts = 0
        self._travel_dist = None
        self.est_poses = None
        self.after_pgo = False
        self.primes = torch.tensor(_PRIMES, dtype=torch.int64, device=self.device)

        self.buffer_pt_index = torch.full((self.buffer_size,), -1, dtype=torch.int32, device=self.device)
        f = self.geo_feature_dim
        self.neural_points = torch.empty((0, 3), dtype=self.dtype, device=self.device)
        self.point_orientations = torch.empty((0, 4), dtype=self.dtype, device=self.device)
        self.geo_features = torch.empty((1, f), dtype=self.dtype, device=self.device)
        self.color_on = bool(config.color_on)
        self.color_features = torch.empty((1, f), dtype=self.dtype, device=self.device) if self.color_on else None
        self.geo_feature_pca = self.color_feature_pca = None
        self.point_ts_create = torch.empty((0,), device=self.device, dtype=torch.int32)
        self.point_ts_update = torch.empty((0,), device=self.device, dtype=torch.int32)
        self.point_certainties = torch.empty((0,), dtype=self.dtype, device=self.device)

        self.local_neural_points = torch.empty((0, 3), dtype=self.dtype, device=self.device)
        self.local_point_orientations = torch.empty((0, 4), dtype=self.dtype, device=self.device)
        self.local_geo_features = nn.Parameter()
        self.local_color_features = nn.Parameter()
        self.local_point_certainties = torch.empty((0,), dtype=self.dtype, device=self.device)
        self.local_point_ts_update = torch.empty((0,), device=self.device, dtype=torch.int32)
        self.local_mask = None
        self._local_idx = None
        self.global2local = None

        self._handles = {}
        self._rec_tables = {}  # index space (local / global) -> [buffer_size, 4] probe-record table, reused across frames
        self.set_search_neighborhood(num_nei_cells=config.num_nei_cells, search_alpha=config.search_alpha)
        self.cur_memory_mb = 0.0
        self.memory_footprint = []
        self.to(self.device)

    # ---------------------------------------------------------------- bookkeeping
    @property
    def travel_dist(self):
        return self._travel_dist

    @travel_dist.setter
    def travel_dist(self, value):  # pin_slam.py:275 assigns a fresh tensor every frame
        self._travel_dist = value
        self._handles = {}

    def _invalidate(self, slots_freed: bool = False):
        """Drop the cached kernel views.  `slots_freed`: hash slots may have been emptied (rehash / pruning), so the
        probe-record tables must be cleared before they are rebuilt (ops.MapHandle.ensure_records)."""
        self._handles = {}
        if slots_freed:
            self._rec_tables = {}

    def is_empty(self):
        return self.neural_points.shape[0] == 0

    def count(self):
        return self.neural_points.shape[0]

    def local_count(self):
        return 0 if self.local_neural_points is None else self.local_neural_points.shape[0]

    def record_memory(self, verbose: bool = True, record_footprint: bool = True):
        dim = self.geo_feature_dim + 3 + 4 + (self.color_feature_dim if self.color_features is not None else 0)
        self.cur_memory_mb = self.count() * dim * 4 / 1024 / 1024
        if verbose:
            print("# Global neural point: %d" % self.count())
            print("# Local  neural point: %d" % self.local_count())
            print("Current map memory consumption: {:.3f} MB".format(self.cur_memory_mb))
        if record_footprint:
            self.memory_footprint.append(self.cur_memory_mb)

    def compute_feature_principle_components(self, down_rate: int = 1):
        def pca(x):
            x = x[::down_rate]
            x = x - x.mean(dim=0, keepdim=True)
            _, _, vh = torch.linalg.svd(x, full_matrices=False)
            return vh[:3].T

        self.geo_feature_pca = pca(self.local_geo_features.detach()[:-1])
        if self.color_features is not None:
            self.color_feature_pca = pca(self.local_color_features.detach()[:-1])

    def get_neural_points_o3d(self, query_global: bool = True, color_mode: int = -1, random_down_ratio: int = 1):
        import open3d as o3d  # visualisation only; not part of the hot path

        pts = self.neural_points if query_global else self.local_neural_points
        pc = o3d.geometry.PointCloud()
        pc.points = o3d.utility.Vector3dVector(pts[::random_down_ratio].detach().cpu().numpy().astype("float64"))
        return pc

    def get_map_o3d_bbx(self):
        import open3d as o3d

        lo = self.neural_points.min(dim=0)[0].cpu().numpy()
        hi = self.neural_points.max(dim=0)[0].cpu().numpy()
        return o3d.geometry.AxisAlignedBoundingBox(lo, hi)

    # ---------------------------------------------------------------- hashing
    def _slots(self, pts: torch.Tensor) -> torch.Tensor:
        """Hash slot of each point's voxel, already wrapped to [0, buffer_size)."""
        cell = (pts / self.resolution).floor().to(torch.int64)
        h = torch.fmod((cell * self.primes).sum(-1), self.buffer_size)
        return torch.where(h < 0, h + self.buffer_size, h)

    _NEIGHBORHOODS = {}  # (num_nei_cells, search_alpha, device) -> (neighbor_dx int64, int32 copy)

    def set_search_neighborhood(self, num_nei_cells: int = 1, search_alpha: float = 1.0):
        # the mapper switches to the 7-cell neighbourhood and back around its certainty pass every frame
        # (utils/mapper.py:388-402): the offset tables are cached, building them costs ~10 torch ops and a host sync
        key = (int(num_nei_cells), float(search_alpha), str(self.device))
        hit = NeuralPoints._NEIGHBORHOODS.get(key)
        if hit is None:
            r = torch.arange(-num_nei_cells, num_nei_cells + 1, device=self.device, dtype=torch.int64)
            cells = torch.stack(torch.meshgrid(r, r, r, indexing="ij"), dim=-1).reshape(-1, 3)
            inside = (cells**2).sum(-1) < (num_nei_cells + search_alpha) ** 2
            dx = cells[inside]
            hit = NeuralPoints._NEIGHBORHOODS[key] = (dx, dx.to(torch.int32).contiguous())
        self.neighbor_dx, self._probe_dx32 = hit
        self.neighbor_K = self.neighbor_dx.shape[0]
        self.max_valid_dist2 = 3 * ((num_nei_cells + 1) * self.resolution) ** 2
        self._invalidate()

    # ---------------------------------------------------------------- map growth
    def update(self, points: torch.Tensor, sensor_position: torch.Tensor, sensor_orientation: torch.Tensor,
               cur_ts: int):
        res = self.resolution
        pick = voxel_down_sample(points, res)
        cand = points[pick]
        if cand.is_cuda and cand.dtype == torch.float32 and self.neural_points.dtype == torch.float32:
            return self._update_device(cand.contiguous(), sensor_position, sensor_orientation, cur_ts)
        slot = self._slots(cand)
        owner = self.buffer_pt_index[slot].long()
        if (not self.is_empty()) and (cur_ts != self.reboot_ts):
            d2 = ((self.neural_points[owner] - cand) ** 2).sum(-1)  # owner == -1 reads the last point, masked below
            grow = (owner == -1) | (d2 > 3 * res**2)
            if self.temporal_local_map_on:
                age = self.travel_dist[cur_ts] - self.travel_dist[self.point_ts_update[owner].long()]
                grow = grow | (age > self.diff_travel_dist_local)
        else:
            grow = torch.ones(owner.shape, dtype=torch.bool, device=self.device)
        fresh = cand[grow]
        n_new = fresh.shape[0]
        ratio = n_new / cand.shape[0]
        base = self.neural_points.shape[0]
        owner[grow] = torch.arange(n_new, dtype=torch.int64, device=self.device) + base
        self.buffer_pt_index[slot] = owner.to(torch.int32)
        self.neural_points = torch.cat((self.neural_points, fresh), 0)
        ident = torch.zeros((n_new, 4), dtype=self.dtype, device=self.device)
        ident[:, 0] = 1.0
        self.point_orientations = torch.cat((self.point_orientations, ident), 0)
        stamp = torch.full((n_new,), cur_ts, device=self.device, dtype=torch.int32)
        self.point_ts_create = torch.cat((self.point_ts_create, stamp), 0)
        self.point_ts_update = torch.cat((self.point_ts_update, stamp), 0)
        # one extra (padding) row; the randn draw is kept even at std 0 so the RNG stream matches the reference
        init = self.geo_feature_std * torch.randn(n_new + 1, self.geo_feature_dim, device=self.device, dtype=self.dtype)
        self.geo_features = torch.cat((self.geo_features[:-1], init), 0)
        if self.color_features is not None:
            init = self.color_feature_std * torch.randn(n_new + 1, self.color_feature_dim, device=self.device,
                                                        dtype=self.dtype)
            self.color_features = torch.cat((self.color_features[:-1], init), 0)
        self.point_certainties = torch.cat(
            (self.point_certainties, torch.zeros(n_new, device=self.device, dtype=self.dtype)), 0)
        self.reset_local_map(sensor_position, sensor_orientation, cur_ts, reboot_map=True)
        return ratio

    def _update_device(self, cand, sensor_position, sensor_orientation, cur_ts):
        """update() on the device: pinb200_map_grow appends into the arenas and rewrites the hash table (4 launches
        instead of ~40 torch ops and seven torch.cat reallocations); ONE host sync remains -- the number of new points,
        which sizes the reference's randn draw for the new feature rows (the RNG stream must advance exactly as in
        model/neural_points.py:395-411, also at feature_std 0)."""
        arena = self.__dict__.get("_arena")
        if arena is None:
            arena = self.__dict__["_arena"] = _MapArena()
        n0, nc = self.count(), cand.shape[0]
        arena.reserve(self, n0 + nc)
        sc = self.__dict__.get("_grow_scratch")
        need = 3 * nc + (nc + 255) // 256 + 8
        if sc is None or sc[0].numel() < need or sc[0].device != cand.device:
            sc = self.__dict__["_grow_scratch"] = (torch.empty(int(need * 1.5), dtype=torch.int32, device=cand.device),
                                                   torch.zeros(1, dtype=torch.int64, device=cand.device))
        grow_all = self.is_empty() or cur_ts == self.reboot_ts
        b = arena.buf
        ops.map_grow(cand, self.buffer_pt_index, self.resolution, b["neural_points"], b["point_orientations"],
                     b["point_ts_create"], b["point_ts_update"], b["point_certainties"], n0,
                     None if grow_all else self.travel_dist, cur_ts, grow_all, self.temporal_local_map_on,
                     self.diff_travel_dist_local, sc[0], sc[1])
        n_new = int(sc[1].item())
        # one extra (padding) row; the randn draw is kept even at std 0 so the RNG stream matches the reference
        init = self.geo_feature_std * torch.randn(n_new + 1, self.geo_feature_dim, device=self.device, dtype=self.dtype)
        b["geo_features"][n0: n0 + n_new + 1].copy_(init)
        if self.color_features is not None:
            init = self.color_feature_std * torch.randn(n_new + 1, self.color_feature_dim, device=self.device,
                                                        dtype=self.dtype)
            b["color_features"][n0: n0 + n_new + 1].copy_(init)
        arena.bind(self, n0 + n_new)
        self.reset_local_map(sensor_position, sensor_orientation, cur_ts, reboot_map=True)
        return n_new / nc

    def reset_local_map(self, sensor_position: torch.Tensor, sensor_orientation: torch.Tensor, cur_ts: int,
                        use_travel_dist: bool = True, diff_ts_local: int = 50, reboot_map: bool = False):
        self.cur_ts = cur_ts
        self.max_ts = max(self.max_ts, cur_ts)
        n = self.count()
        if (self.neural_points.is_cuda and self.neural_points.dtype == torch.float32 and torch.is_tensor(sensor_position)
                and sensor_position.is_cuda and sensor_position.dtype in (torch.float32, torch.float64)):
            return self._reset_local_map_device(sensor_position, sensor_orientation, cur_ts, use_travel_dist,
                                                diff_ts_local, reboot_map)
        if self.temporal_local_map_on:
            if self.config.use_mid_ts:
                ts_used = ((self.point_ts_create + self.point_ts_update) / 2).int()
            else:
                ts_used = self.point_ts_create
            if use_travel_dist:
                recent = torch.abs(self.travel_dist[cur_ts] - self.travel_dist[ts_used.long()]) < self.diff_travel_dist_local
            else:
                recent = torch.abs(cur_ts - ts_used) < diff_ts_local
            if reboot_map:
                recent = recent & (ts_used >= self.reboot_ts)
            # fewer than 100 recent points: keep everything (decided on the device, no host sync)
            recent = recent | (recent.sum() < 100)
        else:
            recent = torch.ones(n, dtype=torch.bool, device=self.device)
        near = ((self.neural_points - sensor_position) ** 2).sum(-1) < self.local_map_radius**2
        keep = recent & near
        # ONE host sync (the local point count); every gather below reuses the index list instead of
        # re-running a boolean-mask compaction per tensor
        idx = torch.nonzero(keep).squeeze(1)
        n_local = idx.shape[0]
        idx_pad = torch.cat((idx, torch.full((1,), n, dtype=idx.dtype, device=self.device)))  # padding row travels along
        self.local_neural_points = self.neural_points.index_select(0, idx)
        self.local_point_orientations = self.point_orientations.index_select(0, idx)
        self.local_point_certainties = self.point_certainties.index_select(0, idx)
        self.local_point_ts_update = self.point_ts_update.index_select(0, idx)
        self.local_mask = torch.cat((keep, torch.ones(1, dtype=torch.bool, device=self.device)))
        self._local_idx = idx_pad
        # Reference quirk kept on purpose (model/neural_points.py:498): `torch.full_like(bool_mask, -1).long()`
        # evaluates to +1, so neural points OUTSIDE the local map translate to local id 1 instead of "invalid";
        # only the trailing padding entry is -1.  STRICT_REFERENCE_G2L=False gives the intended -1.
        miss = 1 if (self.STRICT_REFERENCE_G2L and n_local + 1 > 2) else -1
        g2l = torch.full((n + 1,), miss, dtype=torch.int32, device=self.device)
        g2l[idx] = torch.arange(n_local, dtype=torch.int32, device=self.device)
        g2l[-1] = -1
        self.global2local = g2l
        self.local_geo_features = nn.Parameter(self.geo_features.index_select(0, idx_pad))
        if self.color_features is not None:
            self.local_color_features = nn.Parameter(self.color_features.index_select(0, idx_pad))
        self.local_orientation = sensor_orientation
        self._invalidate()

    def _reset_local_map_device(self, sensor_position, sensor_orientation, cur_ts, use_travel_dist, diff_ts_local,
                                reboot_map):
        """reset_local_map on the device: keep flags + scan (pinb200_local_map_select), ONE host sync for the local point
        count, then index list / global2local / gathers in one launch (pinb200_local_map_gather)."""
        n, dev = self.count(), self.neural_points.device
        sc = self.__dict__.get("_local_scratch")
        need = (n + 1 + 255) // 256 + 1
        if sc is None or sc[0].numel() < need or sc[0].device != dev:
            sc = self.__dict__["_local_scratch"] = (torch.empty(int(need * 1.5) + 64, dtype=torch.int32, device=dev),
                                                    torch.zeros(2, dtype=torch.int64, device=dev))
        mask = torch.empty(n + 1, dtype=torch.bool, device=dev)
        pts, ori = self.neural_points.contiguous(), self.point_orientations.contiguous()
        cert, tsu = self.point_certainties.contiguous(), self.point_ts_update.contiguous()
        temporal = self.temporal_local_map_on
        ops.local_map_select(pts, self.point_ts_create.contiguous() if temporal else None,
                             tsu if (temporal and self.config.use_mid_ts) else None,
                             self.travel_dist if (temporal and use_travel_dist) else None, cur_ts, temporal,
                             self.config.use_mid_ts, use_travel_dist, diff_ts_local, reboot_map, self.reboot_ts,
                             self.diff_travel_dist_local, sensor_position, self.local_map_radius**2, mask, sc[0], sc[1])
        n_local = int(sc[1][1].item())
        idx_pad = torch.empty(n_local + 1, dtype=torch.int64, device=dev)
        g2l = torch.empty(n + 1, dtype=torch.int32, device=dev)
        self.local_neural_points = torch.empty((n_local, 3), dtype=torch.float32, device=dev)
        self.local_point_orientations = torch.empty((n_local, 4), dtype=torch.float32, device=dev)
        self.local_point_certainties = torch.empty((n_local,), dtype=torch.float32, device=dev)
        self.local_point_ts_update = torch.empty((n_local,), dtype=torch.int32, device=dev)
        # reference quirk Q1 (model/neural_points.py:498): points outside the local map translate to local id 1
        miss = 1 if (self.STRICT_REFERENCE_G2L and n_local + 1 > 2) else -1
        ops.local_map_gather(pts, ori, cert, tsu, mask, sc[0], n_local, miss, idx_pad, g2l, self.local_neural_points,
                             self.local_point_orientations, self.local_point_certainties, self.local_point_ts_update)
        self.local_mask = mask
        self._local_idx = idx_pad
        self.global2local = g2l
        self.local_geo_features = nn.Parameter(self.geo_features.index_select(0, idx_pad))
        if self.color_features is not None:
            self.local_color_features = nn.Parameter(self.color_features.index_select(0, idx_pad))
        self.local_orientation = sensor_orientation
        self._invalidate()

    def assign_local_to_global(self):
        idx_pad = getattr(self, "_local_idx", None)
        if idx_pad is None or idx_pad.shape[0] != self.local_geo_features.shape[0]:
            idx_pad = self._local_idx = torch.nonzero(self.local_mask).squeeze(1)
        idx = idx_pad[:-1]
        self.geo_features.index_copy_(0, idx_pad, self.local_geo_features.data)
        if self.color_features is not None:
            self.color_features.index_copy_(0, idx_pad, self.local_color_features.data)
        self.point_certainties.index_copy_(0, idx, self.local_point_certainties)
        self.point_ts_update.index_copy_(0, idx, self.local_point_ts_update)

    # ---------------------------------------------------------------- kernel views
    def map_handle(self, query_locally: bool = True) -> ops.MapHandle:
        """The pinb200_map_view of the current map (cached until the map changes)."""
        key = bool(query_locally)
        h = self._handles.get(key)
        if h is not None:
            return h
        if query_locally and self.global2local is None:
            raise RuntimeError("local map is not set: call update()/reset_local_map() first")
        loc = query_locally
        h = ops.MapHandle(
            slot_table=self.buffer_pt_index,
            buffer_size=self.buffer_size,
            points=self.neural_points,
            ts_create=self.point_ts_create,
            travel_dist=self.travel_dist,
            global2local=self.global2local if loc else None,
            nb_points=self.local_neural_points if loc else self.neural_points,
            nb_orient=self.local_point_orientations if loc else self.point_orientations,
            geo_feat=self.local_geo_features.data if loc else self.geo_features,
            color_feat=(self.local_color_features.data if loc else self.color_features) if self.color_on else None,
            certainty=self.local_point_certainties if loc else self.point_certainties,
            ts_update=self.local_point_ts_update if loc else self.point_ts_update,
            probe_dx=self._probe_dx32,
            resolution=self.resolution,
            max_valid_dist2=self.max_valid_dist2,
            time_filter=self.temporal_local_map_on and loc and self.travel_dist is not None,
            cur_ts=self.cur_ts,
            diff_travel_dist_local=self.diff_travel_dist_local,
            after_pgo=self.after_pgo,
            rec_cache=(self._rec_tables, key),
        )
        self._handles[key] = h
        return h

    def query_sdf(self, query_points: torch.Tensor, sdf_decoder, *, query_ts=None, training_mode=False,
                  query_locally=True, need_grad=True, color_decoder=None, color_grad=False, transform=None,
                  save_knn=False, want_xyz=False, out=None):
        """Fused K1: kNN search + IDW interpolation + decoder (+ analytic gradient) in one launch.
        Equivalent to query_feature -> Decoder.sdf -> (IDW over K) -> get_gradient of the reference
        (utils/tracker.py:297-335), returning dict(sdf, grad, sdf_std, nn_count, certainty, ...)."""
        return ops.query_sdf(self.map_handle(query_locally), sdf_decoder.handle(), query_points,
                             nn_k=self.config.query_nn_k, weighted_first=self.config.weighted_first,
                             training_mode=training_mode, need_grad=need_grad, query_ts=query_ts,
                             color_dec=None if color_decoder is None else color_decoder.handle(sigmoid_out=True),
                             color_grad=color_grad, transform=transform, save_knn=save_knn, want_xyz=want_xyz,
                             out=out)

    def query_sdf_host(self, query_host: torch.Tensor, sdf_decoder, host_out: dict, *, chunks: int = 4,
                       query_locally: bool = True, need_grad: bool = True):
        """Host-facing fused query: `query_host` [N,3] fp32 in (pinned) host memory in, results written into the
        (pinned) host tensors of `host_out` (any of sdf [N], grad [N,3], sdf_std [N], nn_count [N] i32,
        certainty [N]).  The batch is cut into `chunks` pieces that alternate between two CUDA streams, so the
        host->device copy of piece i+1 and the device->host copies of piece i-1 overlap the kernel of piece i.
        Stream-ordered with respect to the caller's current stream (results are complete when that stream is)."""
        n = query_host.shape[0]
        pipe = self.__dict__.get("_host_pipe")
        if pipe is None:
            pipe = self.__dict__["_host_pipe"] = {"streams": [torch.cuda.Stream(self.device) for _ in range(2)],
                                                  "work": [{}, {}], "q": [None, None]}
        cur = torch.cuda.current_stream()
        # build (and cache) the kernel views on the caller's stream BEFORE forking: the probe-record table of a fresh
        # handle is written by a kernel, and the side streams only wait on `start`
        self.map_handle(query_locally).ensure_records()
        sdf_decoder.handle()
        start = torch.cuda.Event()
        start.record(cur)
        step = max(32, -(-n // max(1, chunks)))
        for i, head in enumerate(range(0, n, step)):
            tail = min(head + step, n)
            s = pipe["streams"][i % 2]
            if i < 2:
                s.wait_event(start)
            with torch.cuda.stream(s):
                qd = pipe["q"][i % 2]
                if qd is None or qd.shape[0] < tail - head:
                    qd = pipe["q"][i % 2] = torch.empty((step, 3), dtype=torch.float32, device=self.device)
                qv = qd[: tail - head]
                qv.copy_(query_host[head:tail], non_blocking=True)
                o = self.query_sdf(qv, sdf_decoder, query_locally=query_locally, need_grad=need_grad,
                                   out=pipe["work"][i % 2])
                for name, h in host_out.items():
                    h[head:tail].copy_(o[name], non_blocking=True)
        for s in pipe["streams"]:
            done = torch.cuda.Event()
            done.record(s)
            cur.wait_event(done)
        return host_out

    # ---------------------------------------------------------------- reference-compatible queries
    def radius_neighborhood_search(self, points: torch.Tensor, time_filtering: bool = False):
        """dist2 [N,C], global ids [N,C] (int64 like the reference)."""
        h = self.map_handle(False)
        if time_filtering:
            h = ops.MapHandle(**{**h.keep, "buffer_size": self.buffer_size, "resolution": self.resolution,
                                 "max_valid_dist2": self.max_valid_dist2, "time_filter": True, "cur_ts": self.cur_ts,
                                 "diff_travel_dist_local": self.diff_travel_dist_local, "after_pgo": self.after_pgo})
        d2, idx = ops.radius_search(h, points.detach().contiguous())
        return d2, idx.long()

    def query_certainty(self, query_points: torch.Tensor):
        return ops.query_certainty(self.map_handle(False), query_points.detach().contiguous())

    FUSED_QUERY_FEATURE = True  # inference-mode weighted_first queries return lazy handles (model/fused_features.py)

    def query_feature(self, query_points: torch.Tensor, query_ts: torch.Tensor = None, training_mode: bool = True,
                      query_locally: bool = True, query_geo_feature: bool = True, query_color_feature: bool = False):
        """Reference-compatible query (model/neural_points.py:530-746).  Inference-mode `weighted_first` queries on
        the GPU return `FusedFeatures` handles in place of the feature tensors: `Decoder.sdf` /
        `Decoder.regress_color` then run the fused K1 kernel and `torch.autograd.grad` receives the kernel's
        analytic gradient, so the reference's unchanged tracker / mesher code gets one fused launch per decoder.
        Everything else takes the eager path below."""
        if not query_geo_feature and not query_color_feature:
            sys.exit("you need to at least query one kind of feature")
        if (self.FUSED_QUERY_FEATURE and self.config.weighted_first and not training_mode and query_points.is_cuda
                and query_geo_feature):
            from .fused_features import FusedFeatures, _Group

            k = self.config.query_nn_k
            idx32, _, w, cnt, _ = ops.knn_search(self.map_handle(query_locally), query_points.detach().contiguous(), k,
                                                 want_gidx=True)
            cert_tab = self.local_point_certainties if query_locally else self.point_certainties
            valid = idx32 >= 0
            certainty = (cert_tab[idx32.long().clamp(min=0)] * valid * w).sum(dim=1)
            grp = _Group(self, query_points, query_locally)
            geo = FusedFeatures(grp, "geo")
            col = FusedFeatures(grp, "color") if (query_color_feature and self.color_features is not None) else None
            return geo, col, w.unsqueeze(-1), cnt.long(), certainty
        return self._query_feature_eager(query_points, query_ts, training_mode, query_locally, query_geo_feature,
                                         query_color_feature)

    def _query_feature_eager(self, query_points: torch.Tensor, query_ts: torch.Tensor = None, training_mode: bool = True,
                             query_locally: bool = True, query_geo_feature: bool = True,
                             query_color_feature: bool = False):
        """The kNN search (the reference's "slow part") runs in the CUDA kernel; the returned feature vectors are
        assembled from the neighbour ids with differentiable torch ops, so callers may keep using autograd (first
        and second order) exactly as before."""
        k = self.config.query_nn_k
        h = self.map_handle(query_locally)
        idx32, _, _, cnt, gidx32 = ops.knn_search(h, query_points.detach().contiguous(), k, want_gidx=True)
        idx = idx32.long()
        valid = idx >= 0
        safe = idx.clamp(min=0)
        nn_counts = cnt.long()
        pts = self.local_neural_points if query_locally else self.neural_points
        ori = self.local_point_orientations if query_locally else self.point_orientations
        cert_tab = self.local_point_certainties if query_locally else self.point_certainties
        nb = pts[safe]
        # squared distance to the point the hash returned (global array), differentiable w.r.t. the query
        d2 = ((self.neural_points[gidx32.long().clamp(min=0)] - query_points.view(-1, 1, 3)) ** 2).sum(-1)
        d2 = torch.where(valid, d2, torch.full_like(d2, 9e3))
        vm = valid.unsqueeze(-1)
        nvec = query_points.view(-1, 1, 3) - nb
        if self.after_pgo:
            nvec = _quat_rotate_passive(ori[safe], nvec)
        nvec = nvec * vm
        geo_vec = col_vec = None
        if query_geo_feature:
            tab = self.local_geo_features if query_locally else self.geo_features
            geo_vec = torch.cat((tab[safe] * vm, nvec), dim=2)
        if query_color_feature and self.color_features is not None:
            tab = self.local_color_features if query_locally else self.color_features
            col_vec = torch.cat((tab[safe] * vm, nvec), dim=2)
        eps = 1e-15
        w = (1.0 / (d2 + eps)) * valid
        w = torch.where((nn_counts == 0).unsqueeze(1), torch.full_like(w, eps), w)
        w = (w / w.sum(dim=1, keepdim=True)) * valid
        with torch.no_grad():
            certainty = cert_tab[safe] * valid
            if training_mode:
                flat = (safe * valid).flatten()
                cert_tab.scatter_add_(0, flat, w.detach().flatten())
                if query_locally and query_ts is not None:
                    stamps = (query_ts.view(-1, 1).repeat(1, k) * valid).flatten()
                    self.local_point_ts_update.scatter_reduce_(0, flat, stamps, reduce="amax", include_self=True)
            queried_certainty = (certainty * w).sum(dim=1)
        w = w.unsqueeze(-1)
        if self.config.weighted_first:
            if geo_vec is not None:
                geo_vec = (geo_vec * w).sum(dim=1)
            if col_vec is not None:
                col_vec = (col_vec * w).sum(dim=1)
        return geo_vec, col_vec, w, nn_counts, queried_certainty

    # ---------------------------------------------------------------- map surgery
    def prune_map(self, prune_certainty_thre, min_prune_count=500, global_prune=False):
        weak = self.point_certainties < prune_certainty_thre
        if not global_prune:
            stale = torch.abs(self.travel_dist[self.cur_ts] - self.travel_dist[self.point_ts_update.long()])
            weak = weak & (stale > self.diff_travel_dist_local)
        n_drop = int(weak.sum().item())
        if n_drop <= min_prune_count:
            return False
        if not self.silence:
            print("# Prune neural points: ", n_drop)
        keep = ~weak
        self.neural_points = self.neural_points[keep]
        self.point_orientations = self.point_orientations[keep]
        self.point_ts_create = self.point_ts_create[keep]
        self.point_ts_update = self.point_ts_update[keep]
        self.point_certainties = self.point_certainties[keep]
        keep_pad = torch.cat((keep, torch.ones(1, dtype=torch.bool, device=self.device)))
        self.geo_features = self.geo_features[keep_pad]
        if self.color_features is not None:
            self.color_features = self.color_features[keep_pad]
        self._invalidate(slots_freed=True)
        return True

    def adjust_map(self, pose_diff_torch):
        """Move every neural point by the pose correction of its frame (after PGO)."""
        self.after_pgo = True
        if self.config.use_mid_ts:
            ts = ((self.point_ts_create + self.point_ts_update) / 2).int().long()
        else:
            ts = self.point_ts_create.long()
        if self.neural_points.is_cuda and self.neural_points.dtype == torch.float32:
            # one streaming kernel over the points (pinb200_frame_transform); the per-frame quaternions are tiny
            pts, ori = self.neural_points.clone(), self.point_orientations.contiguous().clone()
            ops.frame_transform(pts, self.point_ts_create.contiguous(), pose_diff_torch, quat=ori,
                                dquat=_rotmat_to_quat(pose_diff_torch[:, :3, :3]),
                                ts_b=self.point_ts_update.contiguous() if self.config.use_mid_ts else None)
            self.neural_points, self.point_orientations = pts, ori
        else:
            tf = pose_diff_torch[ts].to(self.neural_points)
            self.neural_points = (tf[:, :3, :3] @ self.neural_points.unsqueeze(-1)).squeeze(-1) + tf[:, :3, 3]
            dq = _rotmat_to_quat(pose_diff_torch[:, :3, :3])[ts].to(self.point_orientations)
            self.point_orientations = _quat_multiply(dq, self.point_orientations)
        self._invalidate()

    def recreate_hash(self, sensor_position: torch.Tensor, sensor_orientation: torch.Tensor, kept_points: bool = True,
                      with_ts: bool = True, cur_ts=0):
        res = self.resolution
        self.buffer_pt_index = torch.full((self.buffer_size,), -1, dtype=torch.int32, device=self.device)
        if with_ts:
            if self.config.use_mid_ts:
                ts_used = ((self.point_ts_create + self.point_ts_update) / 2).int()
            else:
                ts_used = self.point_ts_create
            score = torch.abs(ts_used - cur_ts).float()
        else:
            score = self.point_certainties.max() - self.point_certainties
        pick = voxel_down_sample_min_value(self.neural_points, res, score)
        if kept_points:
            _put_last(self.buffer_pt_index, self._slots(self.neural_points[pick]), pick.to(torch.int32))
        else:
            if not self.silence:
                print("Filter duplicated neural points")
            self.neural_points = self.neural_points[pick]
            self.point_orientations = self.point_orientations[pick]
            self.point_ts_create = self.point_ts_create[pick]
            self.point_ts_update = self.point_ts_update[pick]
            self.point_certainties = self.point_certainties[pick]
            pick_pad = torch.cat((pick, torch.tensor([-1], device=self.device, dtype=pick.dtype)))
            self.geo_features = self.geo_features[pick_pad]
            if self.color_features is not None:
                self.color_features = self.color_features[pick_pad]
            n = self.neural_points.shape[0]
            _put_last(self.buffer_pt_index, self._slots(self.neural_points),
                      torch.arange(n, dtype=torch.int32, device=self.device))
        self._invalidate(slots_freed=True)
        if sensor_position is not None:
            self.reset_local_map(sensor_position, sensor_orientation, cur_ts)
        if not kept_points:
            self.record_memory(verbose=(not self.silence))

    def clear_temp(self, clean_more: bool = False):
        """Drop everything that is rebuilt after unpickling (utils/tools.py:295-317 pickles the module)."""
        self.buffer_pt_index = None
        self.local_neural_points = None
        self.local_point_orientations = None
        self.local_geo_features = nn.Parameter()
        self.local_color_features = nn.Parameter()
        self.local_point_certainties = None
        self.local_point_ts_update = None
        self.local_mask = None
        self._local_idx = None
        self.global2local = None
        self._handles = {}
        self._rec_tables = {}
        if clean_more:
            self.point_ts_create = None
            self.point_ts_update = None
            self.point_certainties = None

    def __setstate__(self, state):
        """Also accepts the state of a map pickled by the UPSTREAM class (utils/tools.py:300-309 pickles the whole
        module after clear_temp()): its plain `travel_dist` attribute becomes `_travel_dist` (a property here), the
        int64 index tensors become int32, and the fields this class adds get their defaults."""
        super().__setstate__(state)
        d = self.__dict__
        if "travel_dist" in d:
            d["_travel_dist"] = d.pop("travel_dist")
        d.setdefault("_travel_dist", None)
        d["_handles"] = {}
        d["_rec_tables"] = {}
        d.setdefault("_local_idx", None)
        d.setdefault("idx_dtype", torch.int32)
        d.setdefault("color_on", d.get("color_features") is not None)
        for name in ("buffer_pt_index", "global2local"):
            t = d.get(name)
            if torch.is_tensor(t) and t.dtype != torch.int32:
                d[name] = t.to(torch.int32)
        if "_probe_dx32" not in d and torch.is_tensor(d.get("neighbor_dx")):
            d["_probe_dx32"] = d["neighbor_dx"].to(torch.int32).contiguous()

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_handles"] = {}  # raw device pointers never travel
        state["_rec_tables"] = {}  # derived data (800 MB per index space at the default buffer_size)
        state.pop("_host_pipe", None)  # CUDA streams / staging buffers of query_sdf_host
        state.pop("_arena", None)
        state.pop("_grow_scratch", None)
        state.pop("_local_scratch", None)
        for k, v in list(state.items()):  # views of the growth arenas: pickle the rows, not the capacity
            if torch.is_tensor(v) and v.untyped_storage().nbytes() > 2 * v.numel() * v.element_size() + 4096:
                state[k] = v.clone()
        return state


def _rotmat_to_quat(r: torch.Tensor) -> torch.Tensor:
    """[N,3,3] -> [N,4] wxyz, branch on the largest diagonal term."""
    m00, m11, m22 = r[:, 0, 0], r[:, 1, 1], r[:, 2, 2]
    q = torch.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22], 1)
    q = torch.sqrt(torch.clamp(q, min=0)) * 0.5
    best = torch.argmax(q, dim=1)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    r21, r02, r10 = r[:, 2, 1] - r[:, 1, 2], r[:, 0, 2] - r[:, 2, 0], r[:, 1, 0] - r[:, 0, 1]
    s01, s02, s12 = r[:, 0, 1] + r[:, 1, 0], r[:, 0, 2] + r[:, 2, 0], r[:, 1, 2] + r[:, 2, 1]
    cand = torch.stack([
        torch.stack([w, r21 / (4 * w), r02 / (4 * w), r10 / (4 * w)], 1),
        torch.stack([r21 / (4 * x), x, s01 / (4 * x), s02 / (4 * x)], 1),
        torch.stack([r02 / (4 * y), s01 / (4 * y), y, s12 / (4 * y)], 1),
        torch.stack([r10 / (4 * z), s02 / (4 * z), s12 / (4 * z), z], 1),
    ], 1)
    return cand[torch.arange(r.shape[0], device=r.device), best]


def _quat_multiply(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)
