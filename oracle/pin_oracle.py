"""CPU oracle for the PIN-SLAM hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

This file restates, op by op in plain PyTorch (CPU by default), the algorithm
of the reference's per-frame data-parallel hot path so that the sm_90a CUDA
kernels in ``pin_slam_b200/csrc`` can be checked against it.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it.  The product path (``pin_slam_b200``) never
imports this module.

Pinning: the reference ships no tests or golden vectors (SURVEY.md §4), so the
oracle is pinned against *outputs of the reference itself* run in the build
container: ``tests/golden/make_golden.py`` imports ``/root/reference`` (with its
optional GUI/IO dependencies stubbed), drives the reference ``NeuralPoints`` /
``Decoder`` / ``Tracker`` / ``Mapper`` code on seeded inputs and stores the
inputs+outputs as ``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks
every function below against those fixtures.

Every function cites the reference file:line (relative to /root/reference) it
follows.  The arithmetic deliberately uses the same ATen ops in the same order
as the reference so that on CPU the results are bit-identical for the integer
parts (cell index, hash slot, neighbour ids, counts) and equal to rounding for
the floating-point parts.
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import torch

PRIMES = (73856093, 19349669, 83492791)  # model/neural_points.py:82-84


# --------------------------------------------------------------------------
# map state
# --------------------------------------------------------------------------
@dataclass
class OracleMap:
    """Tensor state of a neural point map (model/neural_points.py:82-136)."""

    resolution: float
    buffer_size: int
    feature_dim: int
    # global arrays
    neural_points: torch.Tensor  # [Mg,3] f32
    point_orientations: torch.Tensor  # [Mg,4] f32 wxyz
    geo_features: torch.Tensor  # [Mg+1,F] f32 (last row = padding)
    color_features: Optional[torch.Tensor]  # [Mg+1,F] or None
    point_ts_create: torch.Tensor  # [Mg] i32
    point_ts_update: torch.Tensor  # [Mg] i32
    point_certainties: torch.Tensor  # [Mg] f32
    buffer_pt_index: torch.Tensor  # [B] i64, -1 = empty
    # local arrays (reset_local_map, :424-513)
    local_neural_points: Optional[torch.Tensor] = None
    local_point_orientations: Optional[torch.Tensor] = None
    local_geo_features: Optional[torch.Tensor] = None
    local_color_features: Optional[torch.Tensor] = None
    local_point_certainties: Optional[torch.Tensor] = None
    local_point_ts_update: Optional[torch.Tensor] = None
    local_mask: Optional[torch.Tensor] = None
    global2local: Optional[torch.Tensor] = None
    # search neighbourhood (set_search_neighborhood, :910-947)
    neighbor_dx: Optional[torch.Tensor] = None  # [C,3] i64
    max_valid_dist2: float = 0.0
    # temporal window
    travel_dist: Optional[torch.Tensor] = None  # [n_frames] f32
    cur_ts: int = 0
    diff_travel_dist_local: float = 0.0
    temporal_local_map_on: bool = True
    after_pgo: bool = False

    @property
    def device(self):
        return self.neural_points.device

    def primes(self):
        return torch.tensor(PRIMES, dtype=torch.int64, device=self.device)

    def to(self, device):
        for k, v in list(self.__dict__.items()):
            if torch.is_tensor(v):
                setattr(self, k, v.to(device))
        return self

    def clone(self):
        kw = {}
        for k, v in self.__dict__.items():
            kw[k] = v.clone() if torch.is_tensor(v) else v
        return OracleMap(**kw)

    def double(self):
        """fp64 copy: the reference honours config.dtype everywhere on the path, so the same algorithm in
        fp64 is the ground truth that separates a kernel's error from the fp32 reference's own rounding
        (SURVEY.md section 8c)."""
        kw = {}
        for k, v in self.__dict__.items():
            kw[k] = v.double() if (torch.is_tensor(v) and v.dtype == torch.float32) else (
                v.clone() if torch.is_tensor(v) else v)
        return OracleMap(**kw)


def probe_offsets(num_nei_cells: int, search_alpha: float, device="cpu") -> torch.Tensor:
    """Integer cell offsets inside the sphere |dx|^2 < (n+alpha)^2.

    model/neural_points.py:919-932 (meshgrid 'ij' order, i.e. x slowest).
    """
    r = torch.arange(-num_nei_cells, num_nei_cells + 1, dtype=torch.int64, device=device)
    gx, gy, gz = torch.meshgrid(r, r, r, indexing="ij")
    dx = torch.stack((gx, gy, gz), dim=-1).reshape(-1, 3)
    keep = (dx**2).sum(-1) < (num_nei_cells + search_alpha) ** 2
    return dx[keep]


def set_search_neighborhood(m: OracleMap, num_nei_cells: int, search_alpha: float) -> None:
    """model/neural_points.py:910-947."""
    m.neighbor_dx = probe_offsets(num_nei_cells, search_alpha, m.device)
    m.max_valid_dist2 = 3 * ((num_nei_cells + 1) * m.resolution) ** 2


def cell_of(points: torch.Tensor, resolution: float) -> torch.Tensor:
    """fp32 division, floor, int64 (model/neural_points.py:963, :334)."""
    return (points / resolution).floor().to(torch.int64)


def hash_cells(cells: torch.Tensor, buffer_size: int) -> torch.Tensor:
    """C-style fmod of the prime dot product (model/neural_points.py:972-974).

    The result may be negative; the reference uses it directly as an index so
    torch wraps it (h<0 -> h+B).  ``wrap_slot`` makes that explicit.
    """
    primes = torch.tensor(PRIMES, dtype=torch.int64, device=cells.device)
    return torch.fmod((cells * primes).sum(-1), int(buffer_size))


def wrap_slot(h: torch.Tensor, buffer_size: int) -> torch.Tensor:
    return torch.where(h < 0, h + int(buffer_size), h)


# --------------------------------------------------------------------------
# simple map builder used by tests (a fresh map == NeuralPoints.update on an
# empty map, model/neural_points.py:331-420, minus the RNG feature init which
# the caller provides explicitly)
# --------------------------------------------------------------------------
def build_map(
    sample_points: torch.Tensor,
    resolution: float,
    buffer_size: int,
    geo_features: torch.Tensor,
    color_features: Optional[torch.Tensor] = None,
    ts_create: Optional[torch.Tensor] = None,
    certainties: Optional[torch.Tensor] = None,
    orientations: Optional[torch.Tensor] = None,
    num_nei_cells: int = 2,
    search_alpha: float = 0.2,
) -> OracleMap:
    """Insert one point per row into the slot table, last writer wins on a hash
    collision (index_put semantics of ``buffer_pt_index[hash] = cur_pt_idx``,
    model/neural_points.py:377; duplicate-slot write order is the serial CPU
    order here)."""
    dev = sample_points.device
    mg = sample_points.shape[0]
    f = geo_features.shape[1]
    assert geo_features.shape[0] == mg + 1
    table = torch.full((int(buffer_size),), -1, dtype=torch.int64, device=dev)
    slots = wrap_slot(hash_cells(cell_of(sample_points, resolution), buffer_size), buffer_size)
    # serial last-writer-wins (numpy fancy assignment applies duplicates in order => deterministic)
    tnp = table.cpu().numpy()
    tnp[slots.cpu().numpy()] = __import__("numpy").arange(mg, dtype="int64")
    table = torch.from_numpy(tnp).to(dev)
    m = OracleMap(
        resolution=float(resolution),
        buffer_size=int(buffer_size),
        feature_dim=f,
        neural_points=sample_points.clone(),
        point_orientations=(
            orientations.clone()
            if orientations is not None
            else torch.tensor([[1.0, 0, 0, 0]], device=dev).repeat(mg, 1)
        ),
        geo_features=geo_features.clone(),
        color_features=None if color_features is None else color_features.clone(),
        point_ts_create=(
            ts_create.clone().to(torch.int32)
            if ts_create is not None
            else torch.zeros(mg, dtype=torch.int32, device=dev)
        ),
        point_ts_update=(
            ts_create.clone().to(torch.int32)
            if ts_create is not None
            else torch.zeros(mg, dtype=torch.int32, device=dev)
        ),
        point_certainties=(
            certainties.clone() if certainties is not None else torch.zeros(mg, device=dev)
        ),
        buffer_pt_index=table,
    )
    set_search_neighborhood(m, num_nei_cells, search_alpha)
    return m


def reset_local_map(
    m: OracleMap,
    sensor_position: torch.Tensor,
    local_map_radius: float,
    cur_ts: int,
    reboot_ts: int = 0,
    reboot_map: bool = False,
) -> None:
    """model/neural_points.py:424-513 (use_travel_dist=True, use_mid_ts=False)."""
    m.cur_ts = cur_ts
    mg = m.neural_points.shape[0]
    dev = m.device
    if m.temporal_local_map_on:
        ts_used = m.point_ts_create
        delta = torch.abs(m.travel_dist[cur_ts] - m.travel_dist[ts_used.long()])
        time_mask = delta < m.diff_travel_dist_local
        if reboot_map:
            time_mask = time_mask & (ts_used >= reboot_ts)
        if torch.sum(time_mask) < 100:
            time_mask = torch.ones(mg, dtype=torch.bool, device=dev)
    else:
        time_mask = torch.ones(mg, dtype=torch.bool, device=dev)
    vec = m.neural_points[time_mask] - sensor_position
    d2 = torch.sum(vec**2, dim=-1)
    dist_mask = d2 < local_map_radius**2
    tm_idx = torch.nonzero(time_mask).squeeze(-1)
    loc_idx = tm_idx[dist_mask]
    local_mask = torch.zeros(mg, dtype=torch.bool, device=dev)
    local_mask[loc_idx] = True
    m.local_neural_points = m.neural_points[local_mask]
    m.local_point_orientations = m.point_orientations[local_mask]
    m.local_point_certainties = m.point_certainties[local_mask]
    m.local_point_ts_update = m.point_ts_update[local_mask]
    local_mask = torch.cat((local_mask, torch.tensor([True], device=dev)))
    m.local_mask = local_mask
    g2l = torch.full_like(local_mask, -1).long()
    li = torch.nonzero(local_mask).flatten()
    g2l[li] = torch.arange(li.numel(), device=dev)
    g2l[-1] = -1
    m.global2local = g2l
    m.local_geo_features = m.geo_features[local_mask].clone()
    if m.color_features is not None:
        m.local_color_features = m.color_features[local_mask].clone()


# --------------------------------------------------------------------------
# a3: radius search  (model/neural_points.py:950-1009)
# --------------------------------------------------------------------------
def radius_search(m: OracleMap, points: torch.Tensor, time_filtering: bool = False):
    cells = cell_of(points, m.resolution)  # [N,3]
    probe = cells[..., None, :] + m.neighbor_dx  # [N,C,3]
    h = hash_cells(probe, m.buffer_size)  # [N,C] may be negative -> wraps
    nidx = m.buffer_pt_index[h]
    if time_filtering:
        dtd = torch.abs(
            m.travel_dist[m.cur_ts] - m.travel_dist[m.point_ts_create[nidx].long()]
        )
        nidx[~(dtd < m.diff_travel_dist_local)] = -1
    npts = m.neural_points[nidx]
    sub = npts - points.view(-1, 1, 3)
    dist2 = torch.sum(sub**2, dim=-1)
    dist2[nidx == -1] = m.max_valid_dist2
    nidx[dist2 > m.max_valid_dist2] = -1
    return dist2, nidx


def quat_rotate_passive(quat: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """utils/tools.py:428-437 (conjugate quaternion, p' = q^-1 p q)."""
    w = quat[..., 0].unsqueeze(-1)
    xyz = -quat[..., 1:]
    t = 2 * torch.linalg.cross(xyz, v)
    return v + w * t + torch.linalg.cross(xyz, t)


# --------------------------------------------------------------------------
# a4: query_feature  (model/neural_points.py:530-746)
# --------------------------------------------------------------------------
def query_feature(
    m: OracleMap,
    query_points: torch.Tensor,
    query_ts: Optional[torch.Tensor] = None,
    nn_k: int = 6,
    weighted_first: bool = True,
    training_mode: bool = True,
    query_locally: bool = True,
    query_geo_feature: bool = True,
    query_color_feature: bool = False,
    return_idx: bool = False,
):
    n = query_points.shape[0]
    dev = query_points.device
    dists2, idx = radius_search(
        m, query_points, time_filtering=m.temporal_local_map_on and query_locally
    )
    if query_locally:
        idx = m.global2local[idx]
    nn_counts = (idx >= 0).sum(dim=-1)
    dists2[idx == -1] = 9e3
    sd, order = torch.sort(dists2, dim=1)
    sidx = idx.gather(1, order)
    dists2 = sd[:, :nn_k]
    idx = sidx[:, :nn_k]
    valid = idx >= 0
    knn_idx_out = idx.clone()

    geo_tab = m.local_geo_features if query_locally else m.geo_features
    col_tab = m.local_color_features if query_locally else m.color_features
    pts_tab = m.local_neural_points if query_locally else m.neural_points
    ori_tab = m.local_point_orientations if query_locally else m.point_orientations
    cert_tab = m.local_point_certainties if query_locally else m.point_certainties

    geo_vec = col_vec = None
    if query_geo_feature:
        geo = torch.zeros(n, nn_k, m.feature_dim, device=dev, dtype=query_points.dtype)
        geo[valid] = geo_tab[idx[valid]]
    if query_color_feature and col_tab is not None:
        col = torch.zeros(n, nn_k, m.feature_dim, device=dev, dtype=query_points.dtype)
        col[valid] = col_tab[idx[valid]]

    certainty = cert_tab[idx]
    nvec = query_points.view(-1, 1, 3) - pts_tab[idx]
    quat = ori_tab[idx]
    if m.after_pgo:
        nvec = quat_rotate_passive(quat, nvec)
    nvec[~valid] = torch.zeros(1, 3, device=dev, dtype=query_points.dtype)

    if query_geo_feature:
        geo_vec = torch.cat((geo, nvec), dim=2)
    if query_color_feature and col_tab is not None:
        col_vec = torch.cat((col, nvec), dim=2)

    eps = 1e-15
    w = 1.0 / (dists2 + eps)
    w[~valid] = 0.0
    w[nn_counts == 0] = eps
    w = torch.div(w, torch.sum(w, dim=1).unsqueeze(1))
    w[~valid] = 0.0

    with torch.no_grad():
        if training_mode:
            idx[~valid] = 0
            cert_tab.scatter_add_(dim=0, index=idx.flatten(), src=w.flatten())
            if query_locally and query_ts is not None:
                its = query_ts.view(-1, 1).repeat(1, nn_k)
                its[~valid] = 0
                m.local_point_ts_update.scatter_reduce_(
                    dim=0, index=idx.flatten(), src=its.flatten(), reduce="amax", include_self=True
                )
        certainty[~valid] = 0.0
        queried_certainty = torch.sum(certainty * w, dim=1)

    w = w.unsqueeze(-1)
    if weighted_first:
        if geo_vec is not None:
            geo_vec = torch.sum(geo_vec * w, dim=1)
        if col_vec is not None:
            col_vec = torch.sum(col_vec * w, dim=1)
    out = (geo_vec, col_vec, w, nn_counts, queried_certainty)
    if return_idx:
        return out + (knn_idx_out, dists2)
    return out


def query_certainty(m: OracleMap, query_points: torch.Tensor) -> torch.Tensor:
    """model/neural_points.py:1011-1032 (global arrays, no age filter)."""
    _, idx = radius_search(m, query_points)
    c = m.point_certainties[idx]
    c[idx < 0] = 0.0
    return torch.max(c, dim=-1)[0]


# --------------------------------------------------------------------------
# a6: decoder  (model/decoder.py:14-113)
# --------------------------------------------------------------------------
@dataclass
class DecoderParams:
    """weights[i] = (W [H,in], b [H]) per hidden layer; out = (W [out,H], b [out])."""

    hidden: List[Tuple[torch.Tensor, torch.Tensor]]
    out: Tuple[torch.Tensor, torch.Tensor]
    sdf_scale: float = 1.0
    leaky: bool = False

    def tensors(self):
        ts = []
        for w, b in self.hidden:
            ts += [w, b]
        ts += [self.out[0], self.out[1]]
        return ts

    def requires_grad_(self, flag=True):
        for t in self.tensors():
            t.requires_grad_(flag)
        return self

    def clone(self):
        return DecoderParams(
            [(w.detach().clone(), b.detach().clone()) for w, b in self.hidden],
            (self.out[0].detach().clone(), self.out[1].detach().clone()),
            self.sdf_scale,
            self.leaky,
        )

    def double(self):
        return DecoderParams([(w.detach().double(), b.detach().double()) for w, b in self.hidden],
                             (self.out[0].detach().double(), self.out[1].detach().double()), self.sdf_scale,
                             self.leaky)

    def to(self, device):
        return DecoderParams(
            [(w.to(device), b.to(device)) for w, b in self.hidden],
            (self.out[0].to(device), self.out[1].to(device)),
            self.sdf_scale,
            self.leaky,
        )


def make_decoder(in_dim, hidden_dim, hidden_level, out_dim, sdf_scale, seed=0, device="cpu", bias=True):
    """nn.Linear default init (kaiming_uniform a=sqrt(5) -> U(-1/sqrt(in), 1/sqrt(in))).  `bias=False`
    (mlp_bias_on False, model/decoder.py:43-51): the biases are zero, which is the same forward pass as none."""
    g = torch.Generator().manual_seed(seed)
    hs = []
    d = in_dim
    for _ in range(hidden_level):
        bound = 1.0 / math.sqrt(d)
        w = (torch.rand(hidden_dim, d, generator=g) * 2 - 1) * bound
        b = (torch.rand(hidden_dim, generator=g) * 2 - 1) * bound
        hs.append((w.to(device), (b if bias else torch.zeros_like(b)).to(device)))
        d = hidden_dim
    bound = 1.0 / math.sqrt(d)
    wo = (torch.rand(out_dim, d, generator=g) * 2 - 1) * bound
    bo = (torch.rand(out_dim, generator=g) * 2 - 1) * bound
    return DecoderParams(hs, (wo.to(device), (bo if bias else torch.zeros_like(bo)).to(device)), sdf_scale)


def decoder_mlp(p: DecoderParams, x: torch.Tensor) -> torch.Tensor:
    """model/decoder.py:61-79."""
    h = x
    for w, b in p.hidden:
        h = torch.nn.functional.linear(h, w, b)
        h = torch.nn.functional.leaky_relu(h) if p.leaky else torch.relu(h)
    return torch.nn.functional.linear(h, p.out[0], p.out[1])


def decoder_sdf(p: DecoderParams, x: torch.Tensor) -> torch.Tensor:
    """model/decoder.py:83-85."""
    return decoder_mlp(p, x).squeeze(1) * p.sdf_scale


def decoder_color(p: DecoderParams, x: torch.Tensor) -> torch.Tensor:
    """model/decoder.py:112-114."""
    return torch.sigmoid(decoder_mlp(p, x))


def get_gradient(inputs, outputs):
    """utils/tools.py:247-260."""
    return torch.autograd.grad(
        outputs=outputs,
        inputs=inputs,
        grad_outputs=torch.ones_like(outputs),
        create_graph=True,
        retain_graph=True,
        only_inputs=True,
    )[0]


# --------------------------------------------------------------------------
# a8: Tracker.query_source_points  (utils/tracker.py:227-365), single batch
# --------------------------------------------------------------------------
def query_sdf(
    m: OracleMap,
    dec: DecoderParams,
    coord: torch.Tensor,
    nn_k: int,
    weighted_first: bool,
    query_locally: bool = True,
    need_grad: bool = True,
    training_mode: bool = False,
    query_ts: Optional[torch.Tensor] = None,
    color_dec: Optional[DecoderParams] = None,
    color_grad: bool = False,
):
    """Returns dict(sdf, grad, sdf_std, nn_count, certainty[, color, color_grad])."""
    coord = coord.detach().clone()
    if need_grad or color_grad:
        coord.requires_grad_(True)
    geo, col, w, nn_count, cert = query_feature(
        m,
        coord,
        query_ts,
        nn_k,
        weighted_first,
        training_mode=training_mode,
        query_locally=query_locally,
        query_color_feature=color_dec is not None,
    )
    sdf = decoder_sdf(dec, geo)
    sdf_std = torch.zeros(coord.shape[0], device=coord.device, dtype=coord.dtype)
    if not weighted_first:
        # [N,K,1]; decoder_sdf's squeeze(1) drops the K axis when K = 1, and the reference's [N,1] * [N,1,1] would
        # broadcast to [N,N,1] -- the K > 1 semantics apply
        sdf = sdf.reshape(w.shape)
        mean = torch.sum(sdf * w, dim=1)  # [N,1]
        var = torch.sum(w * (sdf - mean.unsqueeze(-1)) ** 2, dim=1)
        sdf_std = torch.sqrt(var).squeeze(1).detach()
        sdf = mean.squeeze(1)
    out = {
        "sdf": sdf.detach(),
        "sdf_std": sdf_std,
        "nn_count": nn_count,
        "certainty": cert.detach(),
        "weight": w.detach(),
    }
    if need_grad:
        out["grad"] = get_gradient(coord, sdf).detach()
    if color_dec is not None:
        c = decoder_color(color_dec, col)
        if not weighted_first:
            c = torch.sum(c * w, dim=1)
        out["color"] = c.detach()
        if color_grad:
            cg = torch.zeros(coord.shape[0], c.shape[1], 3, device=coord.device, dtype=coord.dtype)
            for i in range(c.shape[1]):
                cg[:, i, :] = get_gradient(coord, c[:, i]).detach()
            out["color_grad"] = cg
    return out


# --------------------------------------------------------------------------
# f3: Mesher.query_points  (utils/mesher.py:40-164) -- dense grid query, global map, no grad
# --------------------------------------------------------------------------
def mesher_query_points(
    m: OracleMap,
    dec: DecoderParams,
    coord: torch.Tensor,
    nn_k: int,
    weighted_first: bool,
    color_dec: Optional[DecoderParams] = None,
    query_locally: bool = False,
    mask_min_nn_count: int = 4,
):
    """(sdf [N], color [N,Cc] or None, mc_mask [N] bool).  Rows without any neighbour keep sdf 0
    (`batch_sdf[pred_mask] = ...` with pred_mask = nn_count >= 1, mesher.py:118-131); the colour head decodes
    every row (mesher.py:143-146)."""
    with torch.no_grad():
        geo, col, w, nn_count, _ = query_feature(m, coord, None, nn_k, weighted_first, training_mode=False,
                                                 query_locally=query_locally,
                                                 query_color_feature=color_dec is not None)
        pred = nn_count >= 1
        if weighted_first:
            sdf = torch.zeros(coord.shape[0], dtype=coord.dtype)
            sdf[pred] = decoder_sdf(dec, geo[pred])
        else:
            s = torch.zeros(coord.shape[0], nn_k, 1, dtype=coord.dtype)
            s[pred] = decoder_sdf(dec, geo[pred].reshape(-1, geo.shape[-1])).reshape(-1, nn_k, 1)
            sdf = torch.sum(s * w, dim=1).squeeze(1)
        color = None
        if color_dec is not None:
            color = decoder_color(color_dec, col)
            if not weighted_first:
                color = torch.sum(color * w, dim=1)
        return sdf, color, nn_count >= mask_min_nn_count


# --------------------------------------------------------------------------
# a9/a10: registration step  (utils/tracker.py:367-611, 615-695)
# --------------------------------------------------------------------------
def skew(v):
    s = torch.zeros(3, 3, device=v.device, dtype=v.dtype)
    s[0, 1] = -v[2]
    s[0, 2] = v[1]
    s[1, 2] = -v[0]
    return s - s.T


def expmap(axis_angle: torch.Tensor) -> torch.Tensor:
    """utils/tracker.py:784-795 (no small-angle guard)."""
    angle = axis_angle.norm()
    axis = axis_angle / angle
    eye = torch.eye(3, device=axis_angle.device, dtype=axis_angle.dtype)
    s = skew(axis)
    return eye + s * torch.sin(angle) + (s @ s) * (1.0 - torch.cos(angle))


def implicit_reg(points, sdf_grad, sdf_residual, weight, lm_lambda=0.0):
    """utils/tracker.py:652-679.  Returns T [4,4] f64, N_raw [6,6] f32, g [6] f32."""
    cross = torch.linalg.cross(points, sdf_grad, dim=-1)
    j = torch.cat([cross, sdf_grad], -1)
    n_mat = j.T @ (weight * j)
    n_raw = n_mat.clone()
    n_mat = n_mat + lm_lambda * torch.diag(torch.diag(n_mat))
    g = -(j * weight).T @ sdf_residual
    t = torch.linalg.inv(n_mat.to(torch.float64)) @ g.to(torch.float64)
    tm = torch.eye(4, device=points.device, dtype=torch.float64)
    tm[:3, :3] = expmap(t[:3])
    tm[:3, 3] = t[3:]
    return tm, n_raw, g


def color_to_intensity(c):
    """utils/tools.py:408-410."""
    return (0.299 * c[:, 0] + 0.587 * c[:, 1] + 0.114 * c[:, 2]).unsqueeze(1)


def implicit_color_reg(points, sdf_grad, sdf_residual, color_grad, color_residual, weight, w_photo, lm_lambda):
    """utils/tracker.py:699-744.  color_grad [N,Cc,3], color_residual [N,Cc] (intensity: Cc=1)."""
    jg = torch.cat([torch.linalg.cross(points, sdf_grad), sdf_grad], -1)
    n_mat = jg.T @ (weight * jg)
    g = -(jg * weight).T @ sdf_residual
    for i in range(color_residual.shape[1]):
        jc = torch.cat([torch.linalg.cross(points, color_grad[:, i, :]), color_grad[:, i]], -1)
        n_mat = n_mat + w_photo * (jc.T @ (weight * jc))
        g = g + w_photo * (-(jc * weight).T @ color_residual[:, i])
    n_raw = n_mat.clone()
    n_mat = n_mat + lm_lambda * torch.diag(torch.diag(n_mat))
    t = torch.linalg.inv(n_mat.to(torch.float64)) @ g.to(torch.float64)
    tm = torch.eye(4, device=points.device, dtype=torch.float64)
    tm[:3, :3] = expmap(t[:3])
    tm[:3, 3] = t[3:]
    return tm, n_raw, g


def registration_step(
    points,
    sdf_pred,
    sdf_grad,
    sdf_std,
    nn_count,
    sdf_labels,
    min_nn: int,
    min_grad_norm: float,
    max_grad_norm: float,
    max_sdf_std: float,
    gm_dist: Optional[float],
    gm_grad: Optional[float],
    lm_lambda: float,
    normals: Optional[torch.Tensor] = None,
    colors: Optional[torch.Tensor] = None,
    color_pred: Optional[torch.Tensor] = None,
    color_grad: Optional[torch.Tensor] = None,
    photo_loss_on: bool = False,
    consist_weight_on: bool = True,
    w_photo: float = 0.01,
):
    """utils/tracker.py:409-546 (geometry, colour-consistency weight, photometric term)."""
    grad_norm = sdf_grad.norm(dim=-1, keepdim=True).squeeze()
    grad_unit = sdf_grad / grad_norm.unsqueeze(-1)
    mask = nn_count >= min_nn
    valid = mask & (grad_norm < max_grad_norm) & (grad_norm > min_grad_norm) & (sdf_std < max_sdf_std)
    vp = points[valid]
    nv = vp.shape[0]
    if nv < 10:
        return {
            "T": torch.eye(4, dtype=torch.float64, device=points.device),
            "valid_count": nv,
            "residual_cm": 0.0,
            "valid": valid,
        }
    gn = grad_norm[valid]
    sp = sdf_pred[valid]
    sg = sdf_grad[valid]
    sl = sdf_labels[valid]
    res = sp - sl
    residual_cm = torch.mean(torch.abs(res)).item() * 100.0
    w_grad = 1.0 if gm_grad is None else ((gm_grad / (gm_grad + (gn - 1.0) ** 2)) ** 2).unsqueeze(1)
    w_res = 1.0 if gm_dist is None else ((gm_dist / (gm_dist + res**2)) ** 2).unsqueeze(1)
    w_normal = (
        1.0
        if normals is None
        else (0.5 + torch.abs((normals[valid] * grad_unit[valid]).sum(dim=1))).unsqueeze(1)
    )
    w_color = 1.0
    col_res = None
    if colors is not None:
        c_obs, c_prd = colors[valid], color_pred[valid]
        if c_obs.shape[1] == 3:
            c_obs, c_prd = color_to_intensity(c_obs), color_to_intensity(c_prd)
        if photo_loss_on:
            cg = color_grad[valid]
            if cg.shape[1] == 3:
                cg = color_to_intensity(cg)  # [Nv,1,3]: linear in the channel dimension
            col_res = c_prd - c_obs
        elif consist_weight_on:
            w_color = torch.exp(-torch.mean(torch.abs(c_obs - c_prd), dim=-1)).unsqueeze(1)
    w = w_res * w_grad * w_normal * w_color
    if not isinstance(w, float):
        w = w / (2.0 * torch.mean(w))
    else:
        w = torch.full((nv, 1), w, device=points.device)
    if col_res is not None:
        tm, n_raw, g = implicit_color_reg(vp, sg, res, cg, col_res, w, w_photo, lm_lambda)
    else:
        tm, n_raw, g = implicit_reg(vp, sg, res, w, lm_lambda)
    return {
        "color_residual_mean": None if col_res is None else torch.mean(torch.abs(col_res)).item(),
        "T": tm,
        "N": n_raw,
        "g": g,
        "w": w,
        "valid": valid,
        "valid_count": nv,
        "residual_cm": residual_cm,
        "w_res2_mean": torch.mean(w.squeeze(1) * res**2),
    }


def transform_points(points: torch.Tensor, tmat: torch.Tensor) -> torch.Tensor:
    """utils/tools.py:534-553 (T cast to the point dtype, homogeneous matmul)."""
    ph = torch.cat([points, torch.ones(points.shape[0], 1).to(points)], dim=1)
    return torch.matmul(ph, tmat.to(points).T)[:, :3]


# --------------------------------------------------------------------------
# a12-a15: one mapping iteration  (utils/mapper.py:623-818, utils/loss.py:45-63)
# --------------------------------------------------------------------------
def sdf_bce_loss(pred, label, sigma, weight, weighted):
    """utils/loss.py:45-63."""
    target = torch.sigmoid(label / sigma)
    return torch.nn.functional.binary_cross_entropy_with_logits(
        pred / sigma, target, weight=weight if weighted else None, reduction="mean"
    )


def map_sdf(m, dec, x, nn_k, weighted_first, training_mode=False):
    """utils/mapper.py:940-956 (Mapper.sdf, accumulate_stability -> training_mode)."""
    geo, _, w, nn_count, _ = query_feature(m, x, None, nn_k, weighted_first, training_mode=training_mode)
    s = decoder_sdf(dec, geo)
    if not weighted_first:
        s = torch.sum(s * w, dim=1).squeeze(1)
    return s


def numerical_gradient(m, dec, x, eps, nn_k, weighted_first):
    """utils/mapper.py:986-1036 (two_side=True)."""
    n = x.shape[0]
    ex = torch.tensor([eps, 0.0, 0.0], dtype=x.dtype, device=x.device)
    ey = torch.tensor([0.0, eps, 0.0], dtype=x.dtype, device=x.device)
    ez = torch.tensor([0.0, 0.0, eps], dtype=x.dtype, device=x.device)
    xs = torch.concat((x + ex, x - ex, x + ey, x - ey, x + ez, x - ez), dim=0)
    s = map_sdf(m, dec, xs, nn_k, weighted_first).unsqueeze(-1)
    gx = (s[:n] - s[n : 2 * n]) / (2 * eps)
    gy = (s[2 * n : 3 * n] - s[3 * n : 4 * n]) / (2 * eps)
    gz = (s[4 * n : 5 * n] - s[5 * n :]) / (2 * eps)
    return torch.cat([gx, gy, gz], dim=1)


def mapping_loss(
    m: OracleMap,
    dec: DecoderParams,
    coord,
    sdf_label,
    ts,
    weight,
    nn_k: int,
    weighted_first: bool,
    sigma: float,
    loss_weight_on: bool,
    weight_e: float,
    grad_decimation: int,
    num_grad_eps: float,
    ekional_loss_on: bool = True,
    color_dec: Optional[DecoderParams] = None,
    color_label=None,
    surface_range: float = 0.0,
    weight_i: float = 1.0,
):
    """Forward part of one Mapper.mapping iteration (utils/mapper.py:645-812).
    ``m.local_geo_features`` (and colour) and the decoder tensors must already
    require grad.  Returns (loss, dict of parts)."""
    geo, col, w, _, _ = query_feature(
        m, coord, ts, nn_k, weighted_first, training_mode=True, query_color_feature=color_dec is not None
    )
    pred = decoder_sdf(dec, geo)
    if not weighted_first:
        pred = torch.sum(pred * w, dim=1).squeeze(1)
    parts = {"sdf_pred": pred.detach()}
    wabs = torch.abs(weight).detach()
    loss = sdf_bce_loss(pred, sdf_label, sigma, wabs, loss_weight_on)
    parts["bce"] = loss.detach()
    if ekional_loss_on and weight_e > 0:
        g = numerical_gradient(
            m, dec, coord[::grad_decimation], num_grad_eps, nn_k, weighted_first
        )
        eik = ((g.norm(2, dim=-1) - 1.0) ** 2).mean()
        parts["eikonal"] = eik.detach()
        loss = loss + weight_e * eik
    if color_dec is not None and weight_i > 0:
        cpred = decoder_color(color_dec, col)
        if not weighted_first:
            cpred = torch.sum(cpred * w, dim=1)
        smask = torch.abs(sdf_label) < surface_range
        diff = cpred[smask] - color_label[smask]
        wc = wabs[smask].unsqueeze(1) if loss_weight_on else 1.0
        closs = (wc * torch.abs(diff)).mean()
        parts["color"] = closs.detach()
        loss = loss + weight_i * closs
    return loss, parts


def make_adam(param_groups, lr=0.01, eps=1e-15, weight_decay=0.0):
    """utils/tools.py:153-203: Adam(betas=(0.9,0.99), eps=adam_eps); decoder groups
    first (wd 0), feature group last (wd = config.weight_decay)."""
    groups = []
    for i, ps in enumerate(param_groups):
        groups.append(
            {"params": ps, "lr": lr, "weight_decay": weight_decay if i == len(param_groups) - 1 else 0.0}
        )
    return torch.optim.Adam(groups, betas=(0.9, 0.99), eps=eps)


def idw_tangent_seeds(query, nb_points, valid):
    """Closed form of the forward-mode seeds the warp-specialised decode consumes (pin_slam_b200/csrc/query_dev.cuh:
    tangent_seeds), restated for the tests.  For one query q with K neighbours p_k (model/neural_points.py:665-683):
        u_k = 1 / (|q - p_k|^2 + 1e-15),  w_k = u_k / sum u   (invalid neighbours: 0)
        omega_kj = d w_k / d q_j = w_k (c_k d_kj - sum_m w_m c_m d_mj),   c_k = -2 u_k,  d_k = q - p_k
        P_ji = d (sum_k w_k (q - p_k))_i / d q_j = sum_k omega_kj (d_k - d_0)_i + (sum_k w_k) delta_ij
    query [N,3], nb_points [N,K,3], valid [N,K] bool -> (w [N,K], omega [N,K,3], P [N,3,3] with P[n,j,i])."""
    d = query.unsqueeze(1) - nb_points  # [N,K,3]
    u = (1.0 / ((d**2).sum(-1) + 1e-15)) * valid
    usum = u.sum(1, keepdim=True)
    w = torch.where(usum > 0, u / usum.clamp(min=1e-300), torch.zeros_like(u))
    c = -2.0 * u
    S = (w.unsqueeze(-1) * c.unsqueeze(-1) * d).sum(1, keepdim=True)  # [N,1,3]
    omega = w.unsqueeze(-1) * (c.unsqueeze(-1) * d - S)
    e = d - d[:, :1]
    P = torch.einsum("nkj,nki->nji", omega, e) + w.sum(1).view(-1, 1, 1) * torch.eye(3, dtype=query.dtype)
    return w, omega, P
