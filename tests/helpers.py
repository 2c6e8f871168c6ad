"""Shared test helpers: golden-fixture loading, seeded synthetic maps and the parity bounds of the kernel tests.

Tolerances (SURVEY.md section 8c):
  ids / counts / cell hashing : exact
  SDF                         : |d| <= 1e-5 * max(|ref|, sdf_scale)
  d sdf / d x                 : 1e-4 relative to max(|ref|, typical gradient scale)
  feature / decoder grads     : 1e-4 relative (float atomics reorder the sums)
  post-Adam parameters        : 1e-5 abs, a small fraction of near-zero-gradient outliers allowed
"""
import inspect
import os

import numpy as np
import torch

from oracle import pin_oracle as po

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PARITY_SLACK = []  # filled by assert_rel_close, reported by tests/conftest.py


# ---------------------------------------------------------------------------
# parity bounds
# ---------------------------------------------------------------------------
def assert_sdf_close(got, ref, scale, tol=1e-5):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    bound = tol * np.maximum(np.abs(ref), scale)
    bad = np.abs(got - ref) > bound
    assert not bad.any(), f"{bad.sum()} / {bad.size} sdf values differ; max err {np.abs(got - ref).max():.3e}"


def assert_rel_close(got, ref, tol, floor, ref64=None, kink_rows=0):
    """|got - ref| <= tol * max(|ref|, floor).  When the fp64 evaluation of the same algorithm is given, the
    fp32 reference's own rounding error |ref - ref64| is added to the bound (x4): a kernel only has to be
    as close to the fp64 truth as the fp32 reference is (SURVEY.md section 8c, "higher-precision oracle").

    `kink_rows`: derivatives of a ReLU network are discontinuous where a hidden pre-activation crosses zero; any
    reordering of the fp32 sums (cuBLAS vs MKL vs this kernel) flips the sign of pre-activations that lie within
    rounding of zero (~1e-6 of all activations), which changes that row's gradient by a finite amount.  Up to
    `kink_rows` rows may therefore miss the bound, with their error still limited to 10 % of the largest value."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    tight = tol * np.maximum(np.abs(ref), floor)
    bound = tight
    if ref64 is not None:
        bound = bound + 4.0 * np.abs(ref - np.asarray(ref64, np.float64))
    err = np.abs(got - ref)
    bad = err > bound
    # how much of the allowance was actually used (reported at the end of the session, tests/conftest.py)
    rows_bad = int(bad.reshape(bad.shape[0], -1).any(axis=1).sum()) if bad.ndim else int(bad)
    PARITY_SLACK.append({
        "test": next((f.function for f in inspect.stack() if f.function.startswith("test_")), "?"),
        "elements": int(err.size), "tol": tol, "over_tight_bound": int((err > tight).sum()),
        "needed_fp64_slack": int(((err > tight) & ~bad).sum()), "kink_rows_used": rows_bad if kink_rows else 0,
        "kink_rows_allowed": int(kink_rows), "max_err_over_tight_bound": float((err / np.maximum(tight, 1e-300)).max())})
    if kink_rows and bad.any():
        rows = bad.reshape(bad.shape[0], -1).any(axis=1)
        assert rows.sum() <= kink_rows, f"{int(rows.sum())} rows miss the bound (allowed {kink_rows}); max err {err.max():.3e}"
        assert err.max() <= 0.1 * np.abs(ref).max(), f"kink-row error {err.max():.3e} too large"
        return
    assert not bad.any(), f"max err {err.max():.3e} (bound {bound.min():.3e}); {int(bad.sum())} bad"


def assert_decoder_grad_close(got, ref, ref64):
    """Decoder gradients are sums over ALL sample rows, so one ReLU kink flip (see assert_rel_close) shifts every
    entry a little instead of one row a lot: tight bound first, else the kink-level bound 5e-3 of the largest
    entry on the maximum and 1e-3 on the median (a wrong kernel is off by O(1))."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = np.abs(ref).max()
    try:
        assert_rel_close(got, ref, 1e-4, scale * 5e-2, ref64)
    except AssertionError:
        err = np.abs(got - ref)
        assert err.max() <= 5e-3 * scale and np.median(err) <= 1e-3 * scale, \
            f"decoder gradient: max err {err.max():.3e}, median {np.median(err):.3e}, scale {scale:.3e}"


def assert_close_frac(a, b, atol=1e-5, max_bad_frac=5e-3, max_abs=4e-2):
    """Parameters after a few Adam steps: Adam's eps 1e-15 turns near-zero gradients into +-lr steps whose sign
    follows the summation order, so a small fraction of entries may differ by up to a few lr."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    bad = np.abs(a - b) > atol + 1e-5 * np.abs(b)
    assert bad.mean() <= max_bad_frac, f"{bad.sum()} / {bad.size} differ, max {np.abs(a - b).max():.2e}"
    assert np.abs(a - b).max() <= max_abs


def oracle64(m, dec, q, k, wf, ref32, **kw):
    """fp64 run of the oracle; rows whose neighbour set differs from the fp32 run (a query within one ulp
    of a voxel boundary) fall back to the fp32 values."""
    kw = {a: (b.double() if isinstance(b, po.DecoderParams) else b) for a, b in kw.items()}
    r64 = po.query_sdf(m.double(), dec.double(), q.double(), k, wf, **kw)
    same = (r64["nn_count"] == ref32["nn_count"]).numpy()
    out = {}
    for name in ("sdf", "grad", "sdf_std", "color", "color_grad"):
        if name in r64 and name in ref32:
            a, b = r64[name].numpy(), np.asarray(ref32[name], np.float64)
            sel = same.reshape((-1,) + (1,) * (a.ndim - 1))
            out[name] = np.where(sel, a, b)
    return out


def load_npz(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def t(x, dtype=None):
    y = torch.from_numpy(np.ascontiguousarray(x))
    return y if dtype is None else y.to(dtype)


def map_from_fixture(fx, device="cpu") -> po.OracleMap:
    g = lambda k: fx["map." + k]  # noqa: E731
    bsz = int(g("buffer_size"))
    table = torch.full((bsz,), -1, dtype=torch.int64)
    table[t(g("table_slots"))] = t(g("table_vals"))
    m = po.OracleMap(
        resolution=float(g("resolution")),
        buffer_size=bsz,
        feature_dim=int(g("geo_features").shape[1]),
        neural_points=t(g("neural_points")),
        point_orientations=t(g("point_orientations")),
        geo_features=t(g("geo_features")),
        color_features=t(g("color_features")) if "map.color_features" in fx else None,
        point_ts_create=t(g("point_ts_create")),
        point_ts_update=t(g("point_ts_update")),
        point_certainties=t(g("point_certainties")),
        buffer_pt_index=table,
        local_neural_points=t(g("local_neural_points")),
        local_point_orientations=t(g("local_point_orientations")),
        local_geo_features=t(g("local_geo_features")),
        local_color_features=t(g("local_color_features")) if "map.local_color_features" in fx else None,
        local_point_certainties=t(g("local_point_certainties")),
        local_point_ts_update=t(g("local_point_ts_update")),
        local_mask=t(g("local_mask")),
        global2local=t(g("global2local")),
        neighbor_dx=t(g("neighbor_dx")),
        max_valid_dist2=float(g("max_valid_dist2")),
        travel_dist=t(g("travel_dist")),
        cur_ts=int(g("cur_ts")),
        diff_travel_dist_local=float(g("diff_travel_dist_local")),
        temporal_local_map_on=bool(g("temporal_local_map_on")),
        after_pgo=bool(g("after_pgo")),
    )
    return m.to(device)


def decoder_from_fixture(fx, name, device="cpu") -> po.DecoderParams:
    hidden = []
    i = 0
    while f"{name}.layers.{i}.weight" in fx:
        hidden.append((t(fx[f"{name}.layers.{i}.weight"]), t(fx[f"{name}.layers.{i}.bias"])))
        i += 1
    out = (t(fx[f"{name}.lout.weight"]), t(fx[f"{name}.lout.bias"]))
    return po.DecoderParams(hidden, out, float(fx[f"{name}.sdf_scale"])).to(device)


def synthetic_surface_points(n, seed, extent=20.0):
    """Random points on a floor, walls and a few boxes of a closed room (metres)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda k: torch.rand(k, generator=g)  # noqa: E731
    k = n // 5
    lo, hi = -extent / 2, extent / 2
    u = lambda k: r(k) * (hi - lo) + lo  # noqa: E731
    parts = [
        torch.stack([u(k), u(k), torch.zeros(k)], 1),
        torch.stack([u(k), torch.full((k,), hi), r(k) * 4], 1),
        torch.stack([torch.full((k,), lo), u(k), r(k) * 4], 1),
        torch.stack([u(k), torch.full((k,), lo), r(k) * 4], 1),
        torch.stack([r(n - 4 * k) * 3 + 2, r(n - 4 * k) * 3 - 5, torch.full((n - 4 * k,), 1.5)], 1),
    ]
    p = torch.cat(parts, 0)
    return p + 0.01 * torch.randn(p.shape, generator=g)


def synthetic_map(n_surface=20000, seed=0, resolution=0.4, buffer_size=int(5e7), feature_dim=8,
                  color=False, extent=20.0, n_ts=3, local_radius=None, diff_td=1e9, after_pgo=False,
                  num_nei_cells=2, search_alpha=0.2):
    """A seeded OracleMap built with oracle.build_map (one neural point per voxel)."""
    g = torch.Generator().manual_seed(seed + 17)
    pts = synthetic_surface_points(n_surface, seed, extent)
    cells = po.cell_of(pts, resolution)
    _, first = np.unique(cells.numpy(), axis=0, return_index=True)
    first = torch.from_numpy(np.sort(first))
    sp = pts[first].contiguous()
    mg = sp.shape[0]
    geo = 0.1 * torch.randn(mg + 1, feature_dim, generator=g)
    col = 0.1 * torch.randn(mg + 1, feature_dim, generator=g) if color else None
    ts = torch.randint(0, n_ts, (mg,), generator=g).to(torch.int32)
    cert = torch.rand(mg, generator=g) * 3
    ori = None
    if after_pgo:
        qn = torch.randn(mg, 4, generator=g)
        ori = qn / qn.norm(dim=1, keepdim=True)
    m = po.build_map(sp, resolution, buffer_size, geo, col, ts, cert, ori, num_nei_cells, search_alpha)
    m.after_pgo = after_pgo
    m.travel_dist = torch.arange(n_ts + 1, dtype=torch.float32) * 2.0
    m.diff_travel_dist_local = diff_td
    sensor = torch.tensor([0.0, 0.0, 1.0])
    po.reset_local_map(m, sensor, local_radius if local_radius is not None else 1e6, n_ts - 1)
    return m


def queries_near(m, n, seed, sigma=0.15):
    g = torch.Generator().manual_seed(seed)
    sel = torch.randint(0, m.neural_points.shape[0], (n,), generator=g)
    return (m.neural_points[sel] + sigma * torch.randn(n, 3, generator=g)).contiguous()


# ---------------------------------------------------------------------------
# K2 cases: the instantiation each one must launch (read by the coverage ledger of tests/test_query_paths.py)
# ---------------------------------------------------------------------------
def train_bwd_kernel_name(F, L, aligned=True):
    """The K2 kernel pinb200_train_backward launches for a 64-wide decoder with L hidden layers on F features
    (dispatch_train in train.cu: the tensor-core kernel for 1-2 layers on a 16-byte aligned feature table, else the
    SIMT kernel by padded input width)."""
    if L <= 2 and aligned:
        return f"train_bwd_mma_kernel<{F}, {L}>"
    return f"train_bwd_kernel<64, {next(dp for dp in (12, 20, 36, 68) if F + 3 <= dp)}>"


# (F, K, L, weighted_first, out_dim, after_pgo, leaky, bias, aligned) of
# test_cuda_parity.py::test_train_backward_vs_autograd_synthetic.  aligned=False: the feature table starts 4 bytes
# past a 16-byte boundary.  The SIMT kernel's shared memory fits 3 hidden layers only for F <= 8, so its wider
# instantiations run on 1-2 layer decoders over such tables.
TRAIN_BWD_CASES = [
    (8, 6, 1, False, 1, False, False, True, True), (8, 6, 1, True, 1, False, False, True, True),
    (4, 4, 1, True, 1, True, False, True, True), (16, 5, 2, False, 1, False, False, True, True),
    (32, 8, 2, True, 1, False, False, True, True), (64, 8, 1, False, 1, True, False, True, True),
    (64, 3, 2, True, 3, False, False, True, True), (8, 6, 2, False, 3, False, False, True, True),
    (4, 6, 3, True, 1, False, False, True, True),
    (16, 4, 1, True, 1, False, True, False, True), (32, 7, 1, False, 1, False, False, False, True),
    (4, 5, 2, False, 3, True, True, True, True), (8, 6, 2, True, 1, False, False, False, True),
    (32, 8, 2, False, 3, False, True, False, True), (8, 5, 3, False, 1, False, True, False, True),
    (16, 6, 2, False, 1, False, True, True, False), (32, 8, 1, True, 1, True, False, False, False),
    (64, 3, 2, False, 3, False, False, True, False),
]


def kernels_run(fn, tries=3):
    """fn() under torch.profiler with CUDA activity: (its result, the demangled names of the kernels it launched).
    Now and then the profiler loses a whole activity buffer, and the trace holds no kernel at all; fn() then runs
    again (up to `tries` times), so it must be repeatable."""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = {e.key for e in prof.key_averages()}
        if any("pinb::" in k for k in names):
            break
    return out, names


# ---------------------------------------------------------------------------
# CUDA-side helpers (only used by -m gpu tests, smoke and bench)
# ---------------------------------------------------------------------------
def map_handle_from_oracle(m, query_locally=True, device="cuda", color=True):
    """Upload an OracleMap's tensors and wrap them in a pin_slam_b200.ops.MapHandle."""
    from pin_slam_b200 import ops

    dev = torch.device(device)
    up = lambda x, dt=None: None if x is None else (x if dt is None else x.to(dt)).contiguous().to(dev)  # noqa: E731
    local = query_locally
    return ops.MapHandle(
        slot_table=up(m.buffer_pt_index, torch.int32),
        buffer_size=m.buffer_size,
        points=up(m.neural_points),
        ts_create=up(m.point_ts_create, torch.int32),
        travel_dist=up(m.travel_dist),
        global2local=up(m.global2local, torch.int32) if local else None,
        nb_points=up(m.local_neural_points if local else m.neural_points),
        nb_orient=up(m.local_point_orientations if local else m.point_orientations),
        geo_feat=up((m.local_geo_features if local else m.geo_features).detach()),
        color_feat=up((m.local_color_features if local else m.color_features).detach())
        if (color and m.color_features is not None) else None,
        certainty=up(m.local_point_certainties if local else m.point_certainties),
        ts_update=up(m.local_point_ts_update if local else m.point_ts_update, torch.int32),
        probe_dx=up(m.neighbor_dx, torch.int32),
        resolution=m.resolution,
        max_valid_dist2=m.max_valid_dist2,
        time_filter=m.temporal_local_map_on and local,
        cur_ts=m.cur_ts,
        diff_travel_dist_local=m.diff_travel_dist_local,
        after_pgo=m.after_pgo,
    )


def decoder_handle_from_oracle(dec, device="cuda", sigmoid_out=False, bias=True):
    """`bias=False`: a decoder without biases (mlp_bias_on False) -- the handle passes NULL bias pointers; the oracle
    decoder (po.make_decoder(..., bias=False)) keeps zero biases, which gives the same forward pass."""
    from pin_slam_b200 import ops

    dev = torch.device(device)
    ws = [w.detach().contiguous().to(dev) for w, _ in dec.hidden]
    bs = [b.detach().contiguous().to(dev) if bias else None for _, b in dec.hidden]
    bo = dec.out[1].detach().contiguous().to(dev) if bias else None
    return ops.DecoderHandle(ws, bs, dec.out[0].detach().contiguous().to(dev), bo,
                             out_scale=1.0 if sigmoid_out else dec.sdf_scale, leaky=dec.leaky, sigmoid_out=sigmoid_out)


def flat_decoder_params(dec, bias=True):
    """[w0|b0|w1|b1|...|w_out|b_out] -- the layout pinb200_train_backward / adam use; `bias=False` leaves the bias
    blocks out, as Decoder.flat_parameters() does for a decoder without biases."""
    parts = []
    for w, b in dec.hidden:
        parts += [w.detach().reshape(-1)] + ([b.detach().reshape(-1)] if bias else [])
    parts += [dec.out[0].detach().reshape(-1)] + ([dec.out[1].detach().reshape(-1)] if bias else [])
    return torch.cat(parts)
