"""Map-maintenance, probe-index, registration and loss kernels at full-run sizes and at their decision boundaries.

Every case compares a kernel with a plain formulation written here (torch on the CPU, numpy, or fp64 where the
contract is a bound) or with the drop-in class's own CPU path, which tests/test_oracle_golden.py pins to the reference
fixtures.  The sizes are derived from the kernels' block constants (read from the sources) and the device's SM count,
so that they cross the multi-pass block-sum scans and the grid-stride loops on any H100:
  * pool filter / local map / map growth: single-CTA scans over chunks of SCAN_CHUNK block sums, one more pass per
    chunk (pool.cu PF_IPB samples, localmap.cu LM_TPB points, mapgrow.cu MG_TPB candidates per block);
  * K4 / loss heads / Adam: grid-stride loops above 2 / 4 / 8 x SMs x 256 items;
  * probe index: SCAN_WPBLK words of 32 slots per block.
The distance tests of the pool filter, the local map and map growth are probed with crafted samples whose squared
distance rounds to the other side of the threshold than its exact value: a kernel that contracts the sum of squares
into fused multiply-adds decides them like the exact value, torch decides them like the rounded one.

`test_kernel_ledger` (no GPU) checks that every __global__ kernel of pin_slam_b200/csrc is named in KERNEL_LEDGER by a
test that launches it; the GPU tests of this file assert through tests.helpers.kernels_run that they launch the
kernels the ledger gives them."""
import functools
import os
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

from tests.helpers import kernels_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pin_slam_b200", "csrc")
gpu = pytest.mark.gpu


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(name, file):
    m = re.search(rf"constexpr int {name} = (\d+);", _src(file))
    assert m, f"{name} not found in {file}"
    return int(m.group(1))


PF_IPB = _const("PF_TPB", "pool.cu") * _const("PF_IPT", "pool.cu")  # samples per pool-filter block
LM_TPB = _const("LM_TPB", "localmap.cu")                             # neural points per local-map block
MG_TPB = _const("MG_TPB", "mapgrow.cu")                              # candidates per map-growth block
PROBE_WPBLK = _const("SCAN_TPB", "probe_index.cu") * _const("SCAN_WPT", "probe_index.cu")  # probe words per block
SCAN_CHUNK = 1024  # block sums per pass of the single-CTA scans (pool_scan_kernel & co. run 1024 threads)
PRIMES = np.array([73856093, 19349669, 83492791], dtype=np.int64)
REC_REMAP = 1 << 30
SENT_F, SENT_I = -12345.0, -12345  # sentinel written behind every output


@functools.lru_cache(None)
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _lib():
    from pin_slam_b200 import _lib

    return _lib.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# --------------------------------------------------------------------------------------
# kernel ledger
# --------------------------------------------------------------------------------------
_QUERY_LEDGER = "test_query_paths::test_coverage_ledger"
KERNEL_LEDGER = {
    # this file
    "pool_count_kernel": "test_map_kernels::test_pool_filter_compaction",
    "pool_scan_kernel": "test_map_kernels::test_pool_filter_compaction",
    "pool_scatter_kernel": "test_map_kernels::test_pool_filter_compaction",
    "local_recent_kernel": "test_map_kernels::test_reset_local_map_matches_cpu",
    "local_keep_kernel": "test_map_kernels::test_reset_local_map_matches_cpu",
    "local_scan_kernel": "test_map_kernels::test_reset_local_map_matches_cpu",
    "local_gather_kernel": "test_map_kernels::test_reset_local_map_matches_cpu",
    "grow_flag_kernel": "test_map_kernels::test_map_grow_matches_sequential_rule",
    "grow_scan_kernel": "test_map_kernels::test_map_grow_matches_sequential_rule",
    "grow_append_kernel": "test_map_kernels::test_map_grow_matches_sequential_rule",
    "grow_table_kernel": "test_map_kernels::test_map_grow_matches_sequential_rule",
    "probe_mark_kernel": "test_map_kernels::test_probe_index_layout",
    "probe_blocksum_kernel": "test_map_kernels::test_probe_index_layout",
    "probe_scan_blocksums_kernel": "test_map_kernels::test_probe_index_layout",
    "probe_prefix_kernel": "test_map_kernels::test_probe_index_layout",
    "probe_scatter_kernel": "test_map_kernels::test_probe_index_layout",
    "gn_accumulate_kernel": "test_map_kernels::test_gn_step_vs_fp64",
    "gn_solve_kernel": "test_map_kernels::test_gn_step_vs_fp64",
    "mapping_loss_kernel": "test_map_kernels::test_mapping_loss_vs_fp64_autograd",
    "color_loss_kernel": "test_map_kernels::test_color_loss_vs_fp64_autograd",
    # other files
    "adam_kernel": "test_cuda_parity::test_adam_matches_torch",
    "assemble_batch_kernel": "test_cuda_parity::test_assemble_batch_bit_exact_and_mapping_equivalent",
    "knn_kernel": "test_cuda_parity::test_knn_and_features_match_reference",
    "gather_kernel": "test_cuda_parity::test_knn_and_features_match_reference",
    "radius_kernel": "test_cuda_parity::test_radius_search_matches_reference_bit_exact",
    "voxel_bounds_kernel": "test_cuda_frame_parity::test_cuda_voxel_downsample_equals_reference_formulation",
    "voxel_insert_kernel": "test_cuda_frame_parity::test_cuda_voxel_downsample_equals_reference_formulation",
    "voxel_compact_kernel": "test_cuda_frame_parity::test_cuda_voxel_downsample_equals_reference_formulation",
    "frame_transform_kernel": "test_cuda_frame_parity::test_cuda_loop_closure_transform_matches_reference",
    "ray_sample_kernel": "test_cuda_frame_parity::test_cuda_ray_sampler_kernel_equals_torch_formulation",
    "sort_key_kernel": "test_query_sort::test_sort_runs_and_host_query_with_chunks_is_bit_identical",
    "sort_scatter_kernel": "test_query_sort::test_sort_runs_and_host_query_with_chunks_is_bit_identical",
    # the query and training families: every instantiation is covered by the coverage ledger of test_query_paths.py
    "query_kernel": _QUERY_LEDGER,
    "search_kernel": _QUERY_LEDGER,
    "wsq_decode_kernel": _QUERY_LEDGER,
    "train_bwd_kernel": _QUERY_LEDGER,
    "train_bwd_mma_kernel": _QUERY_LEDGER,
}


def global_kernels():
    """Names of the __global__ functions defined (with a body) in pin_slam_b200/csrc/*.cu and *.cuh."""
    names = set()
    for f in sorted(os.listdir(CSRC)):
        if not f.endswith((".cu", ".cuh")):
            continue
        s = re.sub(r"//[^\n]*|/\*.*?\*/", " ", _src(f), flags=re.S)
        for m in re.finditer(r"\b__global__\b", s):
            i = m.end()
            name = None
            while True:  # skip return type, qualifiers and __launch_bounds__(...) (its arguments may hold parentheses)
                t = re.compile(r"\s*([A-Za-z_]\w*)").match(s, i)
                assert t, f"{f}: cannot parse the kernel after offset {m.start()}"
                i = t.end()
                if t.group(1) == "__launch_bounds__":
                    depth, i = 0, s.index("(", i)
                    while True:
                        depth += {"(": 1, ")": -1}.get(s[i], 0)
                        i += 1
                        if depth == 0:
                            break
                    continue
                if re.compile(r"\s*\(").match(s, i):
                    name = t.group(1)
                    break
            depth, i = 0, s.index("(", i)  # the parameter list, then a body '{' (definition) or ';' (declaration)
            while True:
                depth += {"(": 1, ")": -1}.get(s[i], 0)
                i += 1
                if depth == 0:
                    break
            if re.compile(r"\s*\{").match(s, i):
                names.add(name)
    return names


def _check_launched(names, test):
    """Every kernel the ledger gives `test` was launched (names: demangled kernel names from kernels_run)."""
    want = [k for k, v in KERNEL_LEDGER.items() if v == "test_map_kernels::" + test]
    assert want
    missing = [k for k in want if not any(re.search(rf"\bpinb::{k}\b", n) for n in names)]
    assert not missing, (missing, sorted(n for n in names if "pinb::" in n))


def _launched(fn, *kernels):
    out, names = kernels_run(fn)
    missing = [k for k in kernels if not any(re.search(rf"\bpinb::{k}\b", n) for n in names)]
    assert not missing, (missing, sorted(n for n in names if "pinb::" in n))
    return out, names


# --------------------------------------------------------------------------------------
# crafted distance-test boundaries: exact arithmetic
# --------------------------------------------------------------------------------------
def _round_to(x: Fraction, dt):
    """x rounded to the nearest `dt` value, ties to even (float() of a Fraction is correctly rounded to fp64; fp32 is
    picked among the neighbours of the fp64 value, which avoids double rounding)."""
    if dt is np.float64:
        return np.float64(float(x))
    c = np.float32(float(x))
    cands = [np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))]
    errs = [abs(Fraction(float(v)) - x) for v in cands]
    best = min(errs)
    tied = [v for v, e in zip(cands, errs) if e == best]
    return tied[0] if len(tied) == 1 else next(v for v in tied if int(v.view(np.int32)) % 2 == 0)


def _fma(a, b, c, dt):
    return _round_to(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)), dt)


def _craft(rng, dt, count, radius, less):
    """`count` crafted cases (p [3] fp32, o [3] dt, threshold thr of type dt).  d = p - o is rounded to dt; the sum of
    squares S = ((dx*dx + dy*dy) + dz*dz) with every operation rounded (what torch computes) and the exact value E lie
    on different sides of thr, and so do S and every DFMA/FFMA contraction of the sum (which all decide like E):
      less=True : the test is S < thr  (pool filter, local-map radius)
      less=False: the test is S > thr  (map growth, far2)"""
    out = []
    tries = 0
    while len(out) < count:
        tries += 1
        assert tries < 200 * count, "too few crafted samples qualify"
        o = (rng.uniform(-30, 30, 3) + rng.uniform(0, 1, 3) * 1e-3).astype(dt)
        u = rng.normal(size=3)
        p = (o.astype(np.float64) + u / np.linalg.norm(u) * radius * rng.uniform(0.97, 1.03)).astype(np.float32)
        d = p.astype(dt) - o
        S = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
        E = sum(Fraction(float(v)) ** 2 for v in d)
        sq = [_round_to(Fraction(float(v)) ** 2, dt) for v in d]
        fmas = [_fma(d[2], d[2], _fma(d[1], d[1], sq[0], dt), dt), _fma(d[2], d[2], _fma(d[0], d[0], sq[1], dt), dt),
                _fma(d[2], d[2], sq[0] + sq[1], dt)]
        s_frac = Fraction(float(S))
        up, down = np.nextafter(S, dt(np.inf)), np.nextafter(S, dt(-np.inf))
        if less:
            if s_frac > E:
                thr = S  # S < thr false, E < thr true
                ok = all(f < thr for f in fmas)
            elif Fraction(float(up)) <= E:
                thr = up  # S < thr true, E < thr false
                ok = all(f >= thr for f in fmas)
            else:
                continue
        else:
            if s_frac < E:
                thr = S  # S > thr false, E > thr true
                ok = all(f > thr for f in fmas)
            elif Fraction(float(down)) >= E:
                thr = down  # S > thr true, E > thr false
                ok = all(f <= thr for f in fmas)
            else:
                continue
        if ok:
            out.append((p, o, thr))
    return out


def _embed(rng, o, radius, k=63):
    """k random fp32 samples around o, none of them within 10 % of the threshold radius."""
    u = rng.normal(size=(k, 3))
    r = np.where(rng.random(k) < 0.5, rng.uniform(0.1, 0.9, k), rng.uniform(1.1, 2.0, k)) * radius
    return (o.astype(np.float64) + u / np.linalg.norm(u, axis=1, keepdims=True) * r[:, None]).astype(np.float32)


# --------------------------------------------------------------------------------------
# 1a. pool filter
# --------------------------------------------------------------------------------------
POOL_ORIGIN = (3.1, -7.3, 0.7)  # fp64, not representable in fp32
POOL_NS = [1, PF_IPB - 1, PF_IPB, PF_IPB + 1, PF_IPB * SCAN_CHUNK, PF_IPB * SCAN_CHUNK + 1, 5_000_037]
_CACHE = {}


def _pool_src(n):
    """Seeded pool of n samples on the device (and a CPU copy).  In the patterned mix (radius 50 around POOL_ORIGIN)
    samples i % 2048 == 0 and every other i % 8 == 4 are kept, i % 2048 == 1024 and the other i % 8 == 4 dropped: the
    first fresh sample can then be put on a block or a thread boundary, kept or dropped."""
    if n in _CACHE:
        return _CACHE[n]
    _CACHE.clear()
    g = torch.Generator(device="cuda").manual_seed(n)
    o32 = torch.tensor(POOL_ORIGIN, dtype=torch.float32, device="cuda")
    gc = torch.rand(n, 3, generator=g, device="cuda") * 120 - 60 + o32
    i = torch.arange(n, device="cuda")
    gc[(i // 700) % 3 == 0] += 500.0  # runs of dropped samples across thread and block boundaries
    near, far = o32 + 0.25, o32 + 400.0
    gc[i % 2048 == 0] = near
    gc[i % 2048 == 1024] = far
    gc[(i % 8 == 4) & ((i // 8) % 2 == 0)] = near
    gc[(i % 8 == 4) & ((i // 8) % 2 == 1)] = far
    src = {"coord": torch.rand(n, 3, generator=g, device="cuda"), "gcoord": gc.contiguous(),
           "label": torch.randn(n, generator=g, device="cuda"), "weight": torch.rand(n, generator=g, device="cuda"),
           "ts": torch.randint(0, 1 << 20, (n,), generator=g, device="cuda", dtype=torch.int32),
           "color": torch.rand(n, 3, generator=g, device="cuda")}
    _CACHE[n] = (src, {k: v.cpu() for k, v in src.items()})
    return _CACHE[n]


_POOL_FIELDS = ("coord", "gcoord", "label", "weight", "ts", "color")


def _pool_filter(src, cc, n_tail, origin64, r2, out=None, scratch=None, counts=None):
    """pinb200_pool_filter into sentinel-filled arenas with 8 spare rows; returns (out dict, counts [2])."""
    lib = _lib()
    n = src["label"].shape[0]
    if out is None:
        out = {k: torch.empty((n + 8,) + tuple(src[k].shape[1:]) if k != "color" else (n + 8, cc),
                              dtype=src[k].dtype, device="cuda") for k in _POOL_FIELDS if k != "color" or cc}
    for v in out.values():
        v.fill_(SENT_I if v.dtype == torch.int32 else SENT_F)
    if scratch is None:
        scratch = torch.empty(int(lib.pinb200_pool_filter_scratch(max(n, 1))), dtype=torch.int32, device="cuda")
        counts = torch.empty(2, dtype=torch.int64, device="cuda")
    col = src["color"][:, :cc].contiguous() if cc else None
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    rc = lib.pinb200_pool_filter(p(src["coord"]), p(src["gcoord"]), p(src["label"]), p(src["weight"]), p(src["ts"]),
                                 p(col), cc, n, int(n_tail), origin64.data_ptr(), float(r2), p(out["coord"]),
                                 p(out["gcoord"]), p(out["label"]), p(out["weight"]), p(out["ts"]), p(out.get("color")),
                                 scratch.data_ptr(), counts.data_ptr(), _stream())
    assert rc == 0
    return out, scratch, counts


def _pool_tails(n):
    firsts = {4, 12, PF_IPB, 2 * PF_IPB, PF_IPB * SCAN_CHUNK, PF_IPB * SCAN_CHUNK + PF_IPB}
    return sorted({1, n} | {n - f for f in firsts if 0 < f < n})


@gpu
@pytest.mark.parametrize("cc", [0, 1, 3])
@pytest.mark.parametrize("n", POOL_NS)
def test_pool_filter_compaction(n, cc):
    """pinb200_pool_filter equals the CPU branch of Mapper.process_frame (mask, boolean-mask compaction of every
    array, keep[-n_tail:].sum()) exactly, for no / all / a patterned mix of kept samples, with nothing written
    behind the kept rows."""
    src, cpu = _pool_src(n)
    origin = torch.tensor(POOL_ORIGIN, dtype=torch.float64)
    origin_d = origin.cuda()
    first = True
    out = scratch = counts = None
    for r2 in (0.0, 1e30, 50.0**2):
        keep = ((cpu["gcoord"] - origin) ** 2).sum(-1) < r2  # torch promotes the fp32 pool to fp64
        kept = int(keep.sum())
        exp = {k: (cpu[k][:, :cc] if k == "color" else cpu[k])[keep].cuda() for k in _POOL_FIELDS if k != "color" or cc}
        for n_tail in _pool_tails(n):
            if first:
                (out, scratch, counts), _ = _launched(lambda: _pool_filter(src, cc, n_tail, origin_d, r2),
                                                      "pool_count_kernel", "pool_scan_kernel", "pool_scatter_kernel")
                first = False
            else:
                _pool_filter(src, cc, n_tail, origin_d, r2, out, scratch, counts)
            assert counts.tolist() == [kept, int(keep[n - n_tail:].sum())], (r2, n_tail)
            for k, e in exp.items():
                assert torch.equal(out[k][:kept], e), (k, r2, n_tail)
                sent = SENT_I if e.dtype == torch.int32 else SENT_F
                assert bool((out[k][kept:] == sent).all()), (k, r2, n_tail)


# --------------------------------------------------------------------------------------
# 1b. local map
# --------------------------------------------------------------------------------------
def _npm(device, pts, ts_c, ts_u, cert, ori, geo, travel, radius, use_mid_ts, reboot_ts):
    from pin_slam_b200.config import HotPathConfig
    from pin_slam_b200.model import NeuralPoints

    cfg = HotPathConfig.kitti(device=device, feature_dim=geo.shape[1], buffer_size=1009, local_map_radius=radius,
                              use_mid_ts=use_mid_ts)
    npm = NeuralPoints(cfg)
    dev = torch.device(device)
    npm.neural_points, npm.point_ts_create, npm.point_ts_update = pts.to(dev), ts_c.to(dev), ts_u.to(dev)
    npm.point_certainties, npm.point_orientations, npm.geo_features = cert.to(dev), ori.to(dev), geo.to(dev)
    npm.travel_dist = travel.to(dev)
    npm.diff_travel_dist_local = 5.0
    npm.reboot_ts = reboot_ts
    return npm


def _local_case(n, seed, n_recent=None, near=None):
    """Seeded global map of n points.  n_recent: exactly that many points are recent (ts_create == cur_ts, the others
    far behind in time and travel distance).  near: only points 0 and 1 (at distances 1 and 2 from the sensor) can
    be within the radius."""
    g = torch.Generator().manual_seed(seed)
    pts = torch.rand(n, 3, generator=g) * 200 - 100
    cur = 40
    ts_c = torch.randint(0, cur + 1, (n,), generator=g, dtype=torch.int32)
    ts_u = torch.minimum(ts_c + torch.randint(0, 8, (n,), generator=g, dtype=torch.int32), torch.tensor(cur))
    travel = (torch.arange(cur + 1, dtype=torch.float32) * 0.5).contiguous()  # exact ties with diff 5.0
    if n_recent is not None:
        ts_c = torch.zeros(n, dtype=torch.int32)
        ts_c[torch.randperm(n, generator=g)[:n_recent]] = cur
        ts_u = ts_c.clone()
        travel[cur] = 1000.0
    if near is not None:
        pts = pts.abs() + 50.0
        pts[0], pts[1] = torch.tensor([1.0, 0.0, 0.0]), torch.tensor([0.0, 2.0, 0.0])
    cert = torch.rand(n, generator=g)
    ori = torch.randn(n, 4, generator=g)
    geo = torch.randn(n + 1, 4, generator=g)
    return pts, ts_c, ts_u, cert, ori, geo, travel, cur


# (temporal, use_travel_dist, use_mid_ts, reboot_map, sensor dtype)
LOCAL_OPTS = [(False, True, False, False, torch.float64), (True, True, False, False, torch.float64),
              (True, True, True, True, torch.float32), (True, False, False, True, torch.float64),
              (True, False, True, False, torch.float32), (False, True, False, True, torch.float32)]


def _compare_local(a, b, what):
    for name in ("local_mask", "global2local", "_local_idx", "local_neural_points", "local_point_orientations",
                 "local_point_certainties", "local_point_ts_update", "local_geo_features"):
        x, y = getattr(a, name), getattr(b, name)
        assert torch.equal(x.detach().cpu(), y.detach()), (name, what)


def _reset_both(case, opts, sensor, radius):
    pts, ts_c, ts_u, cert, ori, geo, travel, cur = case
    temporal, use_td, mid, reboot, sdt = opts
    res = []
    for dev in ("cuda", "cpu"):
        npm = _npm(dev, pts, ts_c, ts_u, cert, ori, geo, travel, radius, mid, reboot_ts=cur - 6)
        npm.temporal_local_map_on = temporal
        npm.reset_local_map(sensor.to(sdt).to(dev), torch.eye(3, device=dev), cur, use_travel_dist=use_td,
                            diff_ts_local=9, reboot_map=reboot)
        res.append(npm)
    return res


@gpu
@pytest.mark.parametrize("n", [0, 1, LM_TPB - 1, LM_TPB, LM_TPB * SCAN_CHUNK - 1, LM_TPB * SCAN_CHUNK, 1_500_007])
def test_reset_local_map_matches_cpu(n):
    """NeuralPoints.reset_local_map on CUDA tensors (pinb200_local_map_select / _gather) equals the same call on CPU
    tensors: local_mask, global2local (with the reference's fill value), the index list and every gathered array,
    with the temporal window off / by travel distance / by time stamp, mid time stamps, reboot, fp32 and fp64 sensors."""
    case = _local_case(n, seed=n)
    sensor = torch.tensor([7.123456789012, -3.3, 1.1], dtype=torch.float64)
    for k, opts in enumerate(LOCAL_OPTS):
        if k == 0:
            (a, b), _ = _launched(lambda: _reset_both(case, opts, sensor, 82.0), "local_keep_kernel",
                                  "local_scan_kernel", "local_gather_kernel", *(("local_recent_kernel",) if n else ()))
        else:
            a, b = _reset_both(case, opts, sensor, 82.0)
        _compare_local(a, b, (n, opts))
    if n == 1_500_007:
        _, names = kernels_run(lambda: _reset_both(case, LOCAL_OPTS[1], sensor, 82.0))
        _check_launched(names, "test_reset_local_map_matches_cpu")


@gpu
@pytest.mark.parametrize("n_recent", [99, 100])
@pytest.mark.parametrize("use_td", [True, False])
def test_reset_local_map_fewer_than_100_recent(n_recent, use_td):
    """Exactly 99 recent points keep the whole map (the reference's "fewer than 100" rule), exactly 100 do not."""
    case = _local_case(3000, seed=n_recent, n_recent=n_recent)
    a, b = _reset_both(case, (True, use_td, False, False, torch.float64), torch.zeros(3, dtype=torch.float64), 500.0)
    _compare_local(a, b, n_recent)
    assert a.local_count() == (3000 if n_recent == 99 else 100)


@gpu
@pytest.mark.parametrize("sdt", [torch.float32, torch.float64])
@pytest.mark.parametrize("n_local", [0, 1, 2])
def test_reset_local_map_tiny_local_maps(n_local, sdt):
    """0, 1 and 2 local points: where the global2local miss value switches between -1 and the reference's 1."""
    case = _local_case(600, seed=5, near=True)
    radius = [0.5, 1.5, 2.5][n_local]
    a, b = _reset_both(case, (False, True, False, False, sdt), torch.zeros(3, dtype=torch.float64), radius)
    _compare_local(a, b, n_local)
    assert a.local_count() == n_local
    miss = a.global2local[2].item()
    assert miss == (1 if n_local == 2 else -1)


# --------------------------------------------------------------------------------------
# 1c. map growth
# --------------------------------------------------------------------------------------
def _slots(p, res, B):
    c = np.floor(p / np.float32(res)).astype(np.int64)  # fp32 true division, then floor
    return (c @ PRIMES) % B


def _grow_case(n, B, seed, res=0.4, m0=20000):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-40, 40, (m0, 3)).astype(np.float32)
    table = np.full(B, -1, np.int32)
    s0 = _slots(pts, res, B)
    table[s0] = np.arange(m0, dtype=np.int32)  # any owner per slot will do as input
    owners = table[table >= 0]
    k = n // 3
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    base = pts[owners[rng.integers(0, len(owners), n)]]
    off = u * (np.sqrt(3.0) * res * rng.uniform(0.9, 1.1, n))[:, None]  # owners near and far, around 3 res^2
    cand = np.concatenate([base[:k], (base[k:2 * k] + off[k:2 * k]), rng.uniform(-40, 40, (n - 2 * k, 3))]).astype(np.float32)
    cand = cand[rng.permutation(n)]
    tsu = rng.integers(0, 31, m0).astype(np.int32)
    travel = (np.arange(32) * 0.5).astype(np.float32)  # ages are multiples of 0.5: ties with diff_travel 2.0
    return pts, table, cand, tsu, travel


def _grow_expected(pts, table, cand, tsu, travel, res, cur_ts, grow_all, temporal, diff):
    """NeuralPoints.update's growth test; in every slot the LARGEST candidate index decides the new owner."""
    B = table.shape[0]
    slot = _slots(cand, res, B)
    owner = table[slot]
    if grow_all:
        grow = np.ones(len(cand), bool)
    else:
        o = np.maximum(owner, 0)
        d = pts[o] - cand
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        grow = (owner < 0) | (d2 > np.float32(3 * res**2))
        if temporal:
            age = travel[cur_ts] - travel[tsu[o]]
            grow |= (owner >= 0) & (age > np.float32(diff))
    m0 = pts.shape[0]
    ids = m0 + np.cumsum(grow) - 1
    last = np.full(B, -1, np.int64)
    np.maximum.at(last, slot, np.arange(len(cand)))
    hit = last >= 0
    t = table.copy()
    li = last[hit]
    t[hit] = np.where(grow[li], ids[li], owner[li]).astype(np.int32)
    return grow, t


@gpu
@pytest.mark.parametrize("n", [1, MG_TPB, MG_TPB + 1, MG_TPB * SCAN_CHUNK, MG_TPB * SCAN_CHUNK + 1, 1_000_003])
def test_map_grow_matches_sequential_rule(n):
    """ops.map_grow appends exactly the candidates that pass the growth test, in candidate order, writes nothing behind
    them, and leaves the hash table as the sequential rule does: in each slot the largest candidate index wins
    (buffer_size 1009: hundreds of candidates share a slot)."""
    from pin_slam_b200 import ops

    res, cur_ts, diff = 0.4, 31, 2.0
    first = True
    for grow_all, temporal, B in [(False, False, 1009), (False, True, 1009), (True, False, 1009),
                                  (False, True, 2_000_003)]:
        pts, table, cand, tsu, travel = _grow_case(n, B, seed=n + B)
        m0 = pts.shape[0]
        grow, table_exp = _grow_expected(pts, table, cand, tsu, travel, res, cur_ts, grow_all, temporal, diff)
        n_new = int(grow.sum())
        cap = m0 + n + 8

        def run():
            P = torch.full((cap, 3), SENT_F, device="cuda")
            P[:m0] = torch.from_numpy(pts).cuda()
            Q = torch.full((cap, 4), SENT_F, device="cuda")
            Q[:m0] = 0.5
            TC = torch.full((cap,), SENT_I, dtype=torch.int32, device="cuda")
            TU = TC.clone()
            TU[:m0] = torch.from_numpy(tsu).cuda()
            TC[:m0] = 3
            C = torch.full((cap,), SENT_F, device="cuda")
            C[:m0] = 0.25
            tab = torch.from_numpy(table).cuda()
            sc = torch.empty(int(_lib().pinb200_map_grow_scratch(n)), dtype=torch.int32, device="cuda")
            nn = torch.zeros(1, dtype=torch.int64, device="cuda")
            ops.map_grow(torch.from_numpy(cand).cuda(), tab, res, P, Q, TC, TU, C, m0,
                         None if grow_all else torch.from_numpy(travel).cuda(), cur_ts, grow_all, temporal, diff, sc, nn)
            return P, Q, TC, TU, C, tab, nn

        if first:
            (P, Q, TC, TU, C, tab, nn), names = kernels_run(run)
            _check_launched(names, "test_map_grow_matches_sequential_rule")
            first = False
        else:
            P, Q, TC, TU, C, tab, nn = run()
        what = (n, grow_all, temporal, B)
        assert int(nn.item()) == n_new, what
        assert np.array_equal(tab.cpu().numpy(), table_exp), what
        e = np.full((cap, 3), SENT_F, np.float32)
        e[:m0], e[m0:m0 + n_new] = pts, cand[grow]
        assert np.array_equal(P.cpu().numpy(), e), what
        eq = np.full((cap, 4), SENT_F, np.float32)
        eq[:m0], eq[m0:m0 + n_new] = 0.5, [1.0, 0.0, 0.0, 0.0]
        assert np.array_equal(Q.cpu().numpy(), eq), what
        for arr, old in ((TC, 3), (TU, tsu)):
            ei = np.full(cap, SENT_I, np.int32)
            ei[:m0], ei[m0:m0 + n_new] = old, cur_ts
            assert np.array_equal(arr.cpu().numpy(), ei), what
        ec = np.full(cap, SENT_F, np.float32)
        ec[:m0], ec[m0:m0 + n_new] = 0.25, 0.0
        assert np.array_equal(C.cpu().numpy(), ec), what


# --------------------------------------------------------------------------------------
# 2. probe index
# --------------------------------------------------------------------------------------
def _probe_case(B, seed, res=0.4):
    rng = np.random.default_rng(seed)
    n = 200_000 if B > 1_000_000 else 3000
    pts = rng.uniform(-30, 30, (n, 3)).astype(np.float32)
    slot = _slots(pts, res, B)
    table = np.full(B, -1, np.int32)
    sel = rng.permutation(n)[: int(0.8 * n)]
    table[slot[sel]] = sel.astype(np.int32)
    occupied = np.flatnonzero(table >= 0)
    stale = rng.choice(occupied, max(1, len(occupied) // 20), replace=False)
    table[stale] = rng.integers(0, n, len(stale))  # owners of another slot: unreachable through this one
    ts_c = rng.integers(0, 21, n).astype(np.int32)
    travel = (np.arange(21) * 0.7).astype(np.float32)
    local = rng.random(n) < 0.4
    li = np.flatnonzero(local)
    g2l = np.where(rng.random(n + 1) < 0.1, -1, 1).astype(np.int32)  # the reference's fill value 1, and -1
    g2l[li] = np.arange(len(li), dtype=np.int32)
    g2l[n] = -1
    return pts, slot, table, ts_c, travel, li, g2l


def _probe_expected(pts, slot, table, ts_c, travel, li, g2l, B, local, tf, cur_ts=15, diff=3.5):
    n = pts.shape[0]
    i = np.arange(n)
    ok = table[slot] == i
    ids = g2l[:n].astype(np.int64) if local else i.astype(np.int64)
    ok &= ids >= 0
    if tf:
        ok &= np.abs(travel[cur_ts] - travel[ts_c]) < np.float32(diff)
    if local:
        nb = pts[li]
        same = (nb[np.maximum(ids, 0)] == pts).all(axis=1)
        ids = np.where(same, ids, ids | REC_REMAP)
    s = slot[ok]
    n_words = (B + 31) // 32
    bits = np.zeros(n_words, np.uint32)
    np.bitwise_or.at(bits, s >> 5, (np.uint32(1) << (s & 31).astype(np.uint32)))
    pc = np.zeros(n_words, np.int64)
    np.add.at(pc, s >> 5, 1)
    prefix = (np.cumsum(pc) - pc).astype(np.uint32)
    order = np.argsort(s, kind="stable")
    gi = i[ok][order]
    rec = np.concatenate([pts[gi].view(np.int32), ids[ok][order].astype(np.int32)[:, None]], axis=1)
    return bits, prefix, rec, gi.astype(np.int32)


@gpu
@pytest.mark.parametrize("B", [97, 32, 33, 32767, 32768, 32769, 40009, 100_000_007])
def test_probe_index_layout(B):
    """MapHandle.ensure_records() builds the probe index documented in pinb200.h: occupancy bit of slot s set iff
    table[s] == i, slot(points[i]) == s and the view can return point i; per-word prefix of set bits; the records and
    global ids in rank (slot) order, with PINB200_REC_REMAP on local ids that name another point -- for local and
    global views, with and without the travel-distance filter."""
    from pin_slam_b200 import ops

    pts, slot, table, ts_c, travel, li, g2l = _probe_case(B, seed=B)
    n = pts.shape[0]
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d_pts, d_table, d_ts, d_td, d_g2l, d_nb = c(pts), c(table), c(ts_c), c(travel), c(g2l), c(pts[li])
    first = True
    for local in (False, True):
        for tf in (False, True):
            def build():
                mh = ops.MapHandle(slot_table=d_table, buffer_size=B, points=d_pts, ts_create=d_ts, travel_dist=d_td,
                                   global2local=d_g2l if local else None, nb_points=d_nb if local else d_pts,
                                   nb_orient=None, geo_feat=None, color_feat=None, certainty=None, ts_update=None,
                                   probe_dx=torch.zeros((1, 3), dtype=torch.int32, device="cuda"), resolution=0.4,
                                   max_valid_dist2=1.0, time_filter=tf, cur_ts=15, diff_travel_dist_local=3.5,
                                   after_pgo=False)
                return mh.ensure_records()._probe

            if first:
                (words, rec, gid, scratch), names = kernels_run(build)
                _check_launched(names, "test_probe_index_layout")
                first = False
            else:
                words, rec, gid, scratch = build()
            bits, prefix, rec_e, gid_e = _probe_expected(pts, slot, table, ts_c, travel, li, g2l, B, local, tf)
            w = words.cpu().numpy().view(np.uint32)
            what = (B, local, tf)
            assert np.array_equal(w[:, 0], bits), what
            assert np.array_equal(w[:, 1], prefix), what
            n_rec = len(gid_e)
            n_blocks = (w.shape[0] + PROBE_WPBLK - 1) // PROBE_WPBLK
            assert int(scratch[n_blocks].item()) == n_rec, what
            assert np.array_equal(rec[:n_rec].cpu().numpy().view(np.int32), rec_e), what
            assert np.array_equal(gid[:n_rec].cpu().numpy(), gid_e), what
            if local:
                assert (rec_e[:, 3] & REC_REMAP).any() and not (rec_e[:, 3] & REC_REMAP).all()
    assert n > 0


# --------------------------------------------------------------------------------------
# 3. K4 registration step
# --------------------------------------------------------------------------------------
GN_KW = dict(min_nn=3, min_grad_norm=0.25, max_grad_norm=2.0, max_sdf_std=0.05, gm_dist=0.2, gm_grad=0.1,
             lm_lambda=1e-4)


def _gn_inputs(n, seed, *, label=False, normals=False, std=True, cc=0, axis=False):
    rng = np.random.default_rng(seed)
    u = rng.normal(size=(n, 3))
    p = (u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(2, 80, n)[:, None]).astype(np.float32)
    if axis:  # axis-aligned gradients: exact norms, a diagonal N[3:,3:]
        g = np.zeros((n, 3), np.float32)
        g[np.arange(n), rng.integers(0, 3, n)] = rng.uniform(0.3, 1.8, n) * rng.choice([-1, 1], n)
    else:
        g = rng.normal(size=(n, 3))
        g = g / np.linalg.norm(g, axis=1, keepdims=True) * rng.uniform(0.05, 2.5, n)[:, None]
        nrm = np.linalg.norm(g, axis=1)  # keep random norms away from the bounds (fp32 vs fp64 norm)
        for b in (GN_KW["min_grad_norm"], GN_KW["max_grad_norm"]):
            g[np.abs(nrm - b) < 1e-4] *= 0.9
        g = g.astype(np.float32)
    inp = dict(xyz=p, sdf=rng.normal(0, 0.1, n).astype(np.float32), grad=g,
               nn_count=rng.integers(0, 8, n).astype(np.int32),
               sdf_std=rng.uniform(0, 0.1, n).astype(np.float32) if std else None,
               sdf_label=rng.normal(0, 0.05, n).astype(np.float32) if label else None,
               normals=None, color_obs=None, color_pred=None, color_grad=None)
    if normals:
        nv = rng.normal(size=(n, 3))
        inp["normals"] = (nv / np.linalg.norm(nv, axis=1, keepdims=True)).astype(np.float32)
    if cc:
        inp["color_obs"] = rng.uniform(0, 1, (n, cc)).astype(np.float32)
        inp["color_pred"] = rng.uniform(0, 1, (n, cc)).astype(np.float32)
        inp["color_grad"] = rng.normal(0, 0.5, (n, cc, 3)).astype(np.float32)
    if inp["sdf_std"] is not None:
        inp["sdf_std"][np.abs(inp["sdf_std"] - GN_KW["max_sdf_std"]) < 1e-6] = 0.0
    return inp


def _gn_sums64(inp, kw, color_mode, w_photo):
    """The 47 sums of pinb200_gn_step in fp64 (N [36], g [6], sum w, sum |r|, count, sum w r^2, sum |colour res|),
    plus the sum of |w J r| per entry of g (a bound for its rounding)."""
    d = lambda k: None if inp[k] is None else inp[k].astype(np.float64)  # noqa: E731
    p, g, sdf = d("xyz"), d("grad"), d("sdf")
    gn32 = np.sqrt((inp["grad"] * inp["grad"]).sum(1, dtype=np.float32))
    valid = (inp["nn_count"] >= kw["min_nn"]) & (gn32 < np.float32(kw["max_grad_norm"])) & \
            (gn32 > np.float32(kw["min_grad_norm"]))
    if inp["sdf_std"] is not None:
        valid &= inp["sdf_std"] < np.float32(kw["max_sdf_std"])
    p, g, sdf = p[valid], g[valid], sdf[valid]
    gn = np.linalg.norm(g, axis=1)
    r = sdf - (d("sdf_label")[valid] if inp["sdf_label"] is not None else 0.0)
    w = np.ones(len(r))
    if kw["gm_grad"]:
        w *= (kw["gm_grad"] / (kw["gm_grad"] + (gn - 1) ** 2)) ** 2
    if kw["gm_dist"]:
        w *= (kw["gm_dist"] / (kw["gm_dist"] + r * r)) ** 2
    if inp["normals"] is not None:
        w *= 0.5 + np.abs((d("normals")[valid] * g).sum(1) / gn)
    rc = np.zeros(len(r))
    if color_mode:
        k = np.array([0.299, 0.587, 0.114]) if inp["color_obs"].shape[1] == 3 else np.array([1.0])
        io, ip = d("color_obs")[valid] @ k, d("color_pred")[valid] @ k
        cg = np.einsum("ncj,c->nj", d("color_grad")[valid], k)
        rc = ip - io
        if color_mode == 1:
            w *= np.exp(-np.abs(io - ip))
    J = np.concatenate([np.cross(p, g), g], 1)
    N = np.einsum("n,na,nb->ab", w, J, J)
    gv = -(w * r) @ J
    gabs = np.abs(w * r) @ np.abs(J)
    if color_mode == 2:
        Jc = np.concatenate([np.cross(p, cg), cg], 1)
        wc = w_photo * w
        N += np.einsum("n,na,nb->ab", wc, Jc, Jc)
        gv += -(wc * rc) @ Jc
        gabs += np.abs(wc * rc) @ np.abs(Jc)
    s = np.zeros(47)
    s[:36], s[36:42] = N.reshape(-1), gv
    s[42], s[43], s[44], s[45], s[46] = w.sum(), np.abs(r).sum(), len(r), (w * r * r).sum(), np.abs(rc).sum()
    return s, gabs


def _gn_replay(sums, lm, T0):
    """gn_solve (gn.cu) in numpy from the kernel's own sums: fp32 rounding of N and g, LM damping, pivoted solve,
    expmap, T <- dT T."""
    f32 = lambda x: np.float64(np.float32(x))  # noqa: E731
    cnt = sums[44]
    dT = np.eye(4)
    res = np.zeros(32)
    res[16] = cnt
    if cnt >= 10:
        sc = cnt / (2.0 * sums[42])
        N = np.array([f32(v * sc) for v in sums[:36]]).reshape(6, 6)
        g = np.array([f32(v * sc) for v in sums[36:42]])
        A = N.copy()
        for i in range(6):
            A[i, i] = f32(N[i, i] + np.float64(np.float32(lm)) * N[i, i])
        t = g.copy()
        singular = False
        for c in range(6):
            piv = c
            for r in range(c + 1, 6):
                if abs(A[r, c]) > abs(A[piv, c]):
                    piv = r
            if A[piv, c] == 0.0:
                singular = True
                break
            if piv != c:
                A[[c, piv]] = A[[piv, c]]
                t[[c, piv]] = t[[piv, c]]
            for r in range(c + 1, 6):
                f = A[r, c] / A[c, c]
                A[r, c:] -= f * A[c, c:]
                t[r] -= f * t[c]
        if not singular:
            for c in range(5, -1, -1):
                s = t[c]
                for k in range(c + 1, 6):
                    s -= A[c, k] * t[k]
                t[c] = s / A[c, c]
            ang = np.sqrt(t[0] ** 2 + t[1] ** 2 + t[2] ** 2)
            ax = t[:3] / ang if ang > 0 else np.zeros(3)
            S = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
            dT[:3, :3] = np.eye(3) + S * np.sin(ang) + (S @ S) * (1 - np.cos(ang))
            dT[:3, 3] = t[3:]
        res[17] = sums[43] / cnt * 100.0
        res[18:21] = np.linalg.eigvalsh(N[3:, 3:])
        res[21] = sums[45] * sc / cnt
        res[22:28] = g
        res[28] = sums[46] / cnt
    res[:16] = dT.reshape(-1)
    return res, dT @ T0


def _gn_run(inp, kw, color_mode, w_photo, T0, sums=None, result=None):
    from pin_slam_b200 import ops

    c = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    T = torch.from_numpy(T0.copy()).cuda()
    cg = inp["color_grad"]
    res, sums = ops.gn_step(c(inp["xyz"]), c(inp["sdf"]), c(inp["grad"]), c(inp["sdf_std"]), c(inp["nn_count"]),
                            sdf_label=c(inp["sdf_label"]), normals=c(inp["normals"]), t_inout=T, sums=sums,
                            result=result, color_obs=c(inp["color_obs"]) if color_mode else None,
                            color_pred=c(inp["color_pred"]) if color_mode else None,
                            color_grad=c(None if cg is None else cg.reshape(len(cg), -1)) if color_mode == 2 else None,
                            color_mode=color_mode, w_photo=w_photo, **kw)
    torch.cuda.synchronize()
    return res, sums, T


def _gn_cases():
    thr = 2 * _sms() * 256  # gn_accumulate_kernel runs 2 x SMs blocks of 256 threads
    base = dict(label=False, normals=False, std=True, cc=0)
    opt = [(dict(label=True, normals=True, std=False), dict(gm_dist=0.0, gm_grad=0.0), 0, 0.0),
           (dict(cc=3), {}, 1, 0.0), (dict(cc=1), {}, 1, 0.0), (dict(cc=1, label=True), {}, 2, 0.3),
           (dict(cc=3, normals=True), dict(gm_dist=0.0), 2, 0.05)]
    cases = [(n, base, {}, 0, 0.0) for n in (thr - 1, thr, thr + 1, 1_000_003)]
    for inp_kw, kw, mode, wp in opt:
        cases += [(n, {**base, **inp_kw}, kw, mode, wp) for n in (4000, thr + 1)]
    cases.append((1_000_003, {**base, **opt[3][0]}, opt[3][1], opt[3][2], opt[3][3]))
    return cases


def _gn_check(inp, kw, mode, wp, seed):
    rng = np.random.default_rng(seed)
    a = rng.normal(size=3) * 0.05
    T0 = np.eye(4)
    T0[:3, :3] = np.linalg.qr(np.eye(3) + np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]))[0]
    T0[:3, 3] = rng.normal(size=3)
    res, sums, T = _gn_run(inp, kw, mode, wp, T0)
    s = sums.cpu().numpy()
    ref, gabs = _gn_sums64(inp, kw, mode, wp)
    assert s[44] == ref[44]  # valid count
    Nmax = np.abs(ref[:36]).max() if ref[44] else 1.0
    assert np.all(np.abs(s[:36] - ref[:36]) <= 1e-5 * Nmax), np.abs(s[:36] - ref[:36]).max() / Nmax
    assert np.all(np.abs(s[36:42] - ref[36:42]) <= 1e-5 * np.maximum(gabs, 1e-30)), (s[36:42], ref[36:42])
    for k in (42, 43, 45, 46):
        assert abs(s[k] - ref[k]) <= 1e-5 * abs(ref[k]) + 1e-30, (k, s[k], ref[k])
    r = res.cpu().numpy()
    rep, T_exp = _gn_replay(s, kw["lm_lambda"], T0)
    np.testing.assert_allclose(r[:18], rep[:18], rtol=0, atol=1e-12)
    np.testing.assert_allclose(r[21:29], rep[21:29], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(T.cpu().numpy(), T_exp, rtol=0, atol=1e-12)
    if s[44] >= 10:
        ev = np.sort(r[18:21])
        np.testing.assert_allclose(ev, rep[18:21], rtol=0, atol=1e-10 * np.abs(rep[18:21]).max())
    return s, res, sums


@gpu
def test_gn_step_vs_fp64():
    """pinb200_gn_step at KITTI ranges: the sums against fp64 sums to 1e-5 (counts exact), dT / T against a numpy
    replay of the documented solve from the kernel's own sums to 1e-12, the eigenvalues against eigvalsh; with and
    without sdf_label / normals / sdf_std / GM weights, colour modes 1 and 2 with 1 and 3 channels, below, at and
    above the grid-stride threshold, and n = 0 (gn_solve_kernel)."""
    names = set()
    for k, (n, inp_kw, kw, mode, wp) in enumerate(_gn_cases()):
        inp = _gn_inputs(n, seed=k, **inp_kw)
        if k == 0:
            _, names = kernels_run(lambda: _gn_check(inp, {**GN_KW, **kw}, mode, wp, k))
        else:
            _gn_check(inp, {**GN_KW, **kw}, mode, wp, k)
    # n = 0: identity, T unchanged
    empty = {k: (np.zeros((0, 3), np.float32) if k in ("xyz", "grad") else v[:0] if v is not None else None)
             for k, v in _gn_inputs(4, 0).items()}
    (res, _, T), n0 = kernels_run(lambda: _gn_run(empty, GN_KW, 0, 0.0, np.eye(4) * 2))
    names |= n0
    assert np.array_equal(res.cpu().numpy()[:16], np.eye(4).reshape(-1)) and not res.cpu().numpy()[16:].any()
    assert np.array_equal(T.cpu().numpy(), np.eye(4) * 2)
    _check_launched(names, "test_gn_step_vs_fp64")


@gpu
def test_gn_step_validity_boundaries_and_repeat():
    """Validity decided exactly at its bounds (gradient norm == min or max, nn_count == min_nn, sdf_std == max_std),
    9 and 10 valid points, a diagonal and a nearly isotropic N[3:,3:], and two calls on one sums buffer (the
    last-block ticket is reset: the second call solves again)."""
    kw = GN_KW
    n = 64
    inp = _gn_inputs(n, 11, axis=True)
    g, nn, std = inp["grad"], inp["nn_count"], inp["sdf_std"]
    nn[:] = kw["min_nn"] + 2
    std[:] = 0.01
    g[:8] = 0
    lo, hi = np.float32(kw["min_grad_norm"]), np.float32(kw["max_grad_norm"])
    g[0, 0], g[1, 1] = lo, -hi                                                   # |g| == min, == max: invalid
    g[2, 2], g[3, 0] = np.nextafter(lo, hi), np.nextafter(hi, np.float32(0))    # one ulp inside: valid
    g[4:8, 1] = 1.0
    nn[4], nn[5] = kw["min_nn"], kw["min_nn"] - 1
    std[6], std[7] = kw["max_sdf_std"], np.nextafter(np.float32(kw["max_sdf_std"]), np.float32(0))
    ref, _ = _gn_sums64(inp, kw, 0, 0.0)
    assert ref[44] == n - 4  # 0, 1, 5, 6 invalid
    s, _, _ = _gn_check(inp, kw, 0, 0.0, 1)
    for k_valid in (9, 10):
        sub = {k: (None if v is None else v.copy()) for k, v in _gn_inputs(40, k_valid, axis=True).items()}
        sub["nn_count"][:] = 0
        sub["nn_count"][:k_valid] = kw["min_nn"]
        sub["sdf_std"][:] = 0.0
        s, res, _ = _gn_check(sub, kw, 0, 0.0, k_valid)
        assert s[44] == k_valid
        assert (res.cpu().numpy()[:16] == np.eye(4).reshape(-1)).all() == (k_valid == 9)
    # nearly isotropic: random unit gradients; diagonal: axis-aligned (p1 == 0 branch)
    for axis in (False, True):
        iso = _gn_inputs(30000, 3, axis=axis, std=False)
        iso["nn_count"][:] = 10
        iso["grad"] /= np.linalg.norm(iso["grad"], axis=1, keepdims=True).astype(np.float32)
        s, res, sums = _gn_check(iso, dict(kw, gm_grad=0.0), 0, 0.0, 4)
        if axis:
            assert s[3 * 6 + 4] == s[3 * 6 + 5] == s[4 * 6 + 5] == 0.0
    # repeat on the same sums / result buffers: the second call must solve again
    inp2 = _gn_inputs(2 * 2 * _sms() * 256 + 7, 21)
    r1, sums, T1 = _gn_run(inp2, kw, 0, 0.0, np.eye(4))
    r1 = r1.cpu().numpy()
    result = torch.full((32,), float("nan"), dtype=torch.float64, device="cuda")
    r2, sums2, T2 = _gn_run(inp2, kw, 0, 0.0, np.eye(4), sums=sums, result=result)
    rep, T_exp = _gn_replay(sums2.cpu().numpy(), kw["lm_lambda"], np.eye(4))
    np.testing.assert_allclose(r2.cpu().numpy()[:16], rep[:16], rtol=0, atol=1e-12)
    np.testing.assert_allclose(r2.cpu().numpy()[:16], r1[:16], rtol=0, atol=1e-9)
    np.testing.assert_allclose(T2.cpu().numpy(), T_exp, rtol=0, atol=1e-12)


# --------------------------------------------------------------------------------------
# 4. loss heads
# --------------------------------------------------------------------------------------
def _mapping_ref(sdf, label, weight, n, ne, sigma, weighted, weight_e, eps, gscale):
    s = torch.from_numpy(sdf).double().requires_grad_(True)
    z = s[:n] / sigma
    t = torch.sigmoid(torch.from_numpy(label).double() / sigma)
    w = torch.from_numpy(weight).double().abs() if weighted else torch.ones(n, dtype=torch.float64)
    bce = (w * torch.nn.functional.binary_cross_entropy_with_logits(z, t, reduction="none")).mean()
    loss = bce
    eik = torch.zeros((), dtype=torch.float64)
    zero = np.zeros(ne, bool)
    if ne:
        e = s[n:].reshape(6, ne)
        gx, gy, gz = (e[0] - e[1]) / (2 * eps), (e[2] - e[3]) / (2 * eps), (e[4] - e[5]) / (2 * eps)
        zero = ((gx == 0) & (gy == 0) & (gz == 0)).detach().numpy()
        nrm = torch.sqrt(gx * gx + gy * gy + gz * gz + torch.from_numpy(zero).double())  # |g| = 0 rows: dl = 0
        nrm = torch.where(torch.from_numpy(zero), torch.zeros_like(nrm), nrm)
        eik = ((nrm - 1) ** 2).mean()
        loss = loss + weight_e * eik
    loss.backward()
    dl = s.grad.numpy() * gscale
    if ne:
        for a in range(6):
            dl[n + a * ne: n + (a + 1) * ne][zero] = 0.0
    return dl, float(bce), float(eik), zero


@gpu
def test_mapping_loss_vs_fp64_autograd():
    """pinb200_mapping_loss against fp64 autograd of the same loss: BCE with and without weights, with and without
    Eikonal rows, above the grid-stride threshold, saturated logits (|sdf/sigma|, |label/sigma| up to ~200) and
    Eikonal rows with a zero numerical gradient (dl = 0, no NaN)."""
    from pin_slam_b200 import ops

    thr = 4 * _sms() * 256
    rng = np.random.default_rng(0)
    sigma, eps, weight_e, gscale = 0.08, 0.02, 0.5, 1.7
    first = True
    for n, ne, weighted in [(4096, 0, True), (thr + 1, 0, False), (thr + 1, 700, True), (1_000_003, 50_000, False),
                            (3000, thr + 5, True)]:
        sdf = rng.normal(0, 0.3, n + 6 * ne).astype(np.float32)
        label = rng.normal(0, 0.3, n).astype(np.float32)
        sat = rng.random(n) < 0.05
        sdf[:n][sat] = rng.uniform(-16, 16, sat.sum())   # sdf / sigma up to 200
        label[sat[::-1]] = rng.uniform(-16, 16, sat.sum())
        if ne:
            e = sdf[n:].reshape(6, ne)
            e[1], e[3], e[5] = e[0] - 0.04 * rng.normal(size=ne), e[2] - 0.04 * rng.normal(size=ne), e[4] - 0.04
            zero = rng.random(ne) < 0.02
            e[1][zero], e[3][zero], e[5][zero] = e[0][zero], e[2][zero], e[4][zero]
        weight = rng.uniform(-1.5, 1.5, n).astype(np.float32)
        c = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
        dl = torch.empty(n + 6 * ne, device="cuda")
        losses = torch.zeros(2, device="cuda")
        call = lambda: ops.mapping_loss(c(sdf), c(label), c(weight), n, ne, sigma, weighted, weight_e, eps, dl, losses,  # noqa: E731
                                        grad_scale=gscale)
        if first:
            _, names = kernels_run(call)
            _check_launched(names, "test_mapping_loss_vs_fp64_autograd")
            first = False
        else:
            call()
        got = dl.cpu().numpy().astype(np.float64)
        ref, bce, eik, zero = _mapping_ref(sdf, label, weight, n, ne, sigma, weighted, weight_e, eps, gscale)
        assert np.isfinite(got).all() and np.isfinite(losses.cpu().numpy()).all()
        wmax = np.abs(weight).max() if weighted else 1.0
        bound = 2e-6 * gscale * wmax / (n * sigma) + 1e-5 * np.abs(ref[:n])
        assert (np.abs(got[:n] - ref[:n]) <= bound).all(), np.abs(got[:n] - ref[:n]).max()
        if ne:
            ge, re_ = got[n:].reshape(6, ne), ref[n:].reshape(6, ne)
            assert (ge[:, zero] == 0).all()
            assert (np.abs(ge - re_) <= 1e-5 * np.abs(re_).max() + 1e-5 * np.abs(re_)).all(), np.abs(ge - re_).max()
        l0, l1 = losses.cpu().numpy()
        assert abs(l0 - bce) <= 1e-5 * bce, (l0, bce)
        assert abs(l1 - (eik if ne else 0.0)) <= 1e-5 * eik + 1e-12, (l1, eik)


@gpu
def test_color_loss_vs_fp64_autograd():
    """pinb200_color_loss against fp64 autograd: 1 and 3 channels, weights on and off, exact ties (d = 0: zero
    gradient), no surface samples (everything zero), above the grid-stride threshold."""
    from pin_slam_b200 import ops

    thr = 4 * _sms() * 256
    rng = np.random.default_rng(1)
    surf, weight_i, gscale = 0.1, 0.7, 1.3
    first = True
    for n, cc, weighted, any_surface in [(5000, 1, True, True), (5000, 3, False, True), (thr // 3 + 1, 3, True, True),
                                         (thr + 1, 1, False, True), (700_001, 3, False, True), (4000, 3, True, False)]:
        pred = rng.uniform(0, 1, (n, cc)).astype(np.float32)
        lab = rng.uniform(0, 1, (n, cc)).astype(np.float32)
        tie = rng.random((n, cc)) < 0.1
        lab[tie] = pred[tie]
        sl = rng.uniform(-0.3, 0.3, n).astype(np.float32)
        if not any_surface:
            sl = (np.abs(sl) + surf).astype(np.float32)
        w = rng.uniform(-2, 2, n).astype(np.float32)
        in_s = np.abs(sl) < np.float32(surf)
        ns = torch.tensor([float(in_s.sum())], device="cuda")
        c = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
        dl = torch.empty(n, cc, device="cuda")
        loss = torch.zeros(1, device="cuda")
        call = lambda: (loss.zero_(), ops.color_loss(c(pred), c(lab), c(sl), c(w), surf, weighted, weight_i, ns, dl,  # noqa: E731
                                                     loss, grad_scale=gscale))
        if first:
            _, names = kernels_run(call)
            _check_launched(names, "test_color_loss_vs_fp64_autograd")
            first = False
        else:
            call()
        p64 = torch.from_numpy(pred).double().requires_grad_(True)
        ww = torch.from_numpy(np.abs(w) if weighted else np.ones(n, np.float32)).double()[:, None]
        m = torch.from_numpy(in_s).double()[:, None]
        cnt = max(float(in_s.sum()), 1.0) * cc
        L = (m * ww * (p64 - torch.from_numpy(lab).double()).abs()).sum() / cnt
        (weight_i * gscale * L).backward()
        ref = p64.grad.numpy()
        got = dl.cpu().numpy()
        assert np.array_equal(got[tie & in_s[:, None]], np.zeros((tie & in_s[:, None]).sum(), np.float32))
        assert np.allclose(got, ref, rtol=2e-6, atol=1e-6 * np.abs(ref).max() + 1e-30)
        assert abs(float(loss.item()) - float(L)) <= 1e-5 * float(L) + 1e-12
        if not any_surface:
            assert not got.any() and float(loss.item()) == 0.0


# --------------------------------------------------------------------------------------
# 6. crafted distance-test boundaries
# --------------------------------------------------------------------------------------
N_CRAFTED = 300


@gpu
def test_pool_filter_distance_boundary_matches_torch():
    """Samples whose squared distance to the fp64 origin rounds to the other side of the window radius than its exact
    value: pinb200_pool_filter keeps exactly the samples torch's ((p - o)**2).sum(-1) < r2 keeps."""
    rng = np.random.default_rng(7)
    flips = []
    first = True
    for k, (p, o, r2) in enumerate(_craft(rng, np.float64, N_CRAFTED, 50.0, less=True)):
        others = _embed(rng, o, 50.0)
        at = rng.integers(0, len(others) + 1)
        g = np.insert(others, at, p, axis=0)
        n = len(g)
        src = {"coord": torch.zeros(n, 3, device="cuda"), "gcoord": torch.from_numpy(g).cuda(),
               "label": torch.arange(n, dtype=torch.float32, device="cuda"), "weight": torch.zeros(n, device="cuda"),
               "ts": torch.arange(n, dtype=torch.int32, device="cuda"), "color": torch.zeros(n, 3, device="cuda")}
        og = torch.from_numpy(o).cuda()
        if first:
            (out, _, counts), _ = _launched(lambda: _pool_filter(src, 0, 1, og, float(r2)), "pool_count_kernel",
                                            "pool_scatter_kernel")
            first = False
        else:
            out, _, counts = _pool_filter(src, 0, 1, og, float(r2))
        keep = ((torch.from_numpy(g) - torch.from_numpy(o)) ** 2).sum(-1) < float(r2)
        kept = int(counts[0].item())
        got = np.zeros(n, bool)
        got[out["ts"][:kept].cpu().numpy()] = True
        if not np.array_equal(got, keep.numpy()):
            flips.append(k)
    assert not flips, f"{len(flips)} of {N_CRAFTED} crafted samples decided unlike torch"


def _local_select(pts, sensor, r2):
    from pin_slam_b200 import ops

    n = pts.shape[0]
    mask = torch.empty(n + 1, dtype=torch.bool, device="cuda")
    sc = torch.empty(n // LM_TPB + 4, dtype=torch.int32, device="cuda")
    counts = torch.zeros(2, dtype=torch.int64, device="cuda")
    ops.local_map_select(pts, None, None, None, 0, False, False, False, 50, False, 0, 0.0, sensor, r2, mask, sc, counts)
    return mask


@gpu
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_local_map_radius_boundary_matches_torch(dt):
    """Neural points whose squared distance to the sensor rounds to the other side of local_map_radius^2 than its exact
    value: pinb200_local_map_select decides them as torch's ((p - s)**2).sum(-1) < r2 does, for fp64 and fp32 sensor
    positions."""
    rng = np.random.default_rng(8 if dt is np.float64 else 9)
    flips = []
    for k, (p, o, r2) in enumerate(_craft(rng, dt, N_CRAFTED, 82.0, less=True)):
        others = _embed(rng, o, 82.0)
        at = rng.integers(0, len(others) + 1)
        g = np.insert(others, at, p, axis=0)
        sensor = torch.from_numpy(o)
        if k == 0:
            mask, _ = _launched(lambda: _local_select(torch.from_numpy(g).cuda(), sensor.cuda(), float(r2)),
                                "local_keep_kernel", "local_scan_kernel")
        else:
            mask = _local_select(torch.from_numpy(g).cuda(), sensor.cuda(), float(r2))
        if dt is np.float32:  # the kernel compares with (float)r2; r2 is an fp32 value
            ref = ((torch.from_numpy(g) - sensor) ** 2).sum(-1) < torch.tensor(r2)
        else:
            ref = ((torch.from_numpy(g) - sensor) ** 2).sum(-1) < float(r2)
        if not torch.equal(mask[:-1].cpu(), ref):
            flips.append(k)
    assert not flips, f"{len(flips)} of {N_CRAFTED} crafted points decided unlike torch"


@gpu
def test_map_grow_far_boundary_matches_torch():
    """Candidates whose squared distance to the slot owner rounds to the other side of far2 (3 res^2) than its exact
    value: pinb200_map_grow grows exactly the candidates torch's ((owner - cand)**2).sum(-1) > far2 grows.  With
    buffer_size 1 every candidate shares the slot of owner 0."""
    rng = np.random.default_rng(10)
    lib = _lib()
    flips = []
    for k, (p, o, far2) in enumerate(_craft(rng, np.float32, N_CRAFTED, 0.69, less=False)):
        others = _embed(rng, o, 0.69)
        at = rng.integers(0, len(others) + 1)
        cand = np.insert(others, at, p, axis=0)
        n = len(cand)

        def run():
            pts = torch.zeros(n + 1, 3, device="cuda")
            pts[0] = torch.from_numpy(o).cuda()
            ori = torch.zeros(n + 1, 4, device="cuda")
            tsc = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
            tsu, cert = tsc.clone(), torch.zeros(n + 1, device="cuda")
            table = torch.zeros(1, dtype=torch.int32, device="cuda")
            sc = torch.empty(int(lib.pinb200_map_grow_scratch(n)), dtype=torch.int32, device="cuda")
            nn = torch.zeros(1, dtype=torch.int64, device="cuda")
            cd = torch.from_numpy(cand).cuda()
            rc = lib.pinb200_map_grow(cd.data_ptr(), n, table.data_ptr(), 1, 0.4, pts.data_ptr(), ori.data_ptr(),
                                      tsc.data_ptr(), tsu.data_ptr(), cert.data_ptr(), 1, n + 1, None, 0, 0, 0, 0.0,
                                      float(far2), sc.data_ptr(), nn.data_ptr(), _stream())
            assert rc == 0
            return pts, nn

        if k == 0:
            (pts, nn), _ = _launched(run, "grow_flag_kernel", "grow_append_kernel")
        else:
            pts, nn = run()
        grow = ((torch.from_numpy(o) - torch.from_numpy(cand)) ** 2).sum(-1) > torch.tensor(far2)
        m = int(nn.item())
        if m != int(grow.sum()) or not torch.equal(pts[1:1 + m].cpu(), torch.from_numpy(cand)[grow]):
            flips.append(k)
    assert not flips, f"{len(flips)} of {N_CRAFTED} crafted candidates decided unlike torch"


# --------------------------------------------------------------------------------------
# 7. ledger (no GPU)
# --------------------------------------------------------------------------------------
def test_kernel_ledger():
    """No GPU: every __global__ kernel defined in pin_slam_b200/csrc is named in KERNEL_LEDGER by a test that exists
    (the query and training families by test_query_paths.py::test_coverage_ledger), and the ledger names no kernel
    that is gone.  A new kernel without a test fails here."""
    found = global_kernels()
    assert len(found) >= 30, sorted(found)
    assert found == set(KERNEL_LEDGER), (sorted(found - set(KERNEL_LEDGER)), sorted(set(KERNEL_LEDGER) - found))
    here = os.path.dirname(os.path.abspath(__file__))
    for kernel, ref in KERNEL_LEDGER.items():
        mod, test = ref.split("::")
        with open(os.path.join(here, mod + ".py")) as f:
            assert re.search(rf"^def {test}\(", f.read(), re.M), (kernel, ref)


def test_kernel_ledger_parser():
    """No GPU: the parser finds kernels behind __launch_bounds__ arguments with parentheses and templates, and skips
    declarations."""
    import tempfile

    src = ("template <int A>\n__global__ void __launch_bounds__(TILE, f<A>(2 * (1 + A))) alpha_kernel(int x) {}\n"
           "__global__ void beta_kernel(const float* p);\n__global__ void\ngamma_kernel(int (*f)(int)) { }\n")
    global CSRC
    old = CSRC
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "x.cu"), "w") as f:
            f.write(src)
        CSRC = d
        try:
            assert global_kernels() == {"alpha_kernel", "gamma_kernel"}
        finally:
            CSRC = old
