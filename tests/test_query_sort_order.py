"""The order the split pipeline's search launch actually used when the spatial sort is on (query_sort.cu).

The compact stash block of search tile t records, per lane, the original index of the query that lane searched
(StashS::perm: int32 at 640 t + 608 + lane of the workspace).  Read back, the first n entries must be a permutation of
0..n-1 along which the bucket keys -- the Morton code of the query's cell at 2 map resolutions, b bits per axis,
wrapped, recomputed here with the kernel's fp32 arithmetic -- never decrease.  The histogram width b is the largest
of 7..4 whose arrays fit in the workspace tail behind the stash blocks and seeds; without room for b = 4 the batch runs
unsorted (identity order).  The sizes below take every width and the unsorted case, and every output must be
bit-identical to the same call with the sort off."""
import numpy as np
import pytest
import torch

from oracle import pin_oracle as po
from tests.helpers import decoder_handle_from_oracle, map_handle_from_oracle, queries_near, synthetic_map

WT = 32
STASH_S, STASH_S_PERM = 640, 608  # floats of a compact stash block, offset of its original-index column
STASH, SEEDS = 1536, 1056  # floats per tile of a full stash block and of the forward-mode seeds
SORT_CTAS_PER_SM = 2  # sort_key_kernel: 1024-thread CTAs, all co-resident (__launch_bounds__(1024, 2))
OUT_KEYS = ("sdf", "grad", "sdf_std", "nn_count", "certainty", "knn_idx", "knn_gidx", "knn_dist2", "knn_weight", "xyz")


def _align(b):
    return (b + 255) // 256 * 256


def expected_bits(ws_ptr, ws_bytes, n, sms):
    """The histogram width the room rule of sort_queries picks for a call with d/dq (seeds stored), or None."""
    tiles = -(-n // WT)
    used = tiles * (STASH_S + SEEDS) * 4
    pad = _align(ws_ptr + used) - (ws_ptr + used)
    for b in (7, 6, 5, 4):
        need = pad + _align(16 * n) + 2 * _align(4 * n) + _align(4 << (3 * b)) + _align(4 * SORT_CTAS_PER_SM * sms)
        if need <= ws_bytes - used:
            return b
    return None


def _spread3(v):
    k = np.zeros_like(v)
    for i in range(10):
        k |= ((v >> i) & 1) << (3 * i)
    return k


def bucket_keys(xyz, resolution, bits):
    """sort_key_kernel's bucket of every point: float32 x * float32(1 / (2 res)), floor, masked, interleaved."""
    inv = np.float32(1.0) / (np.float32(2.0) * np.float32(resolution))
    c = np.floor(xyz.astype(np.float32) * inv).astype(np.int64) & ((1 << bits) - 1)
    return _spread3(c[:, 0]) | (_spread3(c[:, 1]) << 1) | (_spread3(c[:, 2]) << 2)


def cell_of_bucket(key, bits):
    c = np.zeros((key.shape[0], 3), dtype=np.int64)
    for i in range(bits):
        for a in range(3):
            c[:, a] |= ((key >> (3 * i + a)) & 1) << i
    return c


def search_order(o, n):
    ws = o["_workspace"].view(torch.int32)
    tiles = -(-n // WT)
    idx = ws[: tiles * STASH_S].view(tiles, STASH_S)[:, STASH_S_PERM:].reshape(-1).cpu().numpy()
    assert (idx[n:] == -1).all()
    return idx[:n]


def test_expected_bits_rule():
    """No GPU: the room rule gives the widths the cases below rely on (132 SMs, a 512-byte aligned workspace)."""
    from pin_slam_b200 import _lib

    lib = _lib.load()
    ws = lambda n: int(lib.pinb200_query_workspace_bytes(n))  # noqa: E731
    got = {n: expected_bits(0, ws(n), n, 132) for n in (200000, 120001, 50003, 5000, 600)}
    assert got == {200000: 7, 120001: 7, 50003: 6, 5000: 5, 600: 4}, got
    assert expected_bits(0, ws(_just_unsorted(132)), _just_unsorted(132), 132) is None
    assert expected_bits(0, ws(_just_unsorted(132) + 1), _just_unsorted(132) + 1, 132) == 4


def _just_unsorted(sms):
    """The largest batch below the first one with room for 4 bits (a 512-byte aligned workspace)."""
    from pin_slam_b200 import _lib

    lib = _lib.load()
    n = 1
    while expected_bits(0, int(lib.pinb200_query_workspace_bytes(n)), n, sms) is None:
        n += 1
    return n - 1


@pytest.fixture(scope="module")
def scene():
    m = synthetic_map(n_surface=60000, seed=11, resolution=0.4, buffer_size=200003, feature_dim=32,
                      local_radius=14.0, diff_td=3.0)
    return m, map_handle_from_oracle(m, True), decoder_handle_from_oracle(po.make_decoder(35, 64, 2, 1, 0.044, seed=3))


def _query(scene, q, sort, transform=None):
    from pin_slam_b200 import ops

    _, mh, dh = scene
    ops.set_option("split_min_queries", 1)
    ops.set_option("sort_min_queries", 1 if sort else 0)
    try:
        o = ops.query_sdf(mh, dh, q, nn_k=8, weighted_first=True, need_grad=True, transform=transform, save_knn=True,
                          want_xyz=True, out={})
        torch.cuda.synchronize()
    finally:
        ops.set_option("split_min_queries", 0)
        ops.set_option("sort_min_queries", ops.SORT_MIN_QUERIES)
    return o


def _case_queries(m, kind, n, g):
    """Seeded query batches of the cases."""
    res = 2 * 0.4
    if kind == "one_bucket":  # every query in the same 0.8 m cell: one histogram counter takes all the ranks
        c = (np.floor(m.neural_points[123].numpy() / res) + 0.5) * res
        return torch.from_numpy(c + (torch.rand(n, 3, generator=g).numpy() - 0.5) * 0.7 * res).float()
    q = queries_near(m, n, seed=int(torch.randint(0, 1 << 30, (1,), generator=g)))
    if kind == "far":  # negative coordinates and coordinates past the 7-bit wrap (128 cells = 102.4 m)
        k = n // 8
        q[:k] += torch.tensor([-230.0, 140.0, -75.0])
        q[k:2 * k] += torch.tensor([310.0, -405.0, 120.0])
    if kind == "slices":  # buckets on both sides of the boundaries between the CTA slices of the 7-bit histogram
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        grid = SORT_CTAS_PER_SM * sms
        s = 2
        while (1 << 21) >> s > grid:
            s += 1
        bounds = np.arange(1, (1 << 21) >> s) << s
        keys = (bounds[:, None] + np.array([-2, -1, 0, 1])[None, :]).reshape(-1)
        cells = cell_of_bucket(keys, 7)
        k = min(n // 2, cells.shape[0] * 8)
        pick = torch.randint(0, cells.shape[0], (k,), generator=g).numpy()
        q[:k] = torch.from_numpy((cells[pick] + 0.1 + 0.8 * torch.rand(k, 3, generator=g).numpy()) * res).float()
    return q.contiguous()


CASES = [  # name, n, kind, expected width on 132 SMs (None: unsorted)
    ("bench_size", 200000, "near", 7),
    ("b7_far", 120001, "far", 7),
    ("b7_slices", 100003, "slices", 7),
    ("b6", 50003, "near", 6),
    ("b6_one_bucket", 40000, "one_bucket", 6),
    ("b5", 5000, "far", 5),
    ("b4", 600, "near", 4),
    ("b4_ragged", 617, "far", 4),
    ("just_unsorted", None, "near", None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,kind,bits", CASES, ids=[c[0] for c in CASES])
def test_sorted_search_order(scene, name, n, kind, bits):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if n is None:
        n = _just_unsorted(sms)
    m = scene[0]
    g = torch.Generator().manual_seed(n)
    q = _case_queries(m, kind, n, g).cuda()
    on = _query(scene, q, True)
    ws = on["_workspace"]
    assert ws.data_ptr() % 256 == 0
    b = expected_bits(ws.data_ptr(), ws.numel(), n, sms)
    if sms == 132:
        assert b == bits, (name, b)
    order = search_order(on, n)
    if b is None:
        assert np.array_equal(order, np.arange(n))
    else:
        assert np.array_equal(np.sort(order), np.arange(n)), "the search order is not a permutation of the batch"
        xyz = q.cpu().numpy()[order]
        assert (np.diff(bucket_keys(xyz, m.resolution, b)) >= 0).all(), f"bucket keys decrease at {b} bits"
        if kind == "slices":
            s = 2
            while (1 << 21) >> s > SORT_CTAS_PER_SM * sms:
                s += 1
            assert len(np.unique(bucket_keys(xyz, m.resolution, 7) >> s)) > 100
        if kind == "one_bucket":
            assert len(np.unique(bucket_keys(xyz, m.resolution, b))) == 1
    off = _query(scene, q, False)
    assert np.array_equal(search_order(off, n), np.arange(n))
    if kind == "near":
        assert int((off["nn_count"] > 0).sum()) > 0.9 * n
    for k in OUT_KEYS:
        assert torch.equal(on[k], off[k]), f"{k} differs with the sort on: {int((on[k] != off[k]).sum())} elements"


@pytest.mark.gpu
def test_sorted_search_order_with_transform(scene):
    """The key is the transformed point (what the search reports as xyz); the search reads the untransformed query
    from the sorted record and transforms it itself."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m = scene[0]
    T = torch.eye(4, dtype=torch.float64)
    T[:3, :3] = po.expmap(torch.tensor([0.3, -0.2, 0.5], dtype=torch.float64))
    T[:3, 3] = torch.tensor([1.5, -0.7, 0.2], dtype=torch.float64)
    n = 30001
    q = po.transform_points(queries_near(m, n, seed=8), torch.linalg.inv(T)).float().cuda()
    Td = T.cuda()
    on = _query(scene, q, True, Td)
    ws = on["_workspace"]
    b = expected_bits(ws.data_ptr(), ws.numel(), n, sms)
    assert b is not None
    order = search_order(on, n)
    assert np.array_equal(np.sort(order), np.arange(n))
    xyz_t = on["xyz"].cpu().numpy()[order]
    assert (np.diff(bucket_keys(xyz_t, m.resolution, b)) >= 0).all()
    assert not (np.diff(bucket_keys(q.cpu().numpy()[order], m.resolution, b)) >= 0).all()
    off = _query(scene, q, False, Td)
    assert int((off["nn_count"] > 0).sum()) > 0.9 * n
    for k in OUT_KEYS:
        assert torch.equal(on[k], off[k]), f"{k} differs with the sort on: {int((on[k] != off[k]).sum())} elements"
