"""Spatial sort of the split pipeline (pinb200_set_option("sort_min_queries", n)): large inference batches are searched
in Morton order of their cells (2x the map resolution) and the results go back to each query's own index.  Each query's search and each tile
row's decode do not depend on which other queries share the tile, so every output must be bit-identical with the
sort on and off."""
import numpy as np
import pytest
import torch

from oracle import pin_oracle as po
from tests.helpers import decoder_handle_from_oracle, map_handle_from_oracle, queries_near, synthetic_map

OUT_KEYS = ("sdf", "grad", "sdf_std", "nn_count", "certainty", "knn_idx", "knn_gidx", "knn_dist2", "knn_weight", "xyz",
            "color", "color_grad")


def test_sort_option_is_validated():
    """Host-side state only (no GPU): 0 switches the sort off, negative thresholds are refused."""
    from pin_slam_b200 import ops

    ops.set_option("sort_min_queries", 0)
    ops.set_option("sort_min_queries", 1)
    with pytest.raises(RuntimeError):
        ops.set_option("sort_min_queries", -1)
    ops.set_option("sort_min_queries_color", 0)
    with pytest.raises(RuntimeError):
        ops.set_option("sort_min_queries_color", -1)
    ops.set_option("sort_min_queries", ops.SORT_MIN_QUERIES)


def _run(fn, sort):
    """fn() with the split pipeline forced on and the sort on (threshold 1) or off; returns the output tensors."""
    from pin_slam_b200 import ops

    ops.set_option("split_min_queries", 1)
    ops.set_option("sort_min_queries", 1 if sort else 0)
    ops.set_option("sort_min_queries_color", 1 if sort else 0)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        ops.set_option("split_min_queries", 0)
        ops.set_option("sort_min_queries", ops.SORT_MIN_QUERIES)
        ops.set_option("sort_min_queries_color", 0)
    return {k: v.clone() for k, v in out.items() if k in OUT_KEYS}


def _assert_equal(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert torch.equal(a[k], b[k]), f"{k} differs with the sort on: {int((a[k] != b[k]).sum())} elements"


@pytest.mark.gpu
@pytest.mark.parametrize("F,K,L,pgo,color", [(32, 8, 2, False, False), (8, 6, 1, False, True), (16, 4, 2, True, False),
                                             (32, 8, 1, True, True)])
@pytest.mark.parametrize("need_grad", [True, False])
def test_sorted_split_pipeline_is_bit_identical(F, K, L, pgo, color, need_grad):
    """Value, d/dq, colour head + Jacobian, after_pgo, kNN outputs, a ragged last tile (20011 queries) and queries
    without neighbours; with d/dq (32-query tiles) and value-only (128-query tiles)."""
    from pin_slam_b200 import ops

    m = synthetic_map(n_surface=60000, seed=F + K, resolution=0.4, buffer_size=200003, feature_dim=F, color=color,
                      after_pgo=pgo, local_radius=14.0, diff_td=3.0)
    dh = decoder_handle_from_oracle(po.make_decoder(F + 3, 64, L, 1, 0.044, seed=3))
    ch = decoder_handle_from_oracle(po.make_decoder(F + 3, 64, L, 3, 1.0, seed=4), sigmoid_out=True) if color else None
    mh = map_handle_from_oracle(m, True)
    q = queries_near(m, 20011, seed=5)
    q[100:116] = torch.tensor([300.0, -200.0, 50.0])  # no neighbours at all
    q = q.cuda()
    fn = lambda: ops.query_sdf(mh, dh, q, nn_k=K, weighted_first=True, need_grad=need_grad, color_dec=ch,  # noqa: E731
                               color_grad=color and need_grad, save_knn=True)
    off, on = _run(fn, False), _run(fn, True)
    assert int((off["nn_count"] == 0).sum()) >= 16
    _assert_equal(off, on)


@pytest.mark.gpu
def test_sorted_split_pipeline_with_transform():
    """opts.transform: the key is taken from the transformed query, the search transforms it again; xyz and every
    other output are unchanged by the sort."""
    from pin_slam_b200 import ops

    m = synthetic_map(n_surface=60000, seed=7, resolution=0.4, buffer_size=200003, feature_dim=32, local_radius=14.0,
                      diff_td=3.0)
    dh = decoder_handle_from_oracle(po.make_decoder(35, 64, 2, 1, 0.044, seed=3))
    mh = map_handle_from_oracle(m, True)
    T = torch.eye(4, dtype=torch.float64)
    T[:3, :3] = po.expmap(torch.tensor([0.01, -0.02, 0.03], dtype=torch.float64))
    T[:3, 3] = torch.tensor([0.1, -0.05, 0.02], dtype=torch.float64)
    q = po.transform_points(queries_near(m, 9001, seed=8), torch.linalg.inv(T)).float().cuda()
    Td = T.cuda()
    fn = lambda: ops.query_sdf(mh, dh, q, nn_k=8, weighted_first=True, need_grad=True, transform=Td,  # noqa: E731
                               want_xyz=True, save_knn=True)
    off, on = _run(fn, False), _run(fn, True)
    assert int((off["nn_count"] > 0).sum()) > 8000
    _assert_equal(off, on)


@pytest.mark.gpu
def test_sort_runs_and_host_query_with_chunks_is_bit_identical():
    """The sort really launches on a large batch (sort_key_kernel in the profile), and NeuralPoints.query_sdf_host
    (pieces pipelined over two streams, each piece sorted on its own) returns the same as with the sort off."""
    from torch.profiler import ProfilerActivity, profile

    from pin_slam_b200.config import HotPathConfig
    from pin_slam_b200.model import Decoder
    from pin_slam_b200.synthetic import build_map, surface_queries

    cfg = HotPathConfig.cfg2(device="cuda")
    npm = build_map(cfg, n_surface=200000, seed=0, extent=40.0)
    torch.manual_seed(0)
    dec = Decoder(cfg, 64, 2, 1)
    q = surface_queries(npm, 50001, seed=3, sigma=0.1)
    with profile(activities=[ProfilerActivity.CUDA]) as tp:
        _run(lambda: npm.query_sdf(q, dec, need_grad=True), True)
    names = [e.key for e in tp.key_averages()]
    assert any("sort_key_kernel" in k for k in names) and any("search_kernel<true, true>" in k for k in names), names

    q_host = q.cpu().pin_memory()
    res = {}
    for sort in (False, True):
        host = {"sdf": torch.empty(q.shape[0]).pin_memory(), "grad": torch.empty(q.shape[0], 3).pin_memory(),
                "sdf_std": torch.empty(q.shape[0]).pin_memory(),
                "nn_count": torch.empty(q.shape[0], dtype=torch.int32).pin_memory(),
                "certainty": torch.empty(q.shape[0]).pin_memory()}

        def fn():
            npm.query_sdf_host(q_host, dec, host, chunks=3)
            torch.cuda.current_stream().synchronize()
            return host

        res[sort] = _run(fn, sort)
    _assert_equal(res[False], res[True])
    assert np.isfinite(res[True]["sdf"].numpy()).all()
