"""The adjoint schedule of wsq_decode_kernel<F, true, false> against the oracle.

With d/dq and a single output channel the warp-specialised decode gathers 64-query groups (value rows, then the three
tangent blocks dx/dq_j) and gets d out / d q_j as v' . (W0 dx/dq_j) with one adjoint vector v' per query, instead of
pushing the tangent rows through every layer.  The cases cover every feature width and depth the kernel takes, leaky
and plain ReLU, decoders with and without biases, a sigmoid output, the spatial sort, and batch sizes that leave the
last group of 64 queries partial (or its second 32-query block empty)."""
from collections import namedtuple
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import pin_oracle as po
from tests.helpers import (assert_rel_close, assert_sdf_close, decoder_handle_from_oracle, kernels_run,
                           map_handle_from_oracle, oracle64, queries_near, synthetic_map)

Case = namedtuple("Case", "F L K leaky bias sigmoid sort n")
CASES = [
    Case(8, 1, 6, False, True, False, False, 1024 + 1),
    Case(8, 2, 6, True, False, False, True, 1024 + 31),
    Case(16, 1, 5, True, True, False, False, 1024 + 32),
    Case(16, 2, 4, False, True, False, True, 1024 + 33),
    Case(16, 1, 5, True, False, True, True, 1024 + 63),
    Case(32, 1, 8, False, False, False, True, 1024 + 63),
    Case(32, 2, 8, True, True, False, False, 1024 + 31),
    Case(32, 2, 8, False, False, False, False, 1024 + 1),
    Case(32, 2, 8, False, True, True, False, 1024 + 33),
    Case(32, 2, 8, True, False, False, True, 1024 + 32),
    Case(32, 2, 8, False, True, False, True, 200000),
    Case(8, 2, 6, True, True, True, False, 200000),
]


def case_id(c):
    return (f"F{c.F}-L{c.L}-K{c.K}" + ("-leaky" if c.leaky else "") + ("" if c.bias else "-nobias")
            + ("-sigmoid" if c.sigmoid else "") + ("-sorted" if c.sort else "") + f"-n{c.n}")


@lru_cache(maxsize=None)
def _map(F):
    return synthetic_map(n_surface=60000, seed=F + 1, resolution=0.4, buffer_size=200003, feature_dim=F,
                         local_radius=14.0, diff_td=3.0)


def _sigmoid_ref(r):
    """sdf = sigmoid(o), d sdf / dq = sdf (1 - sdf) do/dq from an oracle run of the head with sdf_scale 1."""
    s = 1.0 / (1.0 + np.exp(-np.asarray(r["sdf"], np.float64)))
    return {"sdf": s, "grad": (s * (1.0 - s))[:, None] * np.asarray(r["grad"], np.float64)}


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[case_id(c) for c in CASES])
def test_adjoint_decode_vs_oracle(c):
    from pin_slam_b200 import ops

    m = _map(c.F)
    dec = po.make_decoder(c.F + 3, 64, c.L, 1, 1.0 if c.sigmoid else 0.044, seed=7, bias=c.bias)
    dec.leaky = c.leaky
    q = queries_near(m, c.n, seed=8)
    q[:5] = torch.tensor([300.0, -200.0, 50.0])  # no neighbours at all
    ref = po.query_sdf(m, dec, q, c.K, True, need_grad=True)
    r64 = oracle64(m, dec, q, c.K, True, ref, need_grad=True)
    ref_sdf, ref_grad, g64 = ref["sdf"].numpy(), ref["grad"].numpy(), r64["grad"]
    scale = dec.sdf_scale
    if c.sigmoid:
        ref_sdf, ref_grad = (v for v in _sigmoid_ref(ref).values())
        g64 = _sigmoid_ref(r64)["grad"]
        scale = 0.25

    mh = map_handle_from_oracle(m, True)
    dh = decoder_handle_from_oracle(dec, sigmoid_out=c.sigmoid, bias=c.bias)
    qc = q.cuda()
    ops.set_option("split_min_queries", 1)
    ops.set_option("sort_min_queries", 1 if c.sort else 0)
    try:
        call = lambda: ops.query_sdf(mh, dh, qc, nn_k=c.K, weighted_first=True, need_grad=True)  # noqa: E731
        _, names = kernels_run(call)
        out = call()
        torch.cuda.synchronize()
    finally:
        ops.set_option("split_min_queries", 0)
        ops.set_option("sort_min_queries", ops.SORT_MIN_QUERIES)
    assert any(f"wsq_decode_kernel<{c.F}, true, false>" in k for k in names), sorted(names)
    assert any("sort_key_kernel" in k for k in names) == c.sort, sorted(names)

    assert np.array_equal(out["nn_count"].cpu().numpy(), ref["nn_count"].numpy())
    assert_sdf_close(out["sdf"].cpu(), ref_sdf, scale)
    assert float(out["sdf_std"].abs().max()) == 0.0
    gscale = float(np.abs(ref_grad).mean()) + 1e-12
    assert_rel_close(out["grad"].cpu(), ref_grad, 1e-4, gscale, g64, kink_rows=6 if c.n < 100000 else 40)
