"""The A-slot ring of the adjoint schedule of wsq_decode_kernel<F, true, false> at sizes where it wraps many times.

Group i of a CTA lives in slot i % S (S = 3 for two-layer heads, 4 for one-layer heads, from the shared-memory plan)
and its barriers are keyed by (slot, i % 2).  Every case gives each CTA at least 4 S + 1 groups, so that every
(slot, pair) barrier goes through both parities at least twice; CTAs get different group counts and the last group is
partial.  Besides the oracle, each case checks that a random permutation of the batch gives bit-identical results per
query: a query's arithmetic does not depend on its group-mates, so a wrong slot, barrier phase or query index shows up
as a mismatch."""
from collections import namedtuple
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import pin_oracle as po
from tests.helpers import (assert_rel_close, assert_sdf_close, decoder_handle_from_oracle, kernels_run,
                           map_handle_from_oracle, oracle64, queries_near, synthetic_map)

Case = namedtuple("Case", "F L K leaky")
CASES = [Case(F, L, K, L == 2) for F, K in ((8, 6), (16, 5), (32, 8)) for L in (1, 2)]


def ring_slots(L):
    """A slots of the adjoint schedule (plan_ws_layout): 3 next to the transposed layer-1 weights, else 4."""
    return 3 if L == 2 else 4


def batch_size(L, sms):
    """Every CTA of the grid (one per SM) takes >= 4 S + 1 groups of 64 queries, a third of them one more, and the
    last group holds 29 queries."""
    groups = sms * (4 * ring_slots(L) + 1) + sms // 3
    return 64 * groups + 29


@lru_cache(maxsize=None)
def _map(F):
    return synthetic_map(n_surface=60000, seed=F + 11, resolution=0.4, buffer_size=200003, feature_dim=F,
                         local_radius=14.0, diff_td=3.0)


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[f"F{c.F}-L{c.L}" for c in CASES])
def test_adjoint_ring_wraps(c):
    from pin_slam_b200 import ops

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = batch_size(c.L, sms)
    assert (n + 63) // 64 >= sms * (4 * ring_slots(c.L) + 1)
    m = _map(c.F)
    dec = po.make_decoder(c.F + 3, 64, c.L, 1, 0.044, seed=c.F + c.L)
    dec.leaky = c.leaky
    q = queries_near(m, n, seed=c.F * 10 + c.L)
    q[:3] = torch.tensor([300.0, -200.0, 50.0])  # no neighbours at all
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(5))

    mh = map_handle_from_oracle(m, True)
    dh = decoder_handle_from_oracle(dec)
    qc = q.cuda()
    ops.set_option("split_min_queries", 1)
    ops.set_option("sort_min_queries", 0)
    try:
        call = lambda x: ops.query_sdf(mh, dh, x, nn_k=c.K, weighted_first=True, need_grad=True)  # noqa: E731
        # the profiler now and then delivers no kernel record at all for a call (kernels_run): more attempts than the
        # default, since a lost trace says nothing about the kernel
        _, names = kernels_run(lambda: call(qc), tries=6)
        out = {k: v.cpu() for k, v in call(qc).items()}
        outp = {k: v.cpu() for k, v in call(qc[perm.cuda()].contiguous()).items()}
        torch.cuda.synchronize()
    finally:
        ops.set_option("split_min_queries", 0)
        ops.set_option("sort_min_queries", ops.SORT_MIN_QUERIES)
    assert any(f"wsq_decode_kernel<{c.F}, true, false>" in k for k in names), sorted(names)
    assert not any("sort_key_kernel" in k for k in names), sorted(names)

    for name in ("sdf", "grad", "nn_count"):
        a, b = out[name][perm].numpy(), outp[name].numpy()
        same = (a == b) | (np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else a == b
        assert same.all(), f"{name}: {(~same).reshape(n, -1).any(axis=1).sum()} queries differ under a permutation"

    ref = po.query_sdf(m, dec, q, c.K, True, need_grad=True)
    r64 = oracle64(m, dec, q, c.K, True, ref, need_grad=True)
    assert np.array_equal(out["nn_count"].numpy(), ref["nn_count"].numpy())
    assert_sdf_close(out["sdf"], ref["sdf"].numpy(), dec.sdf_scale)
    ref_grad = ref["grad"].numpy()
    gscale = float(np.abs(ref_grad).mean()) + 1e-12
    assert_rel_close(out["grad"], ref_grad, 1e-4, gscale, r64["grad"], kink_rows=40)
