"""Every launch path of the query (K1) against the oracle, and the coverage ledger of the kernel instantiations.

pinb200_query_sdf decodes a batch on one of four paths:
  fused    one query_kernel<F, WF, false> launch (search + decode)
  full     split: search_kernel<false, false> writes full Stash blocks, query_kernel<F, WF, true> decodes them
           (decode-every-neighbour maps, weighted_first decoders wsq_decode_kernel cannot run, training batches of
           such maps)
  compact  split: search_kernel<SEEDS, true> writes compact StashS blocks, wsq_decode_kernel<F, GRAD, false> decodes
  sorted   compact, with the queries spatially sorted first (sort_key_kernel)
Each case below names the kernels it must launch; the profiler trace of the call must show exactly those, so that a
change of the dispatch rules cannot quietly move a case onto another kernel.  The ledger test (no GPU) checks that
the cases, together with the K2 cases of tests/helpers.py, launch every instantiation the sources contain."""
import os
import re
from collections import namedtuple
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import pin_oracle as po
from tests.helpers import (TRAIN_BWD_CASES, assert_close_frac, assert_rel_close, assert_sdf_close,
                           decoder_handle_from_oracle, flat_decoder_params, kernels_run, map_handle_from_oracle,
                           oracle64, queries_near, synthetic_map, train_bwd_kernel_name)

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pin_slam_b200", "csrc")

# color: None, "value" (colour head, value only) or "jac" (colour head and its Jacobian; needs grad)
Case = namedtuple("Case", "path F wf L K grad color leaky bias pgo train")
CASES = [
    # fused: query_kernel<F, WF, false> for every F and both modes
    Case("fused", 4, True, 1, 4, True, None, False, True, True, False),
    Case("fused", 4, False, 2, 3, True, None, True, True, False, False),
    Case("fused", 8, False, 1, 6, True, "jac", False, True, False, False),
    Case("fused", 8, True, 1, 6, True, None, False, False, False, False),
    Case("fused", 16, False, 2, 5, True, None, True, False, False, False),
    Case("fused", 16, True, 3, 7, False, None, False, True, False, False),
    Case("fused", 32, True, 2, 8, True, "value", True, True, False, False),
    Case("fused", 32, False, 1, 1, True, None, False, True, True, False),
    Case("fused", 64, False, 2, 2, True, None, False, True, False, False),
    Case("fused", 64, True, 1, 8, True, None, True, False, False, False),
    Case("fused", 8, False, 1, 6, False, None, False, True, False, True),
    # full stash: decode-every-neighbour maps (K = 1, 3, 5, 6, 8: 32 % K != 0 leaves a short last row tile) ...
    Case("full", 4, False, 1, 5, True, None, False, True, False, False),
    Case("full", 8, False, 1, 6, True, None, False, True, False, False),
    Case("full", 8, False, 1, 6, False, "value", False, True, False, False),
    Case("full", 16, False, 2, 3, True, None, True, False, False, False),
    Case("full", 32, False, 2, 8, True, "jac", False, True, True, False),
    Case("full", 64, False, 1, 1, True, None, False, True, False, False),
    Case("full", 8, False, 1, 6, False, None, False, True, False, True),
    # ... and weighted_first decoders the warp-specialised decode does not take (F = 4 / 64, 3 hidden layers)
    Case("full", 4, True, 2, 4, True, None, False, True, False, False),
    Case("full", 8, True, 3, 6, True, None, False, True, False, False),
    Case("full", 16, True, 3, 5, False, None, True, True, False, False),
    Case("full", 32, True, 3, 8, True, "jac", False, False, False, False),
    Case("full", 64, True, 2, 8, True, None, False, True, True, False),
    Case("full", 4, True, 1, 6, False, None, False, True, False, True),
    # compact stash, warp-specialised decode: every F, with and without d/dq
    Case("compact", 8, True, 1, 6, True, None, False, True, False, False),
    Case("compact", 8, True, 2, 6, False, None, False, True, False, False),
    Case("compact", 16, True, 2, 4, True, None, True, False, False, False),
    Case("compact", 16, True, 1, 5, False, None, False, False, True, False),
    Case("compact", 32, True, 2, 8, True, "jac", True, True, False, False),
    Case("compact", 32, True, 2, 8, False, "value", False, True, False, False),
    Case("compact", 32, True, 2, 8, False, None, False, True, False, True),
    Case("sorted", 32, True, 2, 8, True, None, False, True, True, False),
    Case("sorted", 8, True, 1, 6, False, None, False, False, False, False),
]

FAMILY = re.compile(r"(?<![A-Za-z_])(query_kernel|wsq_decode_kernel|search_kernel|train_bwd_mma_kernel|train_bwd_kernel)"
                    r"<[^<>]*>")


def _b(x):
    return "true" if x else "false"


def expected_kernels(c):
    """The query_kernel / wsq_decode_kernel / search_kernel instantiations the call of case `c` launches."""
    def decode(grad):
        if c.path == "fused":
            return f"query_kernel<{c.F}, {_b(c.wf)}, false>"
        if c.path == "full":
            return f"query_kernel<{c.F}, {_b(c.wf)}, true>"
        return f"wsq_decode_kernel<{c.F}, {_b(grad)}, false>"

    names = {decode(c.grad)}
    if c.color:
        names.add(decode(c.color == "jac"))
    if c.path == "full":
        names.add("search_kernel<false, false>")
    elif c.path in ("compact", "sorted"):
        names.add(f"search_kernel<{_b(c.grad)}, true>")
    return names


def case_id(c):
    return (f"{c.path}-F{c.F}-{'wf' if c.wf else 'nwf'}-L{c.L}-K{c.K}" + ("-grad" if c.grad else "-value")
            + (f"-color_{c.color}" if c.color else "") + ("-leaky" if c.leaky else "") + ("" if c.bias else "-nobias")
            + ("-pgo" if c.pgo else "") + ("-train" if c.train else ""))


def source_instantiations():
    """Kernel instantiations the dispatch code launches (the wsq_decode_kernel profiling variants excluded)."""
    src = {f: open(os.path.join(CSRC, f)).read() for f in ("query.cu", "wsq.cu", "train.cu")}
    q = src["query.cu"]
    names = {f"query_kernel<{F}, {wf}, {sp}>" for F in re.findall(r"launch_query<(\d+), WF, SPLIT>\(", q)
             for wf, sp in re.findall(r"dispatch_query_wf<(true|false), (true|false)>\(", q)}
    names |= {f"search_kernel<{a}, {b}>" for a, b in re.findall(r"search_kernel<(true|false), (true|false)><<<", q)}
    names |= {f"wsq_decode_kernel<{F}, {g}, false>"
              for F, g, prof in re.findall(r"launch_wsq<(\d+), (true|false), (true|false)>\(", src["wsq.cu"])
              if prof == "false"}
    names |= {f"train_bwd_mma_kernel<{F}, {L}>" for F, L in re.findall(r"launch_train_mma<(\d+), (\d+)>\(", src["train.cu"])}
    names |= {f"train_bwd_kernel<{H}, {DP}>" for H, DP in re.findall(r"launch_train<(\d+), (\d+)>\(", src["train.cu"])}
    return names


def test_coverage_ledger():
    """No GPU: the cases of this file and the K2 cases launch, between them, every kernel instantiation of the
    query and training paths -- 20 query_kernel, 6 wsq_decode_kernel, 3 search_kernel, 10 train_bwd_mma_kernel and
    4 train_bwd_kernel -- and nothing else."""
    inst = source_instantiations()
    count = lambda fam: sum(n.startswith(fam + "<") for n in inst)  # noqa: E731
    assert [count(f) for f in ("query_kernel", "wsq_decode_kernel", "search_kernel", "train_bwd_mma_kernel",
                               "train_bwd_kernel")] == [20, 6, 3, 10, 4], sorted(inst)
    covered = set().union(*(expected_kernels(c) for c in CASES))
    covered |= {train_bwd_kernel_name(c[0], c[2], c[8]) for c in TRAIN_BWD_CASES}
    assert covered == inst, (sorted(inst - covered), sorted(covered - inst))
    # the shapes where the decode-every-neighbour split goes wrong first: short last row tiles
    assert {c.K for c in CASES if c.path == "full" and not c.wf} >= {1, 3, 5, 6, 8}
    for path in ("fused", "full", "compact"):
        assert any(c.leaky for c in CASES if c.path == path) and any(not c.bias for c in CASES if c.path == path)


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("oc", [1, 3])
def test_decoder_param_count_matches_flat_parameters(bias, L, oc):
    """No GPU: pinb200_decoder_param_count (the length K2 and the fused Adam step use) equals the length of
    Decoder.flat_parameters() with and without biases.  The view's pointers are never dereferenced."""
    import ctypes as C

    from pin_slam_b200 import _lib
    from pin_slam_b200.config import HotPathConfig
    from pin_slam_b200.model import Decoder

    cfg = HotPathConfig.kitti(device="cpu", mlp_bias_on=bias)
    dec = Decoder(cfg, 64, L, oc)
    v = _lib.DecoderView()
    for i in range(L):
        v.w[i] = 0x1000 + 0x100 * i
        v.b[i] = 0x2000 + 0x100 * i if bias else None
    v.w_out, v.b_out = 0x3000, (0x3100 if bias else None)
    v.n_hidden, v.hidden_dim, v.in_dim, v.out_dim = L, 64, cfg.feature_dim + 3, oc
    n = int(_lib.load().pinb200_decoder_param_count(C.byref(v)))
    assert n == dec.flat_parameters().numel() == sum(p.numel() for p in dec.parameters())


# --------------------------------------------------------------------------------------
# the launch-path matrix (GPU)
# --------------------------------------------------------------------------------------
def _ops():
    from pin_slam_b200 import ops

    return ops


class _Options:
    """Forces (split=True) or forbids (split=False) the two-launch pipeline, with the spatial sort on or off, and
    restores the library defaults afterwards."""

    def __init__(self, split, sort=False):
        self.split, self.sort = split, sort

    def __enter__(self):
        o = _ops()
        o.set_option("split_min_queries", 1 if self.split else 1 << 40)
        o.set_option("sort_min_queries", 1 if self.sort else 0)
        o.set_option("sort_min_queries_color", 1 if self.sort else 0)

    def __exit__(self, *exc):
        o = _ops()
        o.set_option("split_min_queries", 0)
        o.set_option("sort_min_queries", o.SORT_MIN_QUERIES)
        o.set_option("sort_min_queries_color", 0)


@lru_cache(maxsize=None)
def _map(F, pgo, color):
    return synthetic_map(n_surface=60000, seed=F + 1, resolution=0.4, buffer_size=200003, feature_dim=F, color=color,
                         after_pgo=pgo, local_radius=14.0, diff_td=3.0)


SEARCH_KEYS = ("nn_count", "knn_idx", "knn_gidx", "knn_dist2", "knn_weight", "certainty")


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[case_id(c) for c in CASES])
def test_query_path_vs_oracle(c):
    """One launch path on a seeded local map with an age filter: a ragged last tile, 16 queries without neighbours,
    value and d/dq, sdf_std of decode-every-neighbour maps, colour head and Jacobian, certainty; the kernels launched;
    on split paths the search outputs of a fused launch of the same batch, bit for bit; in training mode the
    certainty / ts_update side effects of the first training_rows queries."""
    o = _ops()
    m = _map(c.F, c.pgo, c.color is not None)
    dec = po.make_decoder(c.F + 3, 64, c.L, 1, 0.044, seed=3, bias=c.bias)
    cdec = po.make_decoder(c.F + 3, 64, c.L, 3, 1.0, seed=4, bias=c.bias) if c.color else None
    dec.leaky = c.leaky
    if cdec is not None:
        cdec.leaky = c.leaky
    n = 8011 if c.F == 64 else 20011
    q = queries_near(m, n, seed=5)
    q[:16] = torch.tensor([300.0, -200.0, 50.0])  # no neighbours at all
    jac = c.color == "jac"
    kw = dict(color_dec=cdec, color_grad=jac) if c.color else {}
    ref = po.query_sdf(m, dec, q, c.K, c.wf, need_grad=c.grad, **kw)
    r64 = oracle64(m, dec, q, c.K, c.wf, ref, need_grad=c.grad, **kw) if (c.grad or c.color or not c.wf) else None

    mh = map_handle_from_oracle(m, True)
    dh = decoder_handle_from_oracle(dec, bias=c.bias)
    ch = decoder_handle_from_oracle(cdec, sigmoid_out=True, bias=c.bias) if c.color else None
    qc = q.cuda()
    rows = 15013 if n > 15013 else n - 1000  # training side effects for the first `rows` queries only
    g = torch.Generator().manual_seed(6)
    ts = torch.randint(0, 7, (n,), generator=g, dtype=m.local_point_ts_update.dtype)
    train_kw = dict(training_mode=True, query_ts=ts.to(torch.int32).cuda(), training_rows=rows) if c.train else {}
    split = c.path != "fused"
    if split:  # a fused launch of the same batch: the search outputs must be bit-identical
        with _Options(False):
            fused = o.query_sdf(mh, dh, qc, nn_k=c.K, weighted_first=c.wf, need_grad=False, save_knn=True)
            fused = {k: fused[k].clone() for k in SEARCH_KEYS}
    with _Options(split, sort=c.path == "sorted"):
        call = lambda h: o.query_sdf(h, dh, qc, nn_k=c.K, weighted_first=c.wf, need_grad=c.grad,  # noqa: E731
                                     color_dec=ch, color_grad=jac, save_knn=True, **train_kw)
        _, names = kernels_run(lambda: call(map_handle_from_oracle(m, True)))  # profiled on a copy of the map
        out = call(mh)
        torch.cuda.synchronize()
    ran = {mm.group(0) for k in names for mm in FAMILY.finditer(k)}
    assert ran == expected_kernels(c), (sorted(ran), sorted(names))
    assert any("sort_key_kernel" in k for k in names) == (c.path == "sorted"), sorted(names)

    assert np.array_equal(out["nn_count"].cpu().numpy(), ref["nn_count"].numpy())
    assert int((out["nn_count"] == 0).sum()) >= 16
    assert_sdf_close(out["sdf"].cpu(), ref["sdf"], dec.sdf_scale)
    if c.grad:
        gscale = float(ref["grad"].abs().mean()) + 1e-12
        assert_rel_close(out["grad"].cpu(), ref["grad"], 1e-4, gscale, r64["grad"], kink_rows=6)
    if c.wf:
        assert float(out["sdf_std"].abs().max()) == 0.0
    else:
        assert_rel_close(out["sdf_std"].cpu(), ref["sdf_std"], 1e-4, dec.sdf_scale, r64["sdf_std"])
    if c.color:
        assert_rel_close(out["color"].cpu(), ref["color"], 1e-5, 1.0, r64["color"])
        if jac:
            cscale = float(ref["color_grad"].abs().mean()) + 1e-12
            assert_rel_close(out["color_grad"].cpu(), ref["color_grad"], 1e-4, cscale, r64["color_grad"], kink_rows=8)
    if not c.train:  # (in training mode the certainty read races with the scatter of the same launch)
        np.testing.assert_allclose(out["certainty"].cpu().numpy(), ref["certainty"].numpy(), rtol=1e-5, atol=1e-6)
    if split:
        for k in SEARCH_KEYS:
            if k != "certainty" or not c.train:
                assert torch.equal(out[k], fused[k]), f"{k}: the split search differs from the fused one"
    if c.train:
        mc = m.clone()
        po.query_feature(mc, q[:rows], ts[:rows], c.K, c.wf, training_mode=True)
        np.testing.assert_allclose(mh.keep["certainty"].cpu().numpy(), mc.local_point_certainties.numpy(), rtol=1e-5,
                                   atol=1e-5)
        assert np.array_equal(mh.keep["ts_update"].cpu().numpy(), mc.local_point_ts_update.numpy())
        assert not torch.equal(mc.local_point_certainties, m.local_point_certainties)


@pytest.mark.gpu
def test_map_iterations_without_biases_vs_oracle():
    """Three pinb200_map_iterations steps (batch assembly, training forward, loss, K2, Adam) with a decoder without
    biases (2 x 64, mlp_bias_on False) against autograd + torch Adam through the oracle.  The flat decoder vector,
    its gradient and both Adam moments are followed by sentinel tails the library must not touch."""
    o = _ops()
    F, K, wf, L = 8, 6, False, 2
    m = synthetic_map(n_surface=30000, seed=11, resolution=0.4, buffer_size=200003, feature_dim=F, local_radius=14.0,
                      diff_td=3.0)
    dec = po.make_decoder(F + 3, 64, L, 1, 0.044, seed=5, bias=False)
    g = torch.Generator().manual_seed(3)
    P, bs, n_iter, decim = 20000, 4096, 3, 10
    sigma, weight_e, eik_eps, lr, adam_eps, wd = 0.1, 0.5, 0.02, 0.01, 1e-15, 1e-7
    coord_pool = queries_near(m, P, seed=12)
    label_pool = 0.2 * torch.randn(P, generator=g)
    ts_pool = torch.randint(0, 3, (P,), generator=g, dtype=m.local_point_ts_update.dtype)
    weight_pool = torch.rand(P, generator=g) + 0.5
    index = torch.randint(0, P, (n_iter, bs), generator=g)

    # oracle: the decoder's weights and the local features train, the zero biases stay out of the optimiser
    mo = m.clone()
    deco = dec.clone()
    feat_o = mo.local_geo_features.requires_grad_(True)
    dw = [w.requires_grad_(True) for w, _ in deco.hidden] + [deco.out[0].requires_grad_(True)]
    opt = po.make_adam([dw, [feat_o]], lr=lr, eps=adam_eps, weight_decay=wd)
    for it in range(n_iter):
        i = index[it]
        opt.zero_grad()
        loss, _ = po.mapping_loss(mo, deco, coord_pool[i], label_pool[i], ts_pool[i], weight_pool[i], K, wf, sigma, True,
                                  weight_e, decim, eik_eps)
        loss.backward()
        opt.step()

    mh = map_handle_from_oracle(m, True)
    feat = mh.keep["geo_feat"]
    n_par = flat_decoder_params(dec, bias=False).numel()

    def tailed(init):
        buf = torch.full((n_par + 256,), 12345.0, device="cuda")
        buf[:n_par] = init
        return buf

    bufs = [tailed(flat_decoder_params(dec, bias=False).cuda()), tailed(0.0), tailed(0.0), tailed(0.0)]
    flat, gdec, md, vd = (b[:n_par] for b in bufs)
    ws, off = [], 0
    for w, _ in dec.hidden:
        ws.append(flat[off:off + w.numel()].view_as(w))
        off += w.numel()
    dh = o.DecoderHandle(ws, [None] * L, flat[off:].view_as(dec.out[0]), None, out_scale=dec.sdf_scale)
    assert dh.param_count() == n_par
    gfeat, mf, vf = torch.zeros_like(feat), torch.zeros_like(feat), torch.zeros_like(feat)
    o.map_iterations(mh, dh, n_iter, nn_k=K, weighted_first=wf, coord_pool=coord_pool.cuda(),
                     label_pool=label_pool.cuda(), ts_pool=ts_pool.to(torch.int32).cuda(), weight_pool=weight_pool.cuda(),
                     index=index.cuda(), decimation=decim, eik_eps=eik_eps, sigma=sigma, weight_e=weight_e,
                     loss_weight_on=True, lr=lr, beta1=0.9, beta2=0.99, eps=adam_eps, weight_decay=wd,
                     train_decoder=True, first_step=1, feat=feat, dec_flat=flat, grad_feat=gfeat, grad_dec=gdec,
                     m_feat=mf, v_feat=vf, m_dec=md, v_dec=vd, losses=torch.zeros(2, device="cuda"), work={})
    torch.cuda.synchronize()
    for name, b in zip(("dec_flat", "grad_dec", "m_dec", "v_dec"), bufs):
        assert bool((b[n_par:] == 12345.0).all()), f"map_iterations wrote past the end of {name}"
    assert float(gdec.abs().max()) == 0.0  # zero on exit
    assert_close_frac(feat.cpu().numpy(), feat_o.detach().numpy())
    assert_close_frac(flat.cpu().numpy(), torch.cat([w.detach().reshape(-1) for w in dw]).numpy())
    np.testing.assert_allclose(mh.keep["certainty"].cpu().numpy(), mo.local_point_certainties.numpy(), rtol=1e-4,
                               atol=1e-4)
    assert np.array_equal(mh.keep["ts_update"].cpu().numpy(), mo.local_point_ts_update.numpy())
    # flat vectors of any other length are refused before anything runs
    with pytest.raises(RuntimeError):
        o.map_iterations(mh, dh, 1, nn_k=K, weighted_first=wf, coord_pool=coord_pool.cuda(),
                         label_pool=label_pool.cuda(), ts_pool=ts_pool.to(torch.int32).cuda(),
                         weight_pool=weight_pool.cuda(), index=index[:1].cuda(), decimation=decim, eik_eps=eik_eps,
                         sigma=sigma, weight_e=weight_e, loss_weight_on=True, lr=lr, beta1=0.9, beta2=0.99,
                         eps=adam_eps, weight_decay=wd, train_decoder=True, first_step=1, feat=feat,
                         dec_flat=bufs[0], grad_feat=gfeat, grad_dec=gdec, m_feat=mf, v_feat=vf, m_dec=md, v_dec=vd,
                         losses=torch.zeros(2, device="cuda"), work={})
