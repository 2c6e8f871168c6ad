"""Map training at the sizes a run reaches: K2 (the training backward) and the fused mapping loop.

Both K2 kernels are persistent: a CTA takes tiles blockIdx.x, blockIdx.x + gridDim.x, ... and keeps its decoder
gradients across them (in registers, dacc0 / dacc1, in train_bwd_mma_kernel; in shared memory, s_dW, in
train_bwd_kernel) until one flush at the end.  A KITTI mapper batch gives every CTA about three tiles.

Exact arm: K2's inputs are built directly (no search) from dyadic rationals with few significant bits: weights with at
most 11, so the lo part of their 3xTF32 split is zero; features, positions, IDW weights and d loss / d out such that
every activation and gradient operand is exactly hi + lo in TF32, and every dot product and output sum has terms that
are multiples of one 2^-m with sum |terms| < 2^(23 - m).  Then every partial sum, in any order and under any atomic
interleaving, is exact, so grad_feat and grad_dec must equal the fp64 autograd reference bit for bit.  The test
asserts this premise on its own fp64 intermediates first.  The inputs also put a few per cent of the hidden
pre-activations at exactly 0, which pins the ReLU derivative there to torch's (0).  Every K2 instantiation runs at
n_tiles >= 2 x 16 x SMs (16 CTAs of 128 threads fill an SM), so every CTA runs at least two tiles, with a ragged last
tile, d loss / d out non-zero in every tile, two neural points named by 10^5 rows each, grad_feat 4 bytes off the
16-byte grid on both kernels (the mapper's gradient arena puts the colour-feature block there), n = 1 and qpt - 1 / qpt
/ qpt + 1, a second call into the same buffers, and sentinels behind both outputs.

Random arm: realistic values (0.1 randn features, nn.Linear-initialised decoders, leaky ReLU, sigmoid colour heads,
decoders without biases) at the same sizes and at KITTI's and cfg2's mapper shapes, within the fp32/fp64 bounds of
tests/helpers.py.

pinb200_map_iterations against the oracle (autograd + torch Adam) at full batch sizes, on the branches a run takes:
frozen decoder, weighted_first maps, the split training forward, no Eikonal rows, no loss weights, and the
data-parallel two-call form (stages 1 then 2).  Mapper.mapping with the colour head against the same iterations
issued through ops on separately allocated buffers.

The ledger test (no GPU) checks that the exact and random arms each launch every K2 instantiation."""
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import pin_oracle as po
from tests.helpers import (assert_close_frac, assert_decoder_grad_close, assert_rel_close, kernels_run,
                           map_handle_from_oracle, queries_near, synthetic_map, train_bwd_kernel_name)
from tests.test_query_paths import FAMILY, source_instantiations

# F features, L hidden layers (64 wide), K neighbours, weighted_first, oc outputs, after_pgo quaternions,
# feat_off / gfeat_off: the feature table / grad_feat start this many floats past a 16-byte boundary
K2Case = namedtuple("K2Case", "F L K wf oc pgo feat_off gfeat_off")
EXACT_CASES = [
    # train_bwd_mma_kernel<F, L>; decode-every-neighbour with K in {1, 3, 5, 6, 7, 8}
    K2Case(4, 1, 3, False, 1, True, 0, 0),
    K2Case(4, 2, 8, True, 1, False, 0, 1),
    K2Case(8, 1, 6, False, 1, False, 0, 1),  # KITTI's shape, scalar feature-gradient scatter
    K2Case(8, 2, 5, False, 1, False, 0, 0),
    K2Case(16, 1, 7, False, 1, False, 0, 0),
    K2Case(16, 2, 8, True, 1, True, 0, 1),
    K2Case(32, 1, 1, False, 1, False, 0, 0),
    K2Case(32, 2, 8, True, 1, False, 0, 0),  # cfg2's shape
    K2Case(64, 1, 8, False, 2, False, 0, 1),
    K2Case(64, 2, 4, True, 1, True, 0, 0),
    # train_bwd_kernel<64, DP>: 3 hidden layers, or a feature table off the 16-byte grid
    K2Case(4, 3, 5, False, 1, False, 0, 1),  # aligned table, unaligned grad_feat: scalar scatter
    K2Case(8, 3, 7, True, 1, True, 0, 0),
    K2Case(16, 2, 3, False, 1, False, 1, 0),
    K2Case(32, 1, 8, True, 1, True, 1, 1),
    K2Case(64, 2, 1, False, 2, False, 1, 0),
]

# random arm: + leaky ReLU, biases on/off (oc 3: sigmoid colour head); n None: the multi-tile size
RandCase = namedtuple("RandCase", K2Case._fields + ("leaky", "bias", "n"))
RANDOM_CASES = [
    RandCase(8, 1, 6, False, 1, False, 0, 0, False, True, 26218),  # KITTI mapper: 16 384 samples + 6 x 1 639 shifted
    RandCase(32, 2, 8, True, 1, False, 0, 0, False, True, 26218),  # cfg2 mapper
    RandCase(4, 1, 5, False, 3, False, 0, 0, True, True, None),
    RandCase(4, 2, 3, True, 1, True, 0, 0, False, False, None),
    RandCase(8, 1, 8, True, 3, False, 0, 1, False, True, None),  # colour head, grad_feat where the arena puts it
    RandCase(8, 2, 7, False, 3, False, 0, 1, True, False, None),
    RandCase(16, 1, 8, True, 1, False, 0, 0, True, False, None),
    RandCase(16, 2, 1, False, 1, True, 0, 0, False, True, None),
    RandCase(32, 1, 5, False, 3, False, 0, 1, False, True, None),
    RandCase(64, 1, 3, True, 1, False, 0, 0, True, True, None),
    RandCase(64, 2, 8, False, 1, False, 0, 0, False, False, None),
    RandCase(8, 3, 6, False, 1, False, 0, 1, True, True, None),
    RandCase(16, 2, 5, True, 3, False, 1, 0, False, True, None),
    RandCase(32, 2, 7, False, 1, True, 1, 1, True, False, None),
    RandCase(64, 1, 8, True, 1, False, 1, 0, False, True, None),
]

SENTINEL = 12345.0
TF32_MASK = np.uint32(0xFFFFE000)
# unit quaternions (w, x, y, z) with components in {0, +-1/2, +-1}: rotations of dyadic vectors stay dyadic
QUATS = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1], [0.5, 0.5, 0.5, 0.5], [0.5, -0.5, 0.5, -0.5],
                  [-0.5, 0.5, 0.5, 0.5], [0.5, 0.5, -0.5, -0.5]])

Dec = namedtuple("Dec", "W b Wout bout scale leaky sigmoid")  # numpy arrays; b[l] / bout None: no bias
K2Inputs = namedtuple("K2Inputs", "feat pts ori q idx w dl pgo")


def _case_id(c):
    s = f"F{c.F}-L{c.L}-K{c.K}-{'wf' if c.wf else 'nwf'}-oc{c.oc}" + ("-pgo" if c.pgo else "")
    s += ("-feat+4B" if c.feat_off else "") + ("-gfeat+4B" if c.gfeat_off else "")
    if isinstance(c, RandCase):
        s += ("-leaky" if c.leaky else "") + ("" if c.bias else "-nobias") + (f"-n{c.n}" if c.n else "")
    return s


def _kernel(c):
    return train_bwd_kernel_name(c.F, c.L, c.feat_off == 0)


def _qpt(c):
    return 128 if c.wf else 128 // c.K


def test_k2_case_ledger():
    """No GPU: the exact arm and the random arm each launch every K2 instantiation the dispatch code contains, so a
    new instantiation without a multi-tile case fails here.  Both arms cover decode-every-neighbour row tiles with
    dead rows (128 mod K != 0) and grad_feat off the 16-byte grid on both kernels."""
    inst = {n for n in source_instantiations() if n.startswith(("train_bwd_mma_kernel<", "train_bwd_kernel<"))}
    assert len(inst) == 14, sorted(inst)
    for cases in (EXACT_CASES, RANDOM_CASES):
        assert {_kernel(c) for c in cases} == inst, sorted(inst ^ {_kernel(c) for c in cases})
        for fam in ("train_bwd_mma_kernel<", "train_bwd_kernel<"):
            assert any(c.gfeat_off and c.feat_off == 0 and _kernel(c).startswith(fam) for c in cases)
    assert {c.K for c in EXACT_CASES if not c.wf} >= {1, 3, 5, 7, 8}
    assert any(c.pgo for c in EXACT_CASES) and any(c.oc > 1 for c in EXACT_CASES)
    assert any(c.leaky for c in RANDOM_CASES) and any(not c.bias for c in RANDOM_CASES)
    assert any(c.oc == 3 for c in RANDOM_CASES)


# --------------------------------------------------------------------------------------
# inputs, the fp64 reference and the exactness premise
# --------------------------------------------------------------------------------------
def _multi_tile_n(c, sms):
    """Queries for n_tiles = 2 x 16 x SMs + 1 tiles, the last one ragged."""
    qpt = _qpt(c)
    return 2 * 16 * sms * qpt + max(1, qpt // 3)


def _exact_inputs(c, n, seed, n_pts=40000, hot=2):
    """Dyadic K2 inputs: features in {0, +-1/8, +-1/4}, positions on a 1/8 grid, IDW weights k/4, d loss / d out
    +-1/4 on one query with a neighbour per tile (and nowhere else), `-1` tails and rows without any
    neighbour; `hot` neural points named by 10^5 rows each when the batch is large enough."""
    rng = np.random.default_rng(seed)
    K, qpt = c.K, _qpt(c)
    feat = rng.choice(np.array([-2.0, -1.0, 0.0, 0.0, 1.0, 2.0]), size=(n_pts, c.F)) / 8
    pts = rng.integers(-8, 9, size=(n_pts, 3)) / 8
    ori = QUATS[rng.integers(0, len(QUATS), n_pts)]
    q = rng.integers(-8, 9, size=(n, 3)) / 8
    cnt = np.where(rng.random(n) < 0.7, K, rng.integers(0, K + 1, n))
    chosen = np.minimum(np.arange(0, n, qpt) + rng.integers(0, qpt, (n + qpt - 1) // qpt), n - 1)
    cnt[chosen] = np.maximum(cnt[chosen], 1)
    live = np.arange(K)[None, :] < cnt[:, None]
    idx = np.where(live, rng.integers(hot, n_pts, (n, K)), -1).astype(np.int32)
    slots = np.flatnonzero(live)
    if hot and slots.size >= 2 * hot * 100_000:
        pick = rng.choice(slots, hot * 100_000, replace=False).reshape(hot, -1)
        for h in range(hot):
            idx.reshape(-1)[pick[h]] = h
    w = np.where(live, rng.integers(1, 5, (n, K)) / 4, 0.0)
    dl = np.zeros((n, c.oc))
    dl[chosen] = rng.choice(np.array([-1.0, 1.0]), size=(chosen.size, c.oc)) / 4
    return K2Inputs(feat, pts, ori, q, idx, w, dl, c.pgo)


def _exact_decoder(c, seed):
    """Sparse weights in {0, +-1/4} (2 of 7 non-zero; 2 of 12 for 3 hidden layers, whose sums would not fit 23 bits
    otherwise), biases in {0, +-1/8}, out_scale 1/2, plain ReLU."""
    rng = np.random.default_rng(seed)
    vals = np.array([-1.0] + [0.0] * (5 if c.L < 3 else 10) + [1.0]) / 4
    W, b, d = [], [], c.F + 3
    for _ in range(c.L):
        W.append(rng.choice(vals, (64, d)))
        b.append(rng.choice(np.array([-1.0, 0.0, 0.0, 1.0]), 64) / 8)
        d = 64
    return Dec(W, b, rng.choice(vals, (c.oc, 64)), rng.choice(np.array([-1.0, 0.0, 1.0]), c.oc) / 8, 0.5, False,
               False)


def _random_inputs(c, n, seed, n_pts=40000):
    """0.1 randn features, points and queries in a 0.8 m box, normalised positive IDW weights over the valid
    neighbours, randn d loss / d out; `-1` tails and rows without neighbours."""
    g = np.random.default_rng(seed)
    K = c.K
    feat = (0.1 * g.standard_normal((n_pts, c.F))).astype(np.float32).astype(np.float64)
    pts = (0.8 * g.random((n_pts, 3))).astype(np.float32).astype(np.float64)
    qn = g.standard_normal((n_pts, 4))
    ori = (qn / np.linalg.norm(qn, axis=1, keepdims=True)).astype(np.float32).astype(np.float64)
    q = (0.8 * g.random((n, 3))).astype(np.float32).astype(np.float64)
    cnt = np.where(g.random(n) < 0.8, K, g.integers(0, K + 1, n))
    live = np.arange(K)[None, :] < cnt[:, None]
    idx = np.where(live, g.integers(0, n_pts, (n, K)), -1).astype(np.int32)
    w = np.where(live, g.random((n, K)) + 0.05, 0.0)
    w = (w / np.maximum(w.sum(1, keepdims=True), 1e-30)).astype(np.float32).astype(np.float64)
    dl = g.standard_normal((n, c.oc)).astype(np.float32).astype(np.float64) / n
    return K2Inputs(feat, pts, ori, q, idx, w, dl, c.pgo)


def _random_decoder(c, seed):
    sig = c.oc == 3
    d = po.make_decoder(c.F + 3, 64, c.L, c.oc, 0.044, seed=seed, bias=c.bias)
    W = [w.numpy().astype(np.float64) for w, _ in d.hidden]
    b = [bb.numpy().astype(np.float64) if c.bias else None for _, bb in d.hidden]
    bout = d.out[1].numpy().astype(np.float64) if c.bias else None
    return Dec(W, b, d.out[0].numpy().astype(np.float64), bout, 1.0 if sig else 0.044, c.leaky, sig)


def _flat(parts):
    return np.concatenate([p.reshape(-1) for p in parts if p is not None])


def _k2_reference(inp, dec, wf, dtype, keep=False):
    """d/d(feature table, decoder) of sum(out * dl) by autograd on the CPU: the decoder input rows rebuilt from the
    kNN lists (features and q - p, rotated into the point's frame after PGO, zero for `-1` entries), IDW-summed
    before the decoder (weighted_first) or after it, out = sigmoid(o) or out_scale * o.  `keep`: also the
    intermediates the exactness premise is checked on (in the row order of K2)."""
    cast = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dtype)  # noqa: E731
    n, K = inp.idx.shape
    feat = cast(inp.feat).requires_grad_(True)
    Ws = [cast(w).requires_grad_(True) for w in dec.W]
    bs = [None if b is None else cast(b).requires_grad_(True) for b in dec.b]
    Wo = cast(dec.Wout).requires_grad_(True)
    bo = None if dec.bout is None else cast(dec.bout).requires_grad_(True)
    idx = torch.from_numpy(inp.idx).long()
    valid = idx >= 0
    ii = idx.clamp(min=0)
    w, q, pts, ori = cast(inp.w), cast(inp.q), cast(inp.pts), cast(inp.ori)
    ex = {}

    def row(k):  # decoder input of neighbour slot k: [n, D]
        nv = q - pts[ii[:, k]]
        if inp.pgo:
            nv = po.quat_rotate_passive(ori[ii[:, k]], nv)
        v = valid[:, k:k + 1].to(dtype)
        return torch.cat([feat[ii[:, k]] * v, nv * v], 1)

    if wf:  # one slot at a time: [n, K, D] of fp64 would not fit
        x = 0
        for k in range(K):
            xk = row(k)
            x = x + w[:, k:k + 1] * xk
            if keep:
                with torch.no_grad():
                    ex["gather_abs"] = ex.get("gather_abs", 0) + (w[:, k:k + 1].abs() * xk.abs()).numpy()
                    ex["gather_grain"] = max(ex.get("gather_grain", -64), _grain(xk.numpy()))
    else:
        x = torch.stack([row(k) for k in range(K)], 1).reshape(n * K, -1)
    x.retain_grad()
    h, zs, ins = x, [], []
    for W, b in zip(Ws, bs):
        ins.append(h)
        z = h @ W.T if b is None else torch.addmm(b, h, W.T)
        z.retain_grad()
        zs.append(z)
        h = torch.nn.functional.leaky_relu(z) if dec.leaky else torch.relu(z)
    o = h @ Wo.T if bo is None else torch.addmm(bo, h, Wo.T)
    o.retain_grad()
    out = torch.sigmoid(o) if dec.sigmoid else o * dec.scale
    dl = cast(inp.dl)
    if wf:
        loss = (out * dl).sum()
    else:
        loss = (out.view(n, K, -1) * (w.unsqueeze(2) * dl.unsqueeze(1))).sum()
    loss.backward()
    gdec = _flat([t.grad.numpy() if t is not None else None for pair in zip(Ws, bs) for t in pair]
                 + [Wo.grad.numpy(), None if bo is None else bo.grad.numpy()])
    if keep:
        ex.update(x=x.detach().numpy(), ins=[t.detach().numpy() for t in ins], h_last=h.detach().numpy(),
                  z=[t.detach().numpy() for t in zs], G=[t.grad.numpy() for t in zs], go=o.grad.numpy(),
                  gx=x.grad.numpy())
    return feat.grad.numpy(), gdec, ex


def _grain(*arrays):
    """The smallest m such that every value of the arrays is an integer multiple of 2^-m."""
    m = -64
    for a in arrays:
        a = np.abs(np.asarray(a, np.float64)).ravel()
        a = a[a != 0]
        if a.size:
            mant, e = np.frexp(a)
            mi = (mant * 2.0 ** 53).astype(np.int64)
            low = np.log2((mi & -mi).astype(np.float64)).astype(np.int64)
            m = max(m, int((53 - e - low).max()))
    return m


def _assert_splits_exactly(name, a):
    """a is an fp32 value and exactly hi + lo of split_tf32 (hi = a truncated to TF32, lo = (a - hi) truncated)."""
    a = np.asarray(a, np.float64)
    f = a.astype(np.float32)
    assert np.array_equal(f.astype(np.float64), a), f"{name}: not an fp32 value"
    hi = (f.view(np.uint32) & TF32_MASK).view(np.float32)
    lo = ((f - hi).view(np.uint32) & TF32_MASK).view(np.float32)
    assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), a), f"{name}: not exactly hi + lo in TF32"


def _assert_sum_exact(name, abs_sum, m):
    """Every partial sum of terms that are multiples of 2^-m with sum |terms| < 2^(23 - m) is exact in fp32, in any
    order, and still after a second call adds the same terms again."""
    top = float(np.max(abs_sum)) if np.size(abs_sum) else 0.0
    assert top * 2.0 ** m < 2.0 ** 23, f"{name}: sum |terms| = {top:.4g} in units of 2^-{m} does not fit 23 bits"


def _assert_exact_premise(inp, dec, c, ex, relu_zeros=True):
    """The premise of the exact arm on the fp64 intermediates: TF32 weights, exactly split operands, exact sums,
    and (`relu_zeros`) hidden pre-activations at exactly 0 that carry a non-zero upstream gradient."""
    for l, W in enumerate(dec.W + [dec.Wout]):
        f = W.astype(np.float32)
        assert np.array_equal(f.astype(np.float64), W) and np.array_equal((f.view(np.uint32) & TF32_MASK).view(
            np.float32), f), f"weights {l}: more than 11 significant bits"
    gW = [_grain(W) for W in dec.W]
    gb = [_grain(b) for b in dec.b]
    if c.wf:
        _assert_sum_exact("IDW feature sum", ex["gather_abs"], _grain(inp.w) + ex["gather_grain"])
    _assert_splits_exactly("go", ex["go"])
    for l in range(c.L):
        a = ex["ins"][l]
        _assert_splits_exactly(f"layer {l} input", a)
        _assert_splits_exactly(f"G_{l}", ex["G"][l])
        _assert_sum_exact(f"z_{l}", np.abs(a) @ np.abs(dec.W[l]).T + np.abs(dec.b[l]), max(_grain(a) + gW[l], gb[l]))
        G = ex["G"][l]
        _assert_sum_exact(f"dW_{l}", np.abs(G).T @ np.abs(a), _grain(G) + _grain(a))
        _assert_sum_exact(f"db_{l}", np.abs(G).sum(0), _grain(G))
    go, hl = ex["go"], ex["h_last"]
    _assert_sum_exact("dW_out", np.abs(go).T @ np.abs(hl), _grain(go) + _grain(hl))
    _assert_sum_exact("db_out", np.abs(go).sum(0), _grain(go))
    # the backward chain before the ReLU masks, and the ReLU zeros it meets
    up = [None] * c.L
    up[c.L - 1] = (go @ dec.Wout, np.abs(go) @ np.abs(dec.Wout), _grain(go) + _grain(dec.Wout))
    for l in range(c.L - 1, 0, -1):
        G = ex["G"][l]
        up[l - 1] = (G @ dec.W[l], np.abs(G) @ np.abs(dec.W[l]), _grain(G) + gW[l])
    zero = zero_live = total = 0
    for l in range(c.L):
        v, s, m = up[l]
        _assert_sum_exact(f"G_{l} before its mask", s, m)
        z = ex["z"][l]
        zero += int((z == 0).sum())
        zero_live += int(((z == 0) & (v != 0)).sum())
        total += z.size
    assert not relu_zeros or (zero >= 0.01 * total and zero_live > 0), (zero, zero_live, total)
    G0, gx = ex["G"][0], ex["gx"]
    _assert_sum_exact("gx", np.abs(G0) @ np.abs(dec.W[0]), _grain(G0) + gW[0])
    # the feature-gradient scatter: per neural point, the rows (or IDW-weighted queries) naming it
    F, K = c.F, c.K
    idx = inp.idx.reshape(-1)
    if c.wf:
        terms = (np.abs(inp.w)[:, :, None] * np.abs(gx[:, None, :F])).reshape(-1, F)
        m = _grain(inp.w) + _grain(gx[:, :F])
    else:
        terms, m = np.abs(gx[:, :F]), _grain(gx[:, :F])
    acc = torch.zeros(inp.feat.shape[0], F, dtype=torch.float64)
    acc.index_add_(0, torch.from_numpy(idx[idx >= 0]).long(), torch.from_numpy(terms[idx >= 0]))
    _assert_sum_exact("grad_feat", acc.numpy(), m)


# --------------------------------------------------------------------------------------
# GPU side
# --------------------------------------------------------------------------------------
def _ops():
    from pin_slam_b200 import ops

    return ops


def _cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _offset_copy(a, off, fill=None):
    """A contiguous CUDA tensor of a's shape starting `off` floats into a buffer with 4-float sentinel margins on
    both sides (head margin 4 + off floats: 16-byte aligned for off 0, 4 bytes past the grid for off 1)."""
    a = torch.as_tensor(a, dtype=torch.float32)
    buf = torch.full((a.numel() + 8 + off,), SENTINEL, device="cuda")
    t = buf[4 + off: 4 + off + a.numel()].view(a.shape)
    t.copy_(a if fill is None else torch.full_like(a, fill))
    return buf, t


def _map_handle(pts, ori, feat, pgo):
    """A map view with only what K2 reads: nb_points, nb_orient, the feature width."""
    o = _ops()
    n = pts.shape[0]
    zi = lambda *s: torch.zeros(s, dtype=torch.int32, device="cuda")  # noqa: E731
    return o.MapHandle(slot_table=torch.full((64,), -1, dtype=torch.int32, device="cuda"), buffer_size=64, points=pts,
                       ts_create=zi(n), travel_dist=None, global2local=None, nb_points=pts, nb_orient=ori,
                       geo_feat=feat, color_feat=None, certainty=torch.zeros(n, device="cuda"), ts_update=zi(n),
                       probe_dx=zi(1, 3), resolution=1.0, max_valid_dist2=1.0, time_filter=False, cur_ts=0,
                       diff_travel_dist_local=1e9, after_pgo=pgo)


class _K2Run:
    """K2 inputs on the GPU; grad_feat and grad_dec inside sentinel-margined buffers."""

    def __init__(self, c, inp, dec):
        o = _ops()
        self.c = c
        self.feat_buf, self.feat = _offset_copy(torch.from_numpy(inp.feat), c.feat_off)
        self.mh = _map_handle(_cuda(inp.pts), _cuda(inp.ori), self.feat, inp.pgo)
        ws = [_cuda(w) for w in dec.W]
        bs = [None if b is None else _cuda(b) for b in dec.b]
        self.dh = o.DecoderHandle(ws, bs, _cuda(dec.Wout), None if dec.bout is None else _cuda(dec.bout),
                                  out_scale=dec.scale, leaky=dec.leaky, sigmoid_out=dec.sigmoid)
        self.args = (_cuda(inp.q), _cuda(inp.idx, torch.int32), _cuda(inp.w), _cuda(inp.dl))
        self.gf_buf, self.gfeat = _offset_copy(torch.from_numpy(inp.feat), c.gfeat_off, fill=0.0)
        n_par = self.dh.param_count()
        self.gd_buf, self.gdec = _offset_copy(torch.zeros(n_par), 0)

    def call(self, gfeat=None, gdec=None):
        q, idx, w, dl = self.args
        _ops().train_backward(self.mh, self.dh, self.feat, q, idx, w, dl, self.c.wf,
                              self.gfeat if gfeat is None else gfeat, self.gdec if gdec is None else gdec)

    def scratch_call(self):
        """The same launch into fresh zeroed buffers (for the profiler, which may run it more than once)."""
        _, gf = _offset_copy(self.gfeat.cpu(), self.c.gfeat_off, fill=0.0)
        self.call(gf, torch.zeros_like(self.gdec))

    def assert_margins(self):
        for name, buf, t in (("grad_feat", self.gf_buf, self.gfeat), ("grad_dec", self.gd_buf, self.gdec)):
            head = t.data_ptr() - buf.data_ptr()
            assert bool((buf[:head // 4] == SENTINEL).all()), f"K2 wrote before {name}"
            assert bool((buf[head // 4 + t.numel():] == SENTINEL).all()), f"K2 wrote past the end of {name}"


def _assert_equal(name, got, ref):
    got = got.detach().cpu().numpy().astype(np.float64).reshape(ref.shape)
    bad = got != ref
    assert not bad.any(), f"{name}: {int(bad.sum())} / {bad.size} differ, max {np.abs(got - ref).max():.3e}"


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("c", EXACT_CASES, ids=[_case_id(c) for c in EXACT_CASES])
def test_k2_exact_multi_tile(c):
    """K2 on dyadic inputs equals the fp64 autograd reference bit for bit: grad_feat and grad_dec, at >= 2 tiles per
    CTA and at n = 1, qpt - 1, qpt, qpt + 1; a second call doubles both exactly; nothing around them is touched."""
    seed = 100 * c.F + 10 * c.L + c.K
    dec = _exact_decoder(c, seed)
    qpt = _qpt(c)
    n = _multi_tile_n(c, _sm_count())
    n_tiles = (n + qpt - 1) // qpt
    inp = _exact_inputs(c, n, seed + 1)
    gf_ref, gd_ref, ex = _k2_reference(inp, dec, c.wf, torch.float64, keep=True)
    _assert_exact_premise(inp, dec, c, ex)
    del ex
    assert (gd_ref != 0).mean() > 0.2 and (gf_ref[:2] != 0).any(axis=1).all()

    # the persistent grid is at most SMs x (2048 / 128) CTAs, so every CTA runs at least two tiles
    assert n_tiles >= 2 * 16 * _sm_count()
    run = _K2Run(c, inp, dec)
    _, launched = kernels_run(run.scratch_call, tries=5)
    assert any(_kernel(c) + "(" in k for k in launched), sorted(launched)
    run.call()
    torch.cuda.synchronize()
    _assert_equal("grad_feat", run.gfeat, gf_ref)
    _assert_equal("grad_dec", run.gdec, gd_ref)
    run.call()
    torch.cuda.synchronize()
    _assert_equal("grad_feat (second call)", run.gfeat, 2 * gf_ref)
    _assert_equal("grad_dec (second call)", run.gdec, 2 * gd_ref)
    run.assert_margins()

    for ns in sorted({1, qpt - 1, qpt, qpt + 1} - {0}):
        inp = _exact_inputs(c, ns, seed + ns, n_pts=64)
        gf_ref, gd_ref, ex = _k2_reference(inp, dec, c.wf, torch.float64, keep=True)
        _assert_exact_premise(inp, dec, c, ex, relu_zeros=False)  # too few rows with a gradient for the count
        run = _K2Run(c, inp, dec)
        run.call()
        torch.cuda.synchronize()
        _assert_equal(f"grad_feat (n = {ns})", run.gfeat, gf_ref)
        _assert_equal(f"grad_dec (n = {ns})", run.gdec, gd_ref)
        run.assert_margins()


@pytest.mark.gpu
@pytest.mark.parametrize("c", RANDOM_CASES, ids=[_case_id(c) for c in RANDOM_CASES])
def test_k2_random_multi_tile(c):
    """K2 on realistic values at >= 2 tiles per CTA (or at the mapper's batch shape) against fp32 / fp64 autograd,
    within the bounds of tests/helpers.py; ReLU kink rows are allowed here."""
    seed = 1000 + 100 * c.F + 10 * c.L + c.K
    dec = _random_decoder(c, seed)
    n = c.n or _multi_tile_n(c, _sm_count())
    inp = _random_inputs(c, n, seed + 1)
    gf_ref, gd_ref, _ = _k2_reference(inp, dec, c.wf, torch.float32)
    gf64, gd64, _ = _k2_reference(inp, dec, c.wf, torch.float64)
    run = _K2Run(c, inp, dec)
    _, launched = kernels_run(run.scratch_call, tries=5)
    assert any(_kernel(c) + "(" in k for k in launched), sorted(launched)
    run.call()
    torch.cuda.synchronize()
    rows = n if c.wf else n * c.K
    kink = max(8, rows // 20000)
    assert_rel_close(run.gfeat.cpu(), gf_ref, 1e-4, float(np.abs(gf_ref).max()) * 5e-2, gf64, kink_rows=kink)
    assert_decoder_grad_close(run.gdec.cpu(), gd_ref, gd64)
    run.assert_margins()


# --------------------------------------------------------------------------------------
# pinb200_map_iterations against the oracle
# --------------------------------------------------------------------------------------
# name, F, K, wf, L, bs, decimation, loss_weight_on, train_decoder, split training forward
LoopCase = namedtuple("LoopCase", "name F K wf L bs decim lw train_dec split")
LOOP_CASES = [
    LoopCase("kitti", 8, 6, False, 1, 16384, 10, True, True, False),
    LoopCase("kitti-frozen-decoder", 8, 6, False, 1, 16384, 10, True, False, False),
    LoopCase("cfg2", 32, 8, True, 2, 16384, 10, True, True, False),
    LoopCase("kitti-split-forward", 8, 6, False, 1, 28000, 10, True, True, True),
    LoopCase("no-eikonal-no-weights", 8, 6, False, 1, 16384, 0, False, True, False),
]


def _loop_rows(c):
    return c.bs + (6 * ((c.bs + c.decim - 1) // c.decim) if c.decim else 0)


def test_map_loop_case_sizes():
    """No GPU: the split case crosses the training forward's split threshold and the others stay below it."""
    from pin_slam_b200 import ops

    for c in LOOP_CASES:
        assert (_loop_rows(c) >= ops.SPLIT_MIN_QUERIES) == c.split, (c.name, _loop_rows(c))


@pytest.mark.gpu
@pytest.mark.parametrize("c", LOOP_CASES, ids=[c.name for c in LOOP_CASES])
def test_map_iterations_full_batch_vs_oracle(c):
    """Three pinb200_map_iterations steps at full batch size against autograd + torch Adam through the oracle: the
    post-step features and decoder (assert_close_frac), certainty to 1e-4, ts_update exactly, the losses of the last
    iteration, and the kernels the loop launched.  A frozen decoder stays bit-identical with a zero gradient and
    only the features train.  On the KITTI case the same iterations also run in the data-parallel two-call form
    (stages 1 with grad_scale 1/2, the gradient blocks doubled as a 2-rank all-reduce of equal gradients does, then
    stages 2 with first_step = it + 1), which must match the one-call run and the oracle."""
    o = _ops()
    n_iter, P = 3, 60000
    m = synthetic_map(n_surface=40000, seed=20 + c.F, resolution=0.4, buffer_size=200003, feature_dim=c.F,
                      local_radius=14.0, diff_td=3.0)
    dec = po.make_decoder(c.F + 3, 64, c.L, 1, 0.044, seed=7)
    g = torch.Generator().manual_seed(4)
    sigma, weight_e, eik_eps, lr, adam_eps, wd = 0.1, 0.5, 0.02, 0.01, 1e-15, 1e-7
    coord_pool = queries_near(m, P, seed=21)
    label_pool = 0.2 * torch.randn(P, generator=g)
    ts_pool = torch.randint(0, 3, (P,), generator=g, dtype=m.local_point_ts_update.dtype)
    weight_pool = torch.rand(P, generator=g) + 0.5
    index = torch.randint(0, P, (n_iter, c.bs), generator=g)

    mo = m.clone()
    deco = dec.clone()
    feat_o = mo.local_geo_features.requires_grad_(True)
    dparams = deco.tensors()
    if c.train_dec:
        for p in dparams:
            p.requires_grad_(True)
        opt = po.make_adam([dparams, [feat_o]], lr=lr, eps=adam_eps, weight_decay=wd)
    else:
        opt = po.make_adam([[feat_o]], lr=lr, eps=adam_eps, weight_decay=wd)
    for it in range(n_iter):
        i = index[it]
        opt.zero_grad()
        loss, parts = po.mapping_loss(mo, deco, coord_pool[i], label_pool[i], ts_pool[i], weight_pool[i], c.K, c.wf,
                                      sigma, c.lw, weight_e, c.decim, eik_eps, ekional_loss_on=c.decim > 0)
        loss.backward()
        opt.step()
    flat_ref = torch.cat([p.detach().reshape(-1) for p in dparams]).numpy()

    dev = dict(coord_pool=coord_pool.cuda(), label_pool=label_pool.cuda(), ts_pool=ts_pool.to(torch.int32).cuda(),
               weight_pool=weight_pool.cuda())
    flat0 = torch.cat([t.reshape(-1) for t in dec.tensors()]).cuda()

    def state():
        mh = map_handle_from_oracle(m, True)
        flat = flat0.clone()
        ws, bs, off = [], [], 0
        for w, b in dec.hidden:
            ws.append(flat[off:off + w.numel()].view_as(w))
            off += w.numel()
            bs.append(flat[off:off + b.numel()].view_as(b))
            off += b.numel()
        wo = flat[off:off + dec.out[0].numel()].view_as(dec.out[0])
        off += dec.out[0].numel()
        dh = o.DecoderHandle(ws, bs, wo, flat[off:].view_as(dec.out[1]), out_scale=dec.sdf_scale)
        feat = mh.keep["geo_feat"]
        z = lambda t: torch.zeros_like(t)  # noqa: E731
        return dict(mh=mh, dh=dh, feat=feat, dec_flat=flat, grad_feat=z(feat), grad_dec=z(flat), m_feat=z(feat),
                    v_feat=z(feat), m_dec=z(flat), v_dec=z(flat), losses=torch.zeros(2, device="cuda"), work={})

    def run(s, n, idx, **kw):
        o.map_iterations(s["mh"], s["dh"], n, nn_k=c.K, weighted_first=c.wf, index=idx.cuda(), decimation=c.decim,
                         eik_eps=eik_eps, sigma=sigma, weight_e=weight_e, loss_weight_on=c.lw, lr=lr, beta1=0.9,
                         beta2=0.99, eps=adam_eps, weight_decay=wd, train_decoder=c.train_dec,
                         **{k: s[k] for k in ("feat", "dec_flat", "grad_feat", "grad_dec", "m_feat", "v_feat",
                                              "m_dec", "v_dec", "losses", "work")}, **dev, **kw)

    _, launched = kernels_run(lambda: run(state(), 1, index[:1], first_step=1), tries=5)
    ran = {mm.group(0) for k in launched for mm in FAMILY.finditer(k)}
    want = ({"search_kernel<false, false>", f"query_kernel<{c.F}, {str(c.wf).lower()}, true>"} if c.split
            else {f"query_kernel<{c.F}, {str(c.wf).lower()}, false>"})
    assert ran == want | {train_bwd_kernel_name(c.F, c.L)}, sorted(launched)

    s = state()
    run(s, n_iter, index, first_step=1)
    torch.cuda.synchronize()
    results = [s]
    if c.name == "kitti":
        s2 = state()
        for it in range(n_iter):
            run(s2, 1, index[it:it + 1], first_step=it + 1, stages=1, grad_scale=0.5)
            s2["grad_feat"].mul_(2.0)
            s2["grad_dec"].mul_(2.0)
            run(s2, 1, index[it:it + 1], first_step=it + 1, stages=2)
        torch.cuda.synchronize()
        assert_close_frac(s2["feat"].cpu().numpy(), s["feat"].cpu().numpy())
        assert_close_frac(s2["dec_flat"].cpu().numpy(), s["dec_flat"].cpu().numpy())
        results.append(s2)
    for r in results:
        assert_close_frac(r["feat"].cpu().numpy(), feat_o.detach().numpy())
        if c.train_dec:
            assert_close_frac(r["dec_flat"].cpu().numpy(), flat_ref)
        else:
            assert torch.equal(r["dec_flat"], flat0), "a frozen decoder changed"
        assert float(r["grad_dec"].abs().max()) == 0.0 and float(r["grad_feat"].abs().max()) == 0.0
        np.testing.assert_allclose(r["mh"].keep["certainty"].cpu().numpy(), mo.local_point_certainties.numpy(),
                                   rtol=1e-4, atol=1e-4)
        assert np.array_equal(r["mh"].keep["ts_update"].cpu().numpy(), mo.local_point_ts_update.numpy())
    ref_losses = [float(parts["bce"]), float(parts["eikonal"]) if c.decim else 0.0]
    np.testing.assert_allclose(s["losses"].cpu().numpy(), ref_losses, rtol=1e-3, atol=1e-6)


# --------------------------------------------------------------------------------------
# Mapper.mapping with the colour head
# --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_mapper_mapping_with_colour_head_matches_ops():
    """Mapper.mapping on a Replica-config map (colour head on) keeps its gradients in one arena, where the
    colour-feature block starts 4 bytes past a 16-byte boundary (the decoders have 833 parameters), so K2 scatters it
    with scalar atomics.  The same iterations issued through ops on separately allocated, aligned buffers, with the
    same seeds and batch draws, must give the same features, colour features and decoders."""
    from pin_slam_b200 import ops
    from pin_slam_b200.frame_loop import FrameLoop

    n_it = 4
    states = []
    for via_mapper in (True, False):
        torch.manual_seed(0)
        loop = FrameLoop(device="cuda", n_track_iter=4, n_map_iter=4, rgbd=True)
        loop.step(0, map_iters=2)
        mp, npm, cfg = loop.mapper, loop.neural_points, loop.cfg
        if via_mapper:
            flat = mp.sdf_mlp.flat_parameters()
            n_geo = npm.local_geo_features.numel()
            assert mp.color_mlp is not None and cfg.color_on and cfg.weight_i > 0
            assert ((n_geo + flat.numel()) * 4) % 16 == 4, "the colour-feature gradient block is 16-byte aligned"
            torch.manual_seed(7)
            mp.mapping(n_it)
        else:
            torch.manual_seed(7)
            _mapping_through_ops(ops, mp, npm, cfg, max(1, n_it + mp.adaptive_iter_offset))
        states.append([npm.local_geo_features.detach().clone(), npm.local_color_features.detach().clone(),
                       mp.sdf_mlp.flat_parameters().clone(), mp.color_mlp.flat_parameters().clone(),
                       npm.local_point_certainties.clone()])
    for name, a, b in zip(("features", "colour features", "decoder", "colour decoder", "certainty"), *states):
        bad = (a - b).abs() > 2e-5 + 1e-4 * b.abs()  # K2 atomics reorder sums; Adam eps 1e-15 amplifies
        assert bad.float().mean() < 5e-3 and float((a - b).abs().max()) < 5e-2, name


def _mapping_through_ops(ops, mp, npm, cfg, iters):
    """Mapper.mapping's colour-head iteration (utils/mapper.py) written out on plain ops calls, with every gradient
    and Adam moment in its own zero-initialised (16-byte aligned) tensor."""
    feat, cfeat = npm.local_geo_features.data, npm.local_color_features.data
    flat, cflat = mp.sdf_mlp.flat_parameters(), mp.color_mlp.flat_parameters()
    z = torch.zeros_like
    gfeat, mf, vf, gdec, md, vd = z(feat), z(feat), z(feat), z(flat), z(flat), z(flat)
    gcfeat, mcf, vcf, gcdec, mcd, vcd = z(cfeat), z(cfeat), z(cfeat), z(cflat), z(cflat), z(cflat)
    losses, closs = torch.zeros(2, device="cuda"), torch.zeros(1, device="cuda")
    dec_step = cfg.gradient_decimation
    eik_on = cfg.ekional_loss_on and cfg.weight_e > 0
    eps_num = cfg.voxel_size_m * cfg.num_grad_step_ratio
    train_dec = any(p.requires_grad for p in mp.sdf_mlp.parameters())
    train_cdec = any(p.requires_grad for p in mp.color_mlp.parameters())
    batch, work = {}, {}
    for it in range(iters):
        index = mp.draw_batch_index()
        rows, label, ts, weight, color_label, ne = ops.assemble_batch(
            mp.global_coord_pool, mp.sdf_label_pool, mp.time_pool, mp.weight_pool, mp.color_pool, index,
            dec_step if eik_on else 0, eps_num, batch)
        n = index.shape[0]
        out = ops.query_sdf(npm.map_handle(True), mp.sdf_mlp.handle(), rows, nn_k=cfg.query_nn_k,
                            weighted_first=cfg.weighted_first, training_mode=True, training_rows=n, need_grad=False,
                            query_ts=ts.contiguous(), save_knn=True, out=work,
                            color_dec=mp.color_mlp.handle(sigmoid_out=True))
        dl = torch.empty(rows.shape[0], device="cuda")
        ops.mapping_loss(out["sdf"], label, weight, n, ne, mp.sdf_scale, cfg.loss_weight_on,
                         cfg.weight_e if eik_on else 0.0, eps_num, dl, losses)
        ops.train_backward(npm.map_handle(True), mp.sdf_mlp.handle(), feat, rows, out["knn_idx"], out["knn_weight"],
                           dl, cfg.weighted_first, gfeat, gdec)
        n_surf = (label.abs() < cfg.surface_sample_range_m).sum().float().reshape(1)
        dlc = torch.empty((n, mp.color_mlp.out_dim), device="cuda")
        ops.color_loss(out["color"][:n], color_label, label, weight, cfg.surface_sample_range_m, cfg.loss_weight_on,
                       cfg.weight_i, n_surf, dlc, closs)
        ops.train_backward(npm.map_handle(True), mp.color_mlp.handle(sigmoid_out=True), cfeat, rows[:n],
                           out["knn_idx"][:n], out["knn_weight"][:n], dlc, cfg.weighted_first, gcfeat, gcdec)
        if train_dec:
            ops.adam_step(flat, gdec, md, vd, cfg.lr, 0.9, 0.99, cfg.adam_eps, 0.0, it + 1)
        else:
            gdec.zero_()
        ops.adam_step(feat, gfeat, mf, vf, cfg.lr, 0.9, 0.99, cfg.adam_eps, cfg.weight_decay, it + 1)
        if train_cdec:
            ops.adam_step(cflat, gcdec, mcd, vcd, cfg.lr, 0.9, 0.99, cfg.adam_eps, 0.0, it + 1)
        else:
            gcdec.zero_()
        ops.adam_step(cfeat, gcfeat, mcf, vcf, cfg.lr, 0.9, 0.99, cfg.adam_eps, cfg.weight_decay, it + 1)
