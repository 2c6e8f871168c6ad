"""Tensor-facing wrappers of the C ABI: build the plain-C views from CUDA tensors
and launch on torch's current stream.  No arithmetic happens here."""
import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import DecoderView, GnOpts, MapTrainOpts, MapView, QueryOpts, QueryOut

SPLIT_MIN_QUERIES = 32768  # == PINB200_SPLIT_MIN_QUERIES (default; see set_option)
SPLIT_MIN_QUERIES_WF = 1024  # == PINB200_SPLIT_MIN_QUERIES_WF: weighted_first maps on the tensor-core decode
SORT_MIN_QUERIES = 131072  # == PINB200_SORT_MIN_QUERIES: spatial sort before the search launch (see set_option)


def uses_split(n: int, weighted_first: bool, dec=None, training_mode: bool = False) -> bool:
    """Whether a batch of n queries runs as two launches (search, then decode) -- mirrors pinb200_query_sdf."""
    wf = bool(weighted_first) and not training_mode
    if wf and dec is not None:
        v = dec.view
        wf = v.hidden_dim == 64 and 1 <= v.n_hidden <= 2 and (v.in_dim - 3) in (8, 16, 32)
    return n >= (SPLIT_MIN_QUERIES_WF if wf else SPLIT_MIN_QUERIES)


def set_option(name: str, value: int) -> None:
    """Process-wide tunables of the query path (pinb200_set_option): "split_min_queries", "sort_min_queries"
    (0: never sort), "sort_min_queries_color" (calls with a colour head; default 0)."""
    global SPLIT_MIN_QUERIES, SPLIT_MIN_QUERIES_WF
    _lib.check(_lib.load().pinb200_set_option(name.encode(), int(value)), "pinb200_set_option")
    if name == "split_min_queries":
        SPLIT_MIN_QUERIES = int(value) if int(value) > 0 else 32768
        SPLIT_MIN_QUERIES_WF = int(value) if int(value) > 0 else 1024
    elif name == "split_min_queries_wf":
        SPLIT_MIN_QUERIES_WF = int(value) if int(value) > 0 else 1024
_launches = 0  # kernels launched through this module (bench.py reports it as gpu_launches)


def launch_count():
    return _launches


def _count(n=1):
    global _launches
    _launches += n


def _ptr(t: Optional[torch.Tensor], dtype=None):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("pin_slam_b200: the hot path runs on CUDA tensors only (no CPU fallback)")
    if not t.is_contiguous():
        raise RuntimeError("pin_slam_b200: tensor must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError(f"pin_slam_b200: expected {dtype}, got {t.dtype}")
    return t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class MapHandle:
    """A pinb200_map_view plus references that keep its tensors alive."""

    def __init__(self, *, slot_table, buffer_size, points, ts_create, travel_dist, global2local, nb_points,
                 nb_orient, geo_feat, color_feat, certainty, ts_update, probe_dx, resolution, max_valid_dist2,
                 time_filter, cur_ts, diff_travel_dist_local, after_pgo, rec_cache=None):
        self.keep = dict(slot_table=slot_table, points=points, ts_create=ts_create, travel_dist=travel_dist,
                         global2local=global2local, nb_points=nb_points, nb_orient=nb_orient, geo_feat=geo_feat,
                         color_feat=color_feat, certainty=certainty, ts_update=ts_update, probe_dx=probe_dx)
        v = MapView()
        v.slot_table = _ptr(slot_table, torch.int32)
        v.buffer_size = int(buffer_size)
        v.points = _ptr(points, torch.float32)
        v.ts_create = _ptr(ts_create, torch.int32)
        v.n_global = points.shape[0]
        v.travel_dist = _ptr(travel_dist, torch.float32)
        v.n_travel = 0 if travel_dist is None else travel_dist.shape[0]
        v.global2local = _ptr(global2local, torch.int32)
        v.nb_points = _ptr(nb_points, torch.float32)
        v.nb_orient = _ptr(nb_orient, torch.float32)
        v.geo_feat = _ptr(geo_feat, torch.float32)
        v.color_feat = _ptr(color_feat, torch.float32)
        v.certainty = _ptr(certainty, torch.float32)
        v.ts_update = _ptr(ts_update, torch.int32)
        v.n_nb = 0 if nb_points is None else nb_points.shape[0]
        v.feature_dim = 0 if geo_feat is None else geo_feat.shape[1]
        v.probe_dx = _ptr(probe_dx, torch.int32)
        v.n_probe = probe_dx.shape[0]
        v.resolution = float(resolution)
        v.max_valid_dist2 = float(max_valid_dist2)
        v.time_filter = int(bool(time_filter))
        v.cur_ts = int(cur_ts)
        v.diff_travel_dist_local = float(diff_travel_dist_local)
        v.after_pgo = int(bool(after_pgo))
        if time_filter and (travel_dist is None or cur_ts >= travel_dist.shape[0]):
            raise RuntimeError("time filter needs travel_dist[cur_ts]")
        v.probe_words = None
        v.probe_rec = None
        v.probe_gid = None
        # probe index (built lazily by ensure_records); `rec_cache` = (dict, key) of the map owner, where the
        # 12.5 MB word array is kept across handles so that it is not re-allocated every frame
        self._rec_cache = rec_cache
        self._probe = None
        self.view = v
        self.device = points.device

    def ensure_records(self):
        """Build the probe index of this view (pinb200_map_view.probe_*) once per handle: K1 needs it."""
        if self._probe is not None:
            return self
        lib = _lib.load()
        pts = self.keep["points"]
        dev = pts.device
        bsz = self.view.buffer_size
        n_words = int(lib.pinb200_probe_index_words(bsz))
        n_scr = int(lib.pinb200_probe_index_scratch(bsz))
        cached = None if self._rec_cache is None else self._rec_cache[0].get(self._rec_cache[1])
        if cached is not None and cached[0].shape[0] == n_words and cached[0].device == dev:
            words, scratch = cached
        else:
            words = torch.empty((n_words, 2), dtype=torch.int32, device=dev)
            scratch = torch.empty((n_scr,), dtype=torch.int32, device=dev)
            if self._rec_cache is not None:
                self._rec_cache[0][self._rec_cache[1]] = (words, scratch)
        n_g = max(1, pts.shape[0])
        rec = torch.empty((n_g, 4), dtype=torch.float32, device=dev)
        gid = torch.empty((n_g,), dtype=torch.int32, device=dev)
        _lib.check(lib.pinb200_build_probe_index(C.byref(self.view), _ptr(words), _ptr(rec), _ptr(gid), _ptr(scratch),
                                                 _stream()), "pinb200_build_probe_index")
        _count(5)
        self._probe = (words, rec, gid, scratch)
        self.view.probe_words = _ptr(words)
        self.view.probe_rec = _ptr(rec)
        self.view.probe_gid = _ptr(gid)
        return self

    @property
    def n_nb(self):
        return self.view.n_nb

    @property
    def n_probe(self):
        return self.view.n_probe


class DecoderHandle:
    def __init__(self, weights: Sequence[torch.Tensor], biases: Sequence[Optional[torch.Tensor]], w_out, b_out,
                 out_scale=1.0, leaky=False, sigmoid_out=False):
        self.keep = (list(weights), list(biases), w_out, b_out)
        v = DecoderView()
        if not 1 <= len(weights) <= _lib.MAX_HIDDEN:
            raise RuntimeError("decoder: 1..4 hidden layers supported")
        for i, (w, b) in enumerate(zip(weights, biases)):
            v.w[i] = _ptr(w, torch.float32)
            v.b[i] = _ptr(b, torch.float32)
        v.w_out = _ptr(w_out, torch.float32)
        v.b_out = _ptr(b_out, torch.float32)
        v.n_hidden = len(weights)
        v.hidden_dim = weights[0].shape[0]
        v.in_dim = weights[0].shape[1]
        v.out_dim = w_out.shape[0]
        v.out_scale = float(out_scale)
        v.leaky_relu = int(bool(leaky))
        v.sigmoid_out = int(bool(sigmoid_out))
        self.view = v
        self._n_param = None

    def param_count(self):
        """Length of the flat parameter layout (pinb200_decoder_param_count): absent biases have no slot."""
        if self._n_param is None:
            self._n_param = int(_lib.load().pinb200_decoder_param_count(C.byref(self.view)))
        return self._n_param

    def check_flat(self, **tensors):
        """The kernels read and write exactly param_count() floats of every flat decoder vector."""
        n = self.param_count()
        for name, t in tensors.items():
            if t.numel() != n:
                raise RuntimeError(f"pin_slam_b200: {name} holds {t.numel()} floats, the decoder has {n} parameters")


def _query_args(xyz, nn_k, weighted_first, training_mode, need_grad, color_dec, color_grad, transform, save_knn,
                want_xyz, training_rows, out):
    """Output buffers (held in the dict `o`) + the two plain-C structs of a K1 launch."""
    n = xyz.shape[0]
    dev = xyz.device
    o = {} if out is None else out

    def buf(name, shape, dtype=torch.float32):
        t = o.get(name)
        if t is None or tuple(t.shape) != tuple(shape):
            t = torch.empty(shape, dtype=dtype, device=dev)
            o[name] = t
        return t

    qo = QueryOut()
    qo.sdf = _ptr(buf("sdf", (n,)))
    qo.sdf_std = _ptr(buf("sdf_std", (n,)))
    qo.nn_count = _ptr(buf("nn_count", (n,), torch.int32))
    qo.certainty = _ptr(buf("certainty", (n,)))
    if need_grad:
        qo.grad = _ptr(buf("grad", (n, 3)))
    if save_knn or color_dec is not None:
        qo.knn_idx = _ptr(buf("knn_idx", (n, nn_k), torch.int32))
        qo.knn_dist2 = _ptr(buf("knn_dist2", (n, nn_k)))
        qo.knn_weight = _ptr(buf("knn_weight", (n, nn_k)))
        qo.knn_gidx = _ptr(buf("knn_gidx", (n, nn_k), torch.int32))
    if want_xyz:
        qo.xyz = _ptr(buf("xyz", (n, 3)))
    if color_dec is not None:
        cc = color_dec.view.out_dim
        qo.color = _ptr(buf("color", (n, cc)))
        if color_grad:
            qo.color_grad = _ptr(buf("color_grad", (n, cc, 3)))
    ws_ptr, ws_bytes = None, 0
    if n >= (SPLIT_MIN_QUERIES_WF if (weighted_first and not training_mode) else SPLIT_MIN_QUERIES):  # scratch for the two-launch pipeline
        need = int(_lib.load().pinb200_query_workspace_bytes(n))
        ws = o.get("_workspace")
        if ws is None or ws.numel() < need or ws.device != dev:
            ws = o["_workspace"] = torch.empty((need,), dtype=torch.uint8, device=dev)
        ws_ptr, ws_bytes = ws.data_ptr(), ws.numel()
    opts = QueryOpts(int(nn_k), int(bool(weighted_first)), int(bool(training_mode)), int(bool(need_grad)),
                     int(training_rows), _ptr(transform, torch.float64), ws_ptr, ws_bytes)
    return o, qo, opts


def query_sdf(mh: MapHandle, dec: DecoderHandle, xyz: torch.Tensor, *, nn_k: int, weighted_first: bool,
              training_mode: bool = False, need_grad: bool = True, query_ts: Optional[torch.Tensor] = None,
              color_dec: Optional[DecoderHandle] = None, color_grad: bool = False,
              transform: Optional[torch.Tensor] = None, save_knn: bool = False, want_xyz: bool = False,
              training_rows: int = 0, out: Optional[dict] = None):
    """K1.  Returns a dict of freshly allocated (or caller-provided `out`) CUDA tensors."""
    lib = _lib.load()
    mh.ensure_records()
    o, qo, opts = _query_args(xyz, nn_k, weighted_first, training_mode, need_grad, color_dec, color_grad, transform,
                              save_knn, want_xyz, training_rows, out)
    rc = lib.pinb200_query_sdf(C.byref(mh.view), C.byref(dec.view),
                               C.byref(color_dec.view) if color_dec is not None else None,
                               _ptr(xyz, torch.float32), _ptr(query_ts, torch.int32), xyz.shape[0], C.byref(opts),
                               C.byref(qo), _stream())
    _lib.check(rc, "pinb200_query_sdf")
    _count((2 if color_dec is not None else 1) + (1 if uses_split(xyz.shape[0], weighted_first, dec, training_mode) else 0))
    return o


def track_iterations(mh: MapHandle, dec: DecoderHandle, src: torch.Tensor, t_dev: torch.Tensor, n_iter: int, *,
                     nn_k: int, weighted_first: bool, min_nn, min_grad_norm, max_grad_norm, max_sdf_std, gm_dist,
                     gm_grad, lm_lambda, sums, result, sdf_label=None, normals=None, color_dec=None, color_grad=False,
                     color_obs=None, color_mode=0, w_photo=0.0, out: Optional[dict] = None):
    """`n_iter` x (K1 with the device pose `t_dev` + K4 updating it in place) from ONE host call.
    Returns the K1 output dict of the last iteration; `result`/`sums` hold the last K4 outputs."""
    lib = _lib.load()
    mh.ensure_records()
    o, qo, opts = _query_args(src, nn_k, weighted_first, False, True, color_dec, color_grad, t_dev, False, True, 0, out)
    g = GnOpts(_ptr(sdf_label, torch.float32), _ptr(normals, torch.float32),
               _ptr(color_obs, torch.float32) if color_mode else None,
               0 if color_obs is None else int(color_obs.shape[1]), int(color_mode), int(min_nn), float(min_grad_norm),
               float(max_grad_norm), float(max_sdf_std), float(gm_dist or 0.0), float(gm_grad or 0.0), float(lm_lambda),
               float(w_photo), _ptr(sums, torch.float64), _ptr(result, torch.float64))
    rc = lib.pinb200_track_iterations(C.byref(mh.view), C.byref(dec.view),
                                      C.byref(color_dec.view) if color_dec is not None else None,
                                      _ptr(src, torch.float32), src.shape[0], C.byref(opts), C.byref(qo), C.byref(g),
                                      int(n_iter), _stream())
    _lib.check(rc, "pinb200_track_iterations")
    _count(n_iter * ((2 if color_dec is not None else 1) + 2))
    return o


def knn_search(mh: MapHandle, xyz: torch.Tensor, nn_k: int, want_gidx: bool = False):
    lib = _lib.load()
    n, dev = xyz.shape[0], xyz.device
    idx = torch.empty((n, nn_k), dtype=torch.int32, device=dev)
    gidx = torch.empty((n, nn_k), dtype=torch.int32, device=dev) if want_gidx else None
    d2 = torch.empty((n, nn_k), dtype=torch.float32, device=dev)
    w = torch.empty((n, nn_k), dtype=torch.float32, device=dev)
    cnt = torch.empty((n,), dtype=torch.int32, device=dev)
    rc = lib.pinb200_knn_search(C.byref(mh.view), _ptr(xyz, torch.float32), n, nn_k, _ptr(idx), _ptr(gidx), _ptr(d2),
                                _ptr(w), _ptr(cnt), _stream())
    _lib.check(rc, "pinb200_knn_search")
    _count()
    if want_gidx:
        return idx, d2, w, cnt, gidx
    return idx, d2, w, cnt


def radius_search(mh: MapHandle, xyz: torch.Tensor):
    lib = _lib.load()
    n, dev, c = xyz.shape[0], xyz.device, mh.n_probe
    d2 = torch.empty((n, c), dtype=torch.float32, device=dev)
    idx = torch.empty((n, c), dtype=torch.int32, device=dev)
    rc = lib.pinb200_radius_search(C.byref(mh.view), _ptr(xyz, torch.float32), n, _ptr(d2), _ptr(idx), _stream())
    _lib.check(rc, "pinb200_radius_search")
    _count()
    return d2, idx


def query_certainty(mh: MapHandle, xyz: torch.Tensor):
    lib = _lib.load()
    out = torch.empty((xyz.shape[0],), dtype=torch.float32, device=xyz.device)
    rc = lib.pinb200_query_certainty(C.byref(mh.view), _ptr(xyz, torch.float32), xyz.shape[0], _ptr(out), _stream())
    _lib.check(rc, "pinb200_query_certainty")
    _count()
    return out


def gather_features(mh: MapHandle, feat: torch.Tensor, xyz, knn_idx, knn_weight, weighted_first: bool):
    lib = _lib.load()
    n, k = knn_idx.shape
    d = feat.shape[1] + 3
    out = torch.empty((n, d) if weighted_first else (n, k, d), dtype=torch.float32, device=xyz.device)
    rc = lib.pinb200_gather_features(C.byref(mh.view), _ptr(feat, torch.float32), _ptr(xyz, torch.float32),
                                     _ptr(knn_idx, torch.int32), _ptr(knn_weight, torch.float32), n, k,
                                     int(bool(weighted_first)), _ptr(out), _stream())
    _lib.check(rc, "pinb200_gather_features")
    _count()
    return out


def train_backward(mh: MapHandle, dec: DecoderHandle, feat, xyz, knn_idx, knn_weight, dloss_dout, weighted_first,
                   grad_feat, grad_dec):
    lib = _lib.load()
    n, k = knn_idx.shape
    dec.check_flat(grad_dec=grad_dec)
    rc = lib.pinb200_train_backward(C.byref(mh.view), C.byref(dec.view), _ptr(feat, torch.float32),
                                    _ptr(xyz, torch.float32), _ptr(knn_idx, torch.int32),
                                    _ptr(knn_weight, torch.float32), _ptr(dloss_dout, torch.float32), n, k,
                                    int(bool(weighted_first)), _ptr(grad_feat, torch.float32),
                                    _ptr(grad_dec, torch.float32), _stream())
    _lib.check(rc, "pinb200_train_backward")
    _count()


def mapping_loss(sdf, sdf_label, weight, n_main, n_eik, sigma, loss_weight_on, weight_e, eik_eps, dloss, losses,
                 grad_scale: float = 1.0):
    lib = _lib.load()
    rc = lib.pinb200_mapping_loss(_ptr(sdf, torch.float32), _ptr(sdf_label, torch.float32),
                                  _ptr(weight, torch.float32), n_main, n_eik, float(sigma), int(bool(loss_weight_on)),
                                  float(weight_e), float(eik_eps), float(grad_scale), _ptr(dloss, torch.float32),
                                  _ptr(losses, torch.float32), _stream())
    _lib.check(rc, "pinb200_mapping_loss")
    _count()


def adam_step(param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, step):
    lib = _lib.load()
    rc = lib.pinb200_adam_step(_ptr(param, torch.float32), _ptr(grad, torch.float32), _ptr(exp_avg, torch.float32),
                               _ptr(exp_avg_sq, torch.float32), param.numel(), float(lr), float(beta1), float(beta2),
                               float(eps), float(weight_decay), int(step), _stream())
    _lib.check(rc, "pinb200_adam_step")
    _count()


def gn_step(xyz, sdf, grad, sdf_std, nn_count, *, min_nn, min_grad_norm, max_grad_norm, max_sdf_std, gm_dist,
            gm_grad, lm_lambda, sdf_label=None, normals=None, t_inout=None, sums=None, result=None, color_obs=None,
            color_pred=None, color_grad=None, color_mode=0, w_photo=0.0):
    """K4.  Returns (result[32] f64 device tensor, sums[64] f64 device tensor)."""
    lib = _lib.load()
    dev = xyz.device
    if sums is None:
        sums = torch.empty(64, dtype=torch.float64, device=dev)
    if result is None:
        result = torch.empty(32, dtype=torch.float64, device=dev)
    rc = lib.pinb200_gn_step(_ptr(xyz, torch.float32), _ptr(sdf, torch.float32), _ptr(grad, torch.float32),
                             _ptr(sdf_std, torch.float32), _ptr(nn_count, torch.int32),
                             _ptr(sdf_label, torch.float32), _ptr(normals, torch.float32), xyz.shape[0], int(min_nn),
                             float(min_grad_norm), float(max_grad_norm), float(max_sdf_std),
                             float(gm_dist or 0.0), float(gm_grad or 0.0), float(lm_lambda),
                             _ptr(color_obs, torch.float32), _ptr(color_pred, torch.float32),
                             _ptr(color_grad, torch.float32), 0 if color_obs is None else int(color_obs.shape[1]),
                             int(color_mode), float(w_photo), _ptr(sums, torch.float64), _ptr(result, torch.float64), _ptr(t_inout, torch.float64),
                             _stream())
    _lib.check(rc, "pinb200_gn_step")
    _count(2)
    return result, sums


def color_loss(color_pred, color_label, sdf_label, weight, surface_range, loss_weight_on, weight_i, n_surface, dloss,
               loss, grad_scale: float = 1.0):
    lib = _lib.load()
    n, cc = color_pred.shape
    rc = lib.pinb200_color_loss(_ptr(color_pred, torch.float32), _ptr(color_label, torch.float32),
                                _ptr(sdf_label, torch.float32), _ptr(weight, torch.float32), n, cc, float(surface_range),
                                int(bool(loss_weight_on)), float(weight_i), float(grad_scale),
                                _ptr(n_surface, torch.float32), _ptr(dloss, torch.float32), _ptr(loss, torch.float32),
                                _stream())
    _lib.check(rc, "pinb200_color_loss")
    _count()


def assemble_batch(coord_pool, label_pool, ts_pool, weight_pool, color_pool, index, decimation, eps, out: dict):
    """Pool gathers + numerical-gradient rows of one training iteration in one launch; buffers live in `out`."""
    lib = _lib.load()
    n = index.shape[0]
    dev = index.device
    ne = (n + decimation - 1) // decimation if decimation > 0 else 0
    cc = 0 if color_pool is None else color_pool.shape[1]

    def buf(name, shape, dtype=torch.float32):
        t = out.get(name)
        if t is None or tuple(t.shape) != tuple(shape):
            t = torch.empty(shape, dtype=dtype, device=dev)
            out[name] = t
        return t

    rows = buf("rows", (n + 6 * ne, 3))
    label, ts, weight = buf("label", (n,)), buf("ts", (n,), torch.int32), buf("weight", (n,))
    color = buf("color_label", (n, cc)) if cc else None
    rc = lib.pinb200_assemble_batch(_ptr(coord_pool, torch.float32), _ptr(label_pool, torch.float32),
                                    _ptr(ts_pool, torch.int32), _ptr(weight_pool, torch.float32),
                                    _ptr(color_pool, torch.float32), cc, _ptr(index, torch.int64), n, int(decimation),
                                    float(eps), _ptr(rows), _ptr(label), _ptr(ts), _ptr(weight), _ptr(color), _stream())
    _lib.check(rc, "pinb200_assemble_batch")
    _count()
    return rows, label, ts, weight, color, ne


def map_iterations(mh: MapHandle, dec: DecoderHandle, n_iter: int, *, nn_k, weighted_first, coord_pool, label_pool,
                   ts_pool, weight_pool, index, decimation, eik_eps, sigma, weight_e, loss_weight_on, lr, beta1, beta2,
                   eps, weight_decay, train_decoder, first_step, feat, dec_flat, grad_feat, grad_dec, m_feat, v_feat,
                   m_dec, v_dec, losses, work: dict, stages: int = 3, grad_scale: float = 1.0, nccl_comm=None,
                   reduce_buf=None):
    """The geometry-only training loop of Mapper.mapping in ONE host call (pinb200_map_iterations).
    `index` [n_iter, bs] int64 are the pre-drawn batch indices; scratch buffers live in `work`."""
    lib = _lib.load()
    dec.check_flat(dec_flat=dec_flat, grad_dec=grad_dec, m_dec=m_dec, v_dec=v_dec)
    mh.ensure_records()
    bs = index.shape[1]
    dev = index.device
    ne = (bs + decimation - 1) // decimation if decimation > 0 else 0
    rows = bs + 6 * ne

    def buf(name, shape, dtype=torch.float32):
        t = work.get(name)
        if t is None or tuple(t.shape) != tuple(shape):
            t = torch.empty(shape, dtype=dtype, device=dev)
            work[name] = t
        return t

    rows_t = buf("rows", (rows, 3))
    _, qo, qopts = _query_args(rows_t, nn_k, weighted_first, True, False, None, False, None, True, False, bs, work)
    t = MapTrainOpts()
    t.coord_pool, t.label_pool = _ptr(coord_pool, torch.float32), _ptr(label_pool, torch.float32)
    t.ts_pool, t.weight_pool = _ptr(ts_pool, torch.int32), _ptr(weight_pool, torch.float32)
    t.index, t.bs, t.decimation, t.eik_eps = _ptr(index, torch.int64), bs, int(decimation), float(eik_eps)
    t.sigma, t.weight_e, t.loss_weight_on = float(sigma), float(weight_e), int(bool(loss_weight_on))
    t.lr, t.beta1, t.beta2, t.eps, t.weight_decay = float(lr), float(beta1), float(beta2), float(eps), float(weight_decay)
    t.train_decoder, t.first_step = int(bool(train_decoder)), int(first_step)
    t.stages, t.grad_scale = int(stages), float(grad_scale)
    t.workspace, t.workspace_bytes = qopts.workspace, qopts.workspace_bytes  # the split training forward's scratch
    t.rows = _ptr(rows_t)
    t.label, t.ts, t.weight = _ptr(buf("label", (bs,))), _ptr(buf("ts", (bs,), torch.int32)), _ptr(buf("weight", (bs,)))
    t.dloss, t.losses = _ptr(buf("dl", (rows,))), _ptr(losses, torch.float32)
    t.feat, t.dec_flat = _ptr(feat, torch.float32), _ptr(dec_flat, torch.float32)
    t.grad_feat, t.grad_dec = _ptr(grad_feat, torch.float32), _ptr(grad_dec, torch.float32)
    t.m_feat, t.v_feat = _ptr(m_feat, torch.float32), _ptr(v_feat, torch.float32)
    t.m_dec, t.v_dec = _ptr(m_dec, torch.float32), _ptr(v_dec, torch.float32)
    if nccl_comm is not None:
        t.nccl_comm, t.reduce_buf, t.reduce_count = nccl_comm.handle, _ptr(reduce_buf, torch.float32), reduce_buf.numel()
    rc = lib.pinb200_map_iterations(C.byref(mh.view), C.byref(dec.view), int(nn_k), int(bool(weighted_first)),
                                    C.byref(t), C.byref(qo), int(n_iter), _stream())
    _lib.check(rc, "pinb200_map_iterations")
    _count(n_iter * ((4 if stages & 1 else 0) + (2 if stages & 2 else 0)))


def voxel_downsample(points: torch.Tensor, voxel_size: float, value: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Index of the winning point of every occupied voxel, ascending voxel key (pinb200_voxel_downsample + a sort
    of the few winners).  One host synchronisation (the voxel count), like the reference's torch.unique."""
    lib = _lib.load()
    pts = points.contiguous()
    n, dev = pts.shape[0], pts.device
    if n == 0:
        return torch.empty((0,), dtype=torch.int64, device=dev)
    tsz = int(lib.pinb200_voxel_table_size(n))
    ws = torch.empty((2 * tsz,), dtype=torch.int64, device=dev)
    scal = torch.empty((8,), dtype=torch.int32, device=dev)
    outs = torch.empty((2, n), dtype=torch.int64, device=dev)
    val = None if value is None else value.to(torch.float32).contiguous()
    rc = lib.pinb200_voxel_downsample(_ptr(pts, torch.float32), n, float(voxel_size), _ptr(val, torch.float32),
                                      ws.data_ptr(), ws.data_ptr() + 8 * tsz, tsz, _ptr(scal), outs[0].data_ptr(),
                                      outs[1].data_ptr(), _stream())
    _lib.check(rc, "pinb200_voxel_downsample")
    _count(3)
    m = int(scal[7].item())
    order = torch.argsort(outs[0, :m])
    return outs[1, :m][order]


class NcclComm:
    """A NCCL communicator owned by libpinb200 (pinb200_nccl_init) over the ranks of the default torch.distributed
    process group, which is only used to hand the 128-byte unique id from rank 0 to the others."""

    _instance = None

    def __init__(self, device):
        import torch.distributed as dist

        lib = _lib.load()
        world, rank = dist.get_world_size(), dist.get_rank()
        uid = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            buf = (C.c_uint8 * 128)()
            _lib.check(lib.pinb200_nccl_unique_id(C.cast(buf, C.c_void_p)), "pinb200_nccl_unique_id")
            uid = torch.tensor(list(buf), dtype=torch.uint8)
        uid = uid.to(device) if dist.get_backend() == "nccl" else uid
        dist.broadcast(uid, src=0)
        raw = (C.c_uint8 * 128)(*uid.cpu().tolist())
        comm = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(lib.pinb200_nccl_init(C.cast(raw, C.c_void_p), world, rank, C.byref(comm)), "pinb200_nccl_init")
        self.handle, self.world, self.rank, self.device = comm, world, rank, torch.device(device)

    @classmethod
    def get(cls, device):
        """One communicator per process (one process per GPU)."""
        if cls._instance is None or cls._instance.device != torch.device(device):
            cls._instance = cls(device)
        return cls._instance


def frame_transform(xyz: torch.Tensor, ts_a: torch.Tensor, pose_diff: torch.Tensor, quat: Optional[torch.Tensor] = None,
                    dquat: Optional[torch.Tensor] = None, ts_b: Optional[torch.Tensor] = None) -> None:
    """In place: xyz_i <- R_t xyz_i + t_t (and quat_i <- dquat_t (x) quat_i) with t = the frame of row i
    (pinb200_frame_transform; adjust_map / transform_data_pool of the reference)."""
    tf = pose_diff[:, :3, :].to(torch.float32).contiguous()
    rc = _lib.load().pinb200_frame_transform(_ptr(xyz, torch.float32), _ptr(quat, torch.float32), _ptr(ts_a, torch.int32),
                                             _ptr(ts_b, torch.int32), _ptr(tf, torch.float32),
                                             _ptr(None if dquat is None else dquat.to(torch.float32).contiguous(), torch.float32),
                                             xyz.shape[0], tf.shape[0], _stream())
    _lib.check(rc, "pinb200_frame_transform")
    _count()


def map_grow(cand: torch.Tensor, table: torch.Tensor, resolution: float, points, orient, ts_create, ts_update, certainty,
             n_points: int, travel_dist, cur_ts: int, grow_all: bool, temporal_on: bool, diff_travel: float, scratch,
             n_new: torch.Tensor) -> None:
    """pinb200_map_grow: append the candidates that pass the reference's growth test to the arenas (rows n_points..),
    update the hash table; `n_new` (device int64[1]) receives the count."""
    lib = _lib.load()
    n = cand.shape[0]
    need = int(lib.pinb200_map_grow_scratch(n))
    if scratch.numel() < need:
        raise RuntimeError("map_grow: scratch too small")
    rc = lib.pinb200_map_grow(_ptr(cand, torch.float32), n, _ptr(table, torch.int32), table.shape[0], float(resolution),
                              _ptr(points, torch.float32), _ptr(orient, torch.float32), _ptr(ts_create, torch.int32),
                              _ptr(ts_update, torch.int32), _ptr(certainty, torch.float32), int(n_points), points.shape[0],
                              _ptr(travel_dist, torch.float32), int(cur_ts), int(bool(grow_all)), int(bool(temporal_on)),
                              float(diff_travel), float(3 * resolution**2), _ptr(scratch, torch.int32), n_new.data_ptr(),
                              _stream())
    _lib.check(rc, "pinb200_map_grow")
    _count(4)


def ray_samples(points, colors, z_surf, u_front, u_behind, ns, nf, nb, sigma, begin_ratio, end_dist, max_range,
                dist_weight_on, dist_weight_scale, behind_dropoff_on):
    """pinb200_ray_samples: (coord [n*total,3], label, weight, color or None) in ray-major order."""
    n, dev = points.shape[0], points.device
    total = 1 + ns + nf + nb
    coord = torch.empty((n * total, 3), dtype=torch.float32, device=dev)
    label = torch.empty((n * total,), dtype=torch.float32, device=dev)
    weight = torch.empty((n * total,), dtype=torch.float32, device=dev)
    color = None if colors is None else torch.empty((n * total, colors.shape[1]), dtype=torch.float32, device=dev)
    rc = _lib.load().pinb200_ray_samples(_ptr(points, torch.float32), _ptr(colors, torch.float32),
                                         0 if colors is None else colors.shape[1], n, _ptr(z_surf, torch.float32),
                                         _ptr(u_front, torch.float32), _ptr(u_behind, torch.float32), int(ns), int(nf), int(nb),
                                         float(sigma), float(begin_ratio), float(end_dist), float(max_range),
                                         int(bool(dist_weight_on)), float(dist_weight_scale), int(bool(behind_dropoff_on)),
                                         _ptr(coord), _ptr(label), _ptr(weight), _ptr(color), _stream())
    _lib.check(rc, "pinb200_ray_samples")
    _count()
    return coord, label, weight, color


def local_map_select(points, ts_create, ts_update, travel_dist, cur_ts, temporal_on, use_mid_ts, use_travel_dist,
                     diff_ts_local, reboot_map, reboot_ts, diff_travel, sensor_pos, radius2, local_mask, scratch, counts):
    """pinb200_local_map_select: keep flags -> local_mask [n+1] (bool), counts = {recent, n_local} (device int64[2])."""
    if sensor_pos.dtype not in (torch.float32, torch.float64) or not sensor_pos.is_cuda:
        raise RuntimeError("local_map_select: sensor position must be a float32 / float64 CUDA tensor")
    rc = _lib.load().pinb200_local_map_select(
        _ptr(points, torch.float32), _ptr(ts_create, torch.int32), _ptr(ts_update, torch.int32),
        _ptr(travel_dist, torch.float32), points.shape[0], int(cur_ts), int(bool(temporal_on)), int(bool(use_mid_ts)),
        int(bool(use_travel_dist)), int(diff_ts_local), int(bool(reboot_map)), int(reboot_ts), float(diff_travel),
        sensor_pos.contiguous().data_ptr(), int(sensor_pos.dtype == torch.float64), float(radius2), local_mask.data_ptr(),
        _ptr(scratch, torch.int32), counts.data_ptr(), _stream())
    _lib.check(rc, "pinb200_local_map_select")
    _count(3)


def local_map_gather(points, orient, certainty, ts_update, local_mask, scratch, n_local, miss, idx_pad, g2l, l_points,
                     l_orient, l_cert, l_ts):
    rc = _lib.load().pinb200_local_map_gather(
        _ptr(points, torch.float32), _ptr(orient, torch.float32), _ptr(certainty, torch.float32),
        _ptr(ts_update, torch.int32), local_mask.data_ptr(), _ptr(scratch, torch.int32), points.shape[0], int(n_local),
        int(miss), idx_pad.data_ptr(), _ptr(g2l, torch.int32), _ptr(l_points, torch.float32), _ptr(l_orient, torch.float32),
        _ptr(l_cert, torch.float32), _ptr(l_ts, torch.int32), _stream())
    _lib.check(rc, "pinb200_local_map_gather")
    _count()
