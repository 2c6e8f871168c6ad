"""ctypes binding of libpinb200.so (C ABI declared in include/pinb200.h).

The product path has NO fallback: if the shared library is missing or a call
fails, a RuntimeError is raised."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpinb200.so")

MAX_HIDDEN = 4
MAX_K = 8

c_f32p = C.c_void_p
c_i32p = C.c_void_p
c_f64p = C.c_void_p


class MapView(C.Structure):
    _fields_ = [
        ("slot_table", c_i32p), ("buffer_size", C.c_int64), ("points", c_f32p), ("ts_create", c_i32p),
        ("n_global", C.c_int64), ("travel_dist", c_f32p), ("n_travel", C.c_int64), ("global2local", c_i32p),
        ("nb_points", c_f32p), ("nb_orient", c_f32p), ("geo_feat", c_f32p), ("color_feat", c_f32p),
        ("certainty", c_f32p), ("ts_update", c_i32p), ("n_nb", C.c_int64), ("feature_dim", C.c_int32),
        ("probe_dx", c_i32p), ("n_probe", C.c_int32), ("resolution", C.c_float), ("max_valid_dist2", C.c_float),
        ("time_filter", C.c_int32), ("cur_ts", C.c_int32), ("diff_travel_dist_local", C.c_float),
        ("after_pgo", C.c_int32), ("probe_words", C.c_void_p), ("probe_rec", c_f32p), ("probe_gid", c_i32p),
    ]


class DecoderView(C.Structure):
    _fields_ = [
        ("w", c_f32p * MAX_HIDDEN), ("b", c_f32p * MAX_HIDDEN), ("w_out", c_f32p), ("b_out", c_f32p),
        ("n_hidden", C.c_int32), ("hidden_dim", C.c_int32), ("in_dim", C.c_int32), ("out_dim", C.c_int32),
        ("out_scale", C.c_float), ("leaky_relu", C.c_int32), ("sigmoid_out", C.c_int32),
    ]


class QueryOpts(C.Structure):
    _fields_ = [("nn_k", C.c_int32), ("weighted_first", C.c_int32), ("training_mode", C.c_int32),
                ("need_grad", C.c_int32), ("training_rows", C.c_int64), ("transform", c_f64p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64)]


class QueryOut(C.Structure):
    _fields_ = [("sdf", c_f32p), ("grad", c_f32p), ("sdf_std", c_f32p), ("nn_count", c_i32p),
                ("certainty", c_f32p), ("color", c_f32p), ("color_grad", c_f32p), ("knn_idx", c_i32p),
                ("knn_dist2", c_f32p), ("knn_weight", c_f32p), ("knn_gidx", c_i32p), ("xyz", c_f32p)]


class GnOpts(C.Structure):
    _fields_ = [("sdf_label", c_f32p), ("normals", c_f32p), ("color_obs", c_f32p), ("color_channels", C.c_int32),
                ("color_mode", C.c_int32), ("min_nn", C.c_int32), ("min_grad_norm", C.c_float),
                ("max_grad_norm", C.c_float), ("max_sdf_std", C.c_float), ("gm_dist", C.c_float),
                ("gm_grad", C.c_float), ("lm_lambda", C.c_float), ("w_photo", C.c_float), ("sums", c_f64p),
                ("result", c_f64p)]


class MapTrainOpts(C.Structure):
    _fields_ = [("coord_pool", c_f32p), ("label_pool", c_f32p), ("ts_pool", c_i32p), ("weight_pool", c_f32p),
                ("index", C.c_void_p), ("bs", C.c_int64), ("decimation", C.c_int32), ("eik_eps", C.c_float),
                ("sigma", C.c_float), ("weight_e", C.c_float), ("loss_weight_on", C.c_int32), ("lr", C.c_double),
                ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double), ("weight_decay", C.c_double),
                ("train_decoder", C.c_int32), ("first_step", C.c_int32), ("stages", C.c_int32),
                ("grad_scale", C.c_float), ("rows", c_f32p), ("label", c_f32p),
                ("ts", c_i32p), ("weight", c_f32p), ("dloss", c_f32p), ("losses", c_f32p), ("feat", c_f32p),
                ("dec_flat", c_f32p), ("grad_feat", c_f32p), ("grad_dec", c_f32p), ("m_feat", c_f32p),
                ("v_feat", c_f32p), ("m_dec", c_f32p), ("v_dec", c_f32p), ("nccl_comm", C.c_void_p),
                ("reduce_buf", c_f32p), ("reduce_count", C.c_int64), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_int64)]


# name -> (restype, argtypes); every symbol include/pinb200.h declares
SIGNATURES = {
    "pinb200_version": (C.c_int, []),
    "pinb200_last_error": (C.c_char_p, []),
    "pinb200_query_sdf": (C.c_int, [C.POINTER(MapView), C.POINTER(DecoderView), C.POINTER(DecoderView), c_f32p,
                                    c_i32p, C.c_int64, C.POINTER(QueryOpts), C.POINTER(QueryOut), C.c_void_p]),
    "pinb200_query_workspace_bytes": (C.c_int64, [C.c_int64]),
    "pinb200_set_option": (C.c_int, [C.c_char_p, C.c_int64]),
    "pinb200_debug_read": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int64]),
    "pinb200_knn_search": (C.c_int, [C.POINTER(MapView), c_f32p, C.c_int64, C.c_int32, c_i32p, c_i32p, c_f32p, c_f32p,
                                     c_i32p, C.c_void_p]),
    "pinb200_radius_search": (C.c_int, [C.POINTER(MapView), c_f32p, C.c_int64, c_f32p, c_i32p, C.c_void_p]),
    "pinb200_query_certainty": (C.c_int, [C.POINTER(MapView), c_f32p, C.c_int64, c_f32p, C.c_void_p]),
    "pinb200_gather_features": (C.c_int, [C.POINTER(MapView), c_f32p, c_f32p, c_i32p, c_f32p, C.c_int64, C.c_int32,
                                          C.c_int32, c_f32p, C.c_void_p]),
    "pinb200_decoder_param_count": (C.c_int64, [C.POINTER(DecoderView)]),
    "pinb200_train_backward": (C.c_int, [C.POINTER(MapView), C.POINTER(DecoderView), c_f32p, c_f32p, c_i32p, c_f32p,
                                         c_f32p, C.c_int64, C.c_int32, C.c_int32, c_f32p, c_f32p, C.c_void_p]),
    "pinb200_mapping_loss": (C.c_int, [c_f32p, c_f32p, c_f32p, C.c_int64, C.c_int64, C.c_float, C.c_int32,
                                       C.c_float, C.c_float, C.c_float, c_f32p, c_f32p, C.c_void_p]),
    "pinb200_adam_step": (C.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, C.c_int64, C.c_double, C.c_double, C.c_double,
                                    C.c_double, C.c_double, C.c_int32, C.c_void_p]),
    "pinb200_gn_step": (C.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, c_i32p, c_f32p, c_f32p, C.c_int64, C.c_int32,
                                  C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, c_f32p, c_f32p,
                                  c_f32p, C.c_int32, C.c_int32, C.c_float, c_f64p, c_f64p, c_f64p, C.c_void_p]),
    "pinb200_probe_index_words": (C.c_int64, [C.c_int64]),
    "pinb200_probe_index_scratch": (C.c_int64, [C.c_int64]),
    "pinb200_build_probe_index": (C.c_int, [C.POINTER(MapView), C.c_void_p, c_f32p, c_i32p, c_i32p, C.c_void_p]),
    "pinb200_voxel_table_size": (C.c_int64, [C.c_int64]),
    "pinb200_voxel_downsample": (C.c_int, [c_f32p, C.c_int64, C.c_float, c_f32p, C.c_void_p, C.c_void_p, C.c_int64,
                                           c_i32p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pinb200_local_map_scratch": (C.c_int64, [C.c_int64]),
    "pinb200_local_map_select": (C.c_int, [c_f32p, c_i32p, c_i32p, c_f32p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_int32,
                                           C.c_double, C.c_void_p, c_i32p, C.c_void_p, C.c_void_p]),
    "pinb200_local_map_gather": (C.c_int, [c_f32p, c_f32p, c_f32p, c_i32p, C.c_void_p, c_i32p, C.c_int64, C.c_int64,
                                           C.c_int32, C.c_void_p, c_i32p, c_f32p, c_f32p, c_f32p, c_i32p, C.c_void_p]),
    "pinb200_ray_samples": (C.c_int, [c_f32p, c_f32p, C.c_int32, C.c_int64, c_f32p, c_f32p, c_f32p, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_float, C.c_int32,
                                      c_f32p, c_f32p, c_f32p, c_f32p, C.c_void_p]),
    "pinb200_map_grow_scratch": (C.c_int64, [C.c_int64]),
    "pinb200_map_grow": (C.c_int, [c_f32p, C.c_int64, c_i32p, C.c_int64, C.c_float, c_f32p, c_f32p, c_i32p, c_i32p, c_f32p,
                                   C.c_int64, C.c_int64, c_f32p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, c_i32p,
                                   C.c_void_p, C.c_void_p]),
    "pinb200_frame_transform": (C.c_int, [c_f32p, c_f32p, c_i32p, c_i32p, c_f32p, c_f32p, C.c_int64, C.c_int32, C.c_void_p]),
    "pinb200_pool_filter_scratch": (C.c_int64, [C.c_int64]),
    "pinb200_pool_filter": (C.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, c_i32p, c_f32p, C.c_int32, C.c_int64, C.c_int64,
                                      c_f64p, C.c_double, c_f32p, c_f32p, c_f32p, c_f32p, c_i32p, c_f32p, c_i32p,
                                      C.c_void_p, C.c_void_p]),
    "pinb200_assemble_batch": (C.c_int, [c_f32p, c_f32p, c_i32p, c_f32p, c_f32p, C.c_int32, C.c_void_p, C.c_int64,
                                         C.c_int32, C.c_float, c_f32p, c_f32p, c_i32p, c_f32p, c_f32p, C.c_void_p]),
    "pinb200_track_iterations": (C.c_int, [C.POINTER(MapView), C.POINTER(DecoderView), C.POINTER(DecoderView), c_f32p,
                                           C.c_int64, C.POINTER(QueryOpts), C.POINTER(QueryOut), C.POINTER(GnOpts),
                                           C.c_int32, C.c_void_p]),
    "pinb200_map_iterations": (C.c_int, [C.POINTER(MapView), C.POINTER(DecoderView), C.c_int32, C.c_int32,
                                         C.POINTER(MapTrainOpts), C.POINTER(QueryOut), C.c_int32, C.c_void_p]),
    "pinb200_nccl_unique_id": (C.c_int, [C.c_void_p]),
    "pinb200_nccl_init": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "pinb200_nccl_destroy": (C.c_int, [C.c_void_p]),
    "pinb200_color_loss": (C.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, C.c_int64, C.c_int32, C.c_float, C.c_int32,
                                     C.c_float, C.c_float, c_f32p, c_f32p, c_f32p, C.c_void_p]),
}

_lib = None


def load():
    """Load libpinb200.so (once) and declare every prototype.  Raises if missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or pin_slam_b200/csrc/build.sh -- there is no CPU/PyTorch fallback for the hot path")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().pinb200_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (rc={rc}): {msg}")
