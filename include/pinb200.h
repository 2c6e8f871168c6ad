/*
 * pinb200.h -- C ABI of the H100-native (sm_90a) PIN-SLAM hot path.
 *
 * The reference (PRBonn/PIN_SLAM) is 100 % Python/PyTorch and has no native
 * boundary of its own; the boundary it *does* have for this path is the Python
 * method surface of model/neural_points.py::NeuralPoints and
 * model/decoder.py::Decoder (SURVEY.md section 8b).  The entry points below are
 * what a ctypes binding inside those methods calls (INTEGRATION.md shows the
 * stub); each one names the reference code it replaces (file:line relative to
 * the reference checkout).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless stated otherwise; the caller
 *    (PyTorch) owns every buffer, outputs are pre-allocated by the caller;
 *  - all floating data is fp32, ids are int32 (the library keeps int32 mirrors
 *    of the reference's int64 `buffer_pt_index` / `global2local`), timestamps
 *    int32, the optional rigid transform is fp64 (poses are fp64 in the
 *    reference, utils/config.py:316);
 *  - `stream` is a cudaStream_t passed as void*; calls are stream-ordered and
 *    never synchronise;
 *  - return value 0 = ok, negative = error (pinb200_last_error() has the text);
 *    no global mutable state apart from that thread-local error string.
 */
#ifndef PINB200_H
#define PINB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PINB200_VERSION 200 /* round 2: probe index (probe_words / probe_rec / probe_gid) replaces search_rec */
#define PINB200_MAX_HIDDEN_LAYERS 4
#define PINB200_MAX_K 8 /* neighbours kept in registers by the fused search; the reference uses 6 (default) / 8 */

#define PINB200_OK 0
#define PINB200_ERR_BAD_ARG (-1)
#define PINB200_ERR_UNSUPPORTED (-2)
#define PINB200_ERR_CUDA (-3)

#define PINB200_REC_REMAP (1 << 30) /* flag bit of the id word of a probe record, see pinb200_map_view.probe_rec */

/* State of a neural point map as the kernels see it.
 * Mirrors NeuralPoints' tensors, model/neural_points.py:82-136. */
typedef struct pinb200_map_view {
  /* voxel hash over the GLOBAL map */
  const int32_t* slot_table;   /* [buffer_size] hash slot -> global point id, -1 empty   (buffer_pt_index, :88) */
  int64_t buffer_size;         /* must be < 2^31 */
  const float* points;         /* [n_global,3] neural_points (:92) */
  const int32_t* ts_create;    /* [n_global] point_ts_create (:112) */
  int64_t n_global;
  const float* travel_dist;    /* [n_travel] travel_dist (:77), NULL if !time_filter */
  int64_t n_travel;
  const int32_t* global2local; /* [n_global+1] (:498-507) or NULL => query the global arrays (query_locally=False) */
  /* arrays of the index space being queried: local_* if global2local != NULL, else the global ones */
  const float* nb_points;      /* [n_nb,3] */
  const float* nb_orient;      /* [n_nb,4] wxyz quaternions; may be NULL when !after_pgo */
  const float* geo_feat;       /* [n_nb+1,F] last row = padding */
  const float* color_feat;     /* [n_nb+1,F] or NULL */
  float* certainty;            /* [n_nb]  read; atomically += IDW weight in training mode (:691) */
  int32_t* ts_update;          /* [n_nb]  atomic max with the query ts in training mode (:699); may be NULL */
  int64_t n_nb;
  int32_t feature_dim;         /* F */
  /* search neighbourhood, set_search_neighborhood (:910-947) */
  const int32_t* probe_dx;     /* [n_probe,3] integer cell offsets (neighbor_dx) */
  int32_t n_probe;             /* C */
  float resolution;            /* voxel_size_m */
  float max_valid_dist2;       /* 3*((n+1)*res)^2 */
  /* temporal (travel-distance) window, :982-988 */
  int32_t time_filter;         /* temporal_local_map_on && query_locally */
  int32_t cur_ts;
  float diff_travel_dist_local;
  int32_t after_pgo;           /* rotate neighbour vectors by the point quaternion (:645) */
  /* Probe index (built by pinb200_build_probe_index): a succinct rank structure holding the ANSWERS
   * of the hash table in L2-resident form.  A probe of the fused query reads one 8-byte word and, on a hit, one
   * 16-byte record, both from arrays of a few MB, instead of walking buffer_pt_index -> neural_points /
   * point_ts_create -> travel_dist / global2local (model/neural_points.py:963-999,573) in a table of several
   * hundred MB; the age / local-map tests are folded in when the index is built.
   *   probe_words [ceil(buffer_size/32), 2] u32 = { occupancy bits of 32 consecutive slots, set bits before the word };
   *               bit s is set iff slot s is owned by a point this view can return (id >= 0, inside the
   *               travel-distance window when time_filter)
   *   probe_rec   [n_rec, 4] f32 = { x, y, z, bit-cast int32 id } in slot (rank) order; id = global2local[i] (or i),
   *               bit 30 (PINB200_REC_REMAP) set when nb_points[id] is a different point than points[i] (the
   *               reference's global2local fill value maps points outside the local map to local id 1,
   *               model/neural_points.py:498)
   *   probe_gid   [n_rec] i32 = global ids of the same points
   * Required by pinb200_query_sdf / track_iterations / map_iterations (K1); the search-only entry points
   * (knn_search, radius_search, query_certainty) read the separate arrays. */
  const uint32_t* probe_words;
  const float* probe_rec;
  const int32_t* probe_gid;
} pinb200_map_view;

/* Weights of one Decoder (model/decoder.py:43-51), torch nn.Linear layout. */
typedef struct pinb200_decoder_view {
  const float* w[PINB200_MAX_HIDDEN_LAYERS]; /* w[l]: [hidden_dim, in_l] row-major; in_0 = in_dim, in_l = hidden_dim */
  const float* b[PINB200_MAX_HIDDEN_LAYERS]; /* b[l]: [hidden_dim] or NULL (mlp_bias_on False) */
  const float* w_out;                        /* [out_dim, hidden_dim] */
  const float* b_out;                        /* [out_dim] or NULL */
  int32_t n_hidden;                          /* hidden_level */
  int32_t hidden_dim;
  int32_t in_dim;                            /* feature_dim + 3 (positional encoding off) */
  int32_t out_dim;
  float out_scale;                           /* sdf_scale (decoder.py:54-56); 1 for colour */
  int32_t leaky_relu;                        /* mlp_leaky_relu */
  int32_t sigmoid_out;                       /* 0: out*out_scale (Decoder.sdf), 1: sigmoid(out) (Decoder.regress_color) */
} pinb200_decoder_view;

typedef struct pinb200_query_opts {
  int32_t nn_k;             /* config.query_nn_k */
  int32_t weighted_first;   /* config.weighted_first */
  int32_t training_mode;    /* certainty / ts scatter side effects (:685-710) */
  int32_t need_grad;        /* also produce d sdf / d query (replaces tools.py:247 autograd.grad) */
  int64_t training_rows;    /* side effects only for the first training_rows queries (0 = all); the numerical-
                               gradient rows of a training batch follow the samples and are inference-mode
                               (mapper.py:941) */
  const double* transform;  /* optional device ptr, 4x4 row-major fp64: q = T*p evaluated in fp32 (tools.py:534-553) */
  void* workspace;          /* optional device scratch of >= pinb200_query_workspace_bytes(N) bytes.  With it, batches
                               of >= PINB200_SPLIT_MIN_QUERIES (weighted_first: _WF) queries run as two launches (neighbour search at high
                               occupancy, then gather + decoder on wgmma tiles); without it, or for small batches,
                               one fused launch.  The neighbour search is bit-identical either way; the decoder
                               outputs agree within the 3xTF32 bound (different accumulation order). */
  int64_t workspace_bytes;
} pinb200_query_opts;

#define PINB200_SPLIT_MIN_QUERIES 32768   /* decode-every-neighbour maps */
#define PINB200_SPLIT_MIN_QUERIES_WF 1024 /* weighted_first maps whose decoder runs on the wgmma kernel (hidden 64, 1-2 layers,
                                             F in {8,16,32}): the two-launch pipeline is faster from ~1 k queries on */
#define PINB200_SORT_MIN_QUERIES 81920
int64_t pinb200_query_workspace_bytes(int64_t n_queries);
/* Run-time tunables of the query path (process-wide; for tests and A/B measurements):
     "split_min_queries"  batch size from which the two-launch pipeline is used, both kinds of map (<= 0 restores the
                          defaults PINB200_SPLIT_MIN_QUERIES / PINB200_SPLIT_MIN_QUERIES_WF)
     "split_min_queries_wf"  the same for weighted_first maps only
     "sort_min_queries"   batch size from which inference batches of the two-launch pipeline whose decodes all run on
                          wsq_decode_kernel are sorted spatially (Morton order of their cells) before the neighbour
                          search; 0: never (default PINB200_SORT_MIN_QUERIES).  The outputs are the same either way.
     "sort_min_queries_color"  the same for calls with a colour head (default 0: never; the dense RGB-D query comes
                          in pixel order, already coherent)
     "ws_profile"         1: wsq_decode_kernel records per-warp phase cycle counters (pinb200_debug_read)
   The reference has no equivalent: its decode is model/decoder.py:61-85 + autograd (utils/tools.py:247-260). */
int pinb200_set_option(const char* name, int64_t value);
/* Diagnostics.  "ws_profile": after pinb200_set_option("ws_profile", 1), every wsq_decode_kernel launch records per-warp
   cycle counters; this copies them to `host_out` as uint64 [132 CTAs][16 warps][8 phases] (count = elements). */
int pinb200_debug_read(const char* what, void* host_out, int64_t count);

/* Outputs of the fused query; any pointer may be NULL to skip that output. */
typedef struct pinb200_query_out {
  float* sdf;          /* [N]   IDW-combined SDF prediction in metres */
  float* grad;         /* [N,3] d sdf / d q (w.r.t. the transformed point when `transform` is set) */
  float* sdf_std;      /* [N]   IDW std of the per-neighbour SDFs (0 when weighted_first; tracker.py:317-323) */
  int32_t* nn_count;   /* [N]   valid probes before top-K (:577) */
  float* certainty;    /* [N]   IDW-averaged point certainty (:714) */
  float* color;        /* [N,Cc] sigmoid colour head, needs color decoder */
  float* color_grad;   /* [N,Cc,3] */
  int32_t* knn_idx;    /* [N,K] ids in the queried index space, -1 invalid, ascending distance */
  float* knn_dist2;    /* [N,K] squared distances (9e3 for invalid, :583) */
  float* knn_weight;   /* [N,K] normalised IDW weights (:667-683) */
  int32_t* knn_gidx;   /* [N,K] ids of the same neighbours in the GLOBAL arrays (== knn_idx when global2local is NULL) */
  float* xyz;          /* [N,3] the (transformed) query points actually used */
} pinb200_query_out;

int pinb200_version(void);
const char* pinb200_last_error(void);

/* K1 -- fused voxel-hash kNN + IDW interpolation + decoder MLP (+ analytic
 * gradient).  Replaces, in ONE launch:
 *   NeuralPoints.radius_neighborhood_search  model/neural_points.py:950-1009
 *   NeuralPoints.query_feature               model/neural_points.py:530-746
 *   Decoder.mlp / sdf / regress_color        model/decoder.py:61-85,112
 *   get_gradient (autograd.grad)             utils/tools.py:247-260
 *   the IDW mean/std over K                  utils/tracker.py:313-328, utils/mapper.py:945-952
 * color_dec may be NULL.  query_ts may be NULL. */
int pinb200_query_sdf(const pinb200_map_view* map, const pinb200_decoder_view* sdf_dec,
                      const pinb200_decoder_view* color_dec, const float* query_xyz,
                      const int32_t* query_ts, int64_t n, const pinb200_query_opts* opts,
                      const pinb200_query_out* out, void* stream);

/* Search only (no decoder): top-K ids / distances / weights / nn_count.
 * model/neural_points.py:562-589,665-683. */
int pinb200_knn_search(const pinb200_map_view* map, const float* query_xyz, int64_t n, int32_t nn_k,
                       int32_t* knn_idx, int32_t* knn_gidx, float* knn_dist2, float* knn_weight,
                       int32_t* nn_count, void* stream);

/* All-probe form of the radius search: dist2 [N,C] and GLOBAL ids [N,C] exactly
 * as NeuralPoints.radius_neighborhood_search returns them (:950-1009). */
int pinb200_radius_search(const pinb200_map_view* map, const float* query_xyz, int64_t n,
                          float* dist2, int32_t* idx, void* stream);

/* NeuralPoints.query_certainty (:1011-1032): max certainty over the probed
 * cells, global arrays (map->global2local must be NULL, time_filter 0). */
int pinb200_query_certainty(const pinb200_map_view* map, const float* query_xyz, int64_t n,
                            float* out_certainty, void* stream);

/* Materialise query_feature's per-neighbour feature vectors from saved kNN ids
 * (compat path for callers that index the features, e.g. utils/mesher.py:127):
 * out [N,K,F+3] (weighted_first=0) or [N,F+3] (weighted_first=1). `feat` is
 * map->geo_feat or map->color_feat. model/neural_points.py:597-663,722-731. */
int pinb200_gather_features(const pinb200_map_view* map, const float* feat, const float* query_xyz,
                            const int32_t* knn_idx, const float* knn_weight, int64_t n, int32_t nn_k,
                            int32_t weighted_first, float* out, void* stream);

/* Flat layout of decoder gradients / Adam state used by K2/K3:
 * [w0 | b0 | w1 | b1 | ... | w_out | b_out], each row-major as in the view.  A bias that is NULL in the view
 * (mlp_bias_on False) has no block: a decoder without biases is [w0 | w1 | ... | w_out], which is what
 * Decoder.flat_parameters() builds.  The count is of the blocks present. */
int64_t pinb200_decoder_param_count(const pinb200_decoder_view* dec);

/* K2 -- backward of one map-training batch.  Given the saved kNN ids/weights of
 * the forward (pinb200_query_sdf with training_mode=1) and d loss / d sdf per
 * query row, recomputes the decoder activations and accumulates
 *   grad_feat [n_nb+1,F]  += d loss / d local_geo_features   (atomic scatter)
 *   grad_dec  [param_count] += d loss / d decoder parameters (block-reduced, then atomic)
 * Replaces loss.backward() for the SDF branch, utils/mapper.py:816-817
 * (autograd reverse pass through neural_points.py:597-731 and decoder.py:61-85). */
int pinb200_train_backward(const pinb200_map_view* map, const pinb200_decoder_view* dec,
                           const float* feat, const float* query_xyz, const int32_t* knn_idx,
                           const float* knn_weight, const float* dloss_dout, int64_t n, int32_t nn_k,
                           int32_t weighted_first, float* grad_feat, float* grad_dec, void* stream);

/* Loss heads of Mapper.mapping (utils/mapper.py:728-780, utils/loss.py:45-63):
 * BCE-with-logits on the first n_main rows, Eikonal on the 6*n_eik numerical-
 * gradient rows laid out [x+ | x- | y+ | y- | z+ | z-] after them
 * (mapper.py:1002-1014).  Writes d loss / d sdf for every row (of the total loss
 * bce + weight_e * eikonal, times grad_scale = 1/world_size when the batch is sharded over GPUs and the
 * gradients are summed by an all-reduce) and losses[0]=bce, [1]=eikonal (unweighted). */
int pinb200_mapping_loss(const float* sdf, const float* sdf_label, const float* weight, int64_t n_main,
                         int64_t n_eik, float sigma, int32_t loss_weight_on, float weight_e,
                         float eik_eps, float grad_scale, float* dloss_dsdf, float* losses, void* stream);

/* K3 -- Adam step, arithmetic of torch.optim.Adam (betas .9/.99, no amsgrad)
 * as set up by utils/tools.py:153-203; `step` is the 1-based step count.
 * Zeroes `grad` after use (opt.zero_grad folded in). */
int pinb200_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                      double lr, double beta1, double beta2, double eps, double weight_decay, int32_t step,
                      void* stream);

/* K4 -- registration: validity mask, Geman-McClure weights, and the 6x6 normal
 * equations of point-to-implicit registration accumulated in one pass, then
 * solved on device.  Replaces utils/tracker.py:409-524 (registration_step),
 * :652-679 (implicit_reg) and :699-744 (implicit_color_reg).  Inputs are per source point.
 *  colour (all three NULL when unused): color_obs [N,Cc] measured colours, color_pred [N,Cc] and
 *    color_grad [N,Cc,3] from the colour head; Cc == 3 is converted to intensity
 *    0.299 R + 0.587 G + 0.114 B (utils/tools.py:408); color_mode 1 = consistency weight
 *    exp(-mean|obs-pred|) on every point (tracker.py:509-514), 2 = photometric term
 *    N += w_photo J_c^T W J_c, g += w_photo (-J_c^T W r_c) (tracker.py:720-730)
 *  sums [64] fp64 workspace/outputs (zeroed by the call):
 *    [0..35] J^T W J (row-major 6x6, unnormalised w, colour term included), [36..41] -J^T W r,
 *    [42] sum w, [43] sum |r|, [44] valid count, [45] sum w r^2, [46] sum |r_colour|
 *  result [32] fp64: [0..15] delta T (4x4 row-major), [16] valid count,
 *    [17] mean |r| in cm, [18..20] eigenvalues of the normalised N[3:,3:], [21] mean(w r^2),
 *    [22..27] normalised g, [28] mean |r_colour|
 *  If t_inout != NULL (device 4x4 fp64) it is updated in place: T <- delta_T @ T
 *  (tracker.py:147). */
int pinb200_gn_step(const float* xyz, const float* sdf, const float* grad, const float* sdf_std,
                    const int32_t* nn_count, const float* sdf_label, const float* normals, int64_t n,
                    int32_t min_nn, float min_grad_norm, float max_grad_norm, float max_sdf_std,
                    float gm_dist, float gm_grad, float lm_lambda, const float* color_obs,
                    const float* color_pred, const float* color_grad, int32_t color_channels,
                    int32_t color_mode, float w_photo, double* sums, double* result,
                    double* t_inout, void* stream);

/* Parameters of pinb200_gn_step as one struct (same meaning), for pinb200_track_iterations. */
typedef struct pinb200_gn_opts {
  const float* sdf_label;  /* [N] or NULL */
  const float* normals;    /* [N,3] or NULL */
  const float* color_obs;  /* [N,Cc] or NULL */
  int32_t color_channels;
  int32_t color_mode;
  int32_t min_nn;
  float min_grad_norm;
  float max_grad_norm;
  float max_sdf_std;
  float gm_dist;
  float gm_grad;
  float lm_lambda;
  float w_photo;
  double* sums;   /* [64] */
  double* result; /* [32] */
} pinb200_gn_opts;

/* `n_iter` Gauss-Newton iterations of the tracker loop (utils/tracker.py:104-176) issued by ONE host call:
 * each iteration = pinb200_query_sdf (opts->transform must be the device pose T, want xyz/grad outputs) followed by
 * pinb200_gn_step on its outputs with t_inout = opts->transform, so the pose never leaves the device.
 * With n_iter == 1 this is one iteration of the reference loop (the caller reads result[] for its convergence
 * logic); the fixed-iteration benchmark configuration uses n_iter == 3 without any host sync. */
int pinb200_track_iterations(const pinb200_map_view* map, const pinb200_decoder_view* sdf_dec,
                             const pinb200_decoder_view* color_dec, const float* source_xyz, int64_t n,
                             const pinb200_query_opts* opts, const pinb200_query_out* out,
                             const pinb200_gn_opts* gn, int32_t n_iter, void* stream);

/* The geometry-only training loop of Mapper.mapping (utils/mapper.py:600-844) issued by ONE host call. */
typedef struct pinb200_map_train_opts {
  /* sample pool (utils/mapper.py:482-503) and the pre-drawn batch indices [n_iter, bs] (torch.randint stream) */
  const float* coord_pool;
  const float* label_pool;
  const int32_t* ts_pool;
  const float* weight_pool;
  const int64_t* index;
  int64_t bs;
  int32_t decimation; /* every decimation-th sample gets the 6 numerical-gradient copies; 0 = no Eikonal term */
  float eik_eps;
  /* loss (pinb200_mapping_loss) */
  float sigma;
  float weight_e;
  int32_t loss_weight_on;
  /* Adam (pinb200_adam_step); the decoder is stepped only if train_decoder != 0 */
  double lr;
  double beta1;
  double beta2;
  double eps;
  double weight_decay;
  int32_t train_decoder;
  int32_t first_step; /* 1-based Adam step of the first iteration */
  int32_t stages;     /* bit 0: assemble + forward + loss + backward, bit 1: optimizer; 3 = whole iteration.  Data-parallel
                         training runs stage 1, all-reduces grad_feat/grad_dec, then runs stage 2 */
  float grad_scale;   /* 1/world_size when the batch is sharded over GPUs and gradients are summed, else 1 */
  /* workspaces, rows = bs + 6*ceil(bs/decimation) */
  float* rows;       /* [rows,3] */
  float* label;      /* [bs] */
  int32_t* ts;       /* [bs] */
  float* weight;     /* [bs] */
  float* dloss;      /* [rows] */
  float* losses;     /* [2] accumulated bce / eikonal over the iterations */
  float* feat;       /* [n_nb+1,F] the trained feature table (== map->geo_feat) */
  float* dec_flat;   /* flat decoder parameter vector the decoder view points into */
  float* grad_feat;  /* zero on entry, zero on exit */
  float* grad_dec;   /* zero on entry, zero on exit */
  float* m_feat;     /* Adam moments */
  float* v_feat;
  float* m_dec;
  float* v_dec;
  /* data-parallel training (one process per GPU, the batch sharded over the ranks): when nccl_comm != NULL and
   * stages == 3, every iteration sums reduce_buf[0 .. reduce_count) over the ranks (ncclAllReduce on `stream`) between
   * the backward kernels and the Adam kernels.  reduce_buf must cover grad_feat and grad_dec (the caller lays the
   * gradient blocks out contiguously); grad_scale = 1/world makes the sum the global-batch mean gradient. */
  void* nccl_comm;    /* from pinb200_nccl_init, or NULL */
  float* reduce_buf;
  int64_t reduce_count;
  /* scratch of the training forward (pinb200_query_opts.workspace): with >= pinb200_query_workspace_bytes(rows)
   * bytes, batches of at least PINB200_SPLIT_MIN_QUERIES rows run as two launches like any other query; NULL: one */
  void* workspace;
  int64_t workspace_bytes;
} pinb200_map_train_opts;

/* n_iter x [assemble_batch -> query_sdf(training) -> mapping_loss -> train_backward -> adam(decoder) -> adam(features)].
 * `out` must provide sdf / sdf_std / nn_count / certainty / knn_idx / knn_dist2 / knn_weight / knn_gidx for `rows` rows. */
int pinb200_map_iterations(const pinb200_map_view* map, const pinb200_decoder_view* dec, int32_t nn_k,
                           int32_t weighted_first, const pinb200_map_train_opts* t, const pinb200_query_out* out,
                           int32_t n_iter, void* stream);

/* NCCL communicator owned by the library (libnccl is resolved with dlopen at first use; PyTorch has it loaded).
 * Rank 0 creates the 128-byte unique id, the caller broadcasts it (e.g. torch.distributed), every rank calls
 * pinb200_nccl_init.  Used by pinb200_map_iterations (pinb200_map_train_opts.nccl_comm) for the per-iteration
 * gradient all-reduce of data-parallel map training over NVLink / NVSwitch. */
int pinb200_nccl_unique_id(uint8_t* out128);
int pinb200_nccl_init(const uint8_t* uid128, int32_t world, int32_t rank, void** comm_out);
int pinb200_nccl_destroy(void* comm);

/* Colour head of the training loss (utils/mapper.py:804-812, utils/loss.py:31-41): L1 between the predicted and
 * the measured colour on surface samples (|sdf_label| < surface_range), mean over (n_surface x Cc) elements,
 * times weight_i.  n_surface is read from the device (count computed by the caller without a sync).
 * Writes d loss / d colour [n, Cc] (zero off-surface), adds the unweighted loss to *loss. */
int pinb200_color_loss(const float* color_pred, const float* color_label, const float* sdf_label,
                       const float* weight, int64_t n, int32_t color_channels, float surface_range,
                       int32_t loss_weight_on, float weight_i, float grad_scale, const float* n_surface,
                       float* dloss_dcolor, float* loss, void* stream);

/* Probe index of a map view (pinb200_map_view.probe_words / probe_rec / probe_gid, layout documented there).
 * Six stream-ordered operations (clear, mark, 3-step prefix sum over the words, scatter); call it whenever the map
 * view changes (NeuralPoints.update / reset_local_map / recreate_hash, a new travel_dist or cur_ts).  `map` supplies
 * slot_table, buffer_size, points, n_global, ts_create, travel_dist, global2local, nb_points, resolution and the
 * time-filter fields; its probe_* fields are ignored.  Sizes: probe_words = 2 * pinb200_probe_index_words(B) u32,
 * probe_rec = 4 * n_global f32, probe_gid = n_global i32, scratch = pinb200_probe_index_scratch(B) i32
 * (scratch[last] receives n_rec). */
int64_t pinb200_probe_index_words(int64_t buffer_size);
int64_t pinb200_probe_index_scratch(int64_t buffer_size);
int pinb200_build_probe_index(const pinb200_map_view* map, uint32_t* probe_words, float* probe_rec,
                              int32_t* probe_gid, int32_t* scratch, void* stream);

/* Voxel down-sampling (utils/tools.py:583-626 voxel_down_sample_torch; with `value` != NULL :629-668
 * voxel_down_sample_min_value_torch): per occupied voxel the index of the point with the smallest selection value
 * (distance to the voxel centre, or value[i] >= 0), quantised to 1000 levels of its maximum, ties to the smaller
 * index.  Writes the (voxel key, winner index) pairs of the occupied voxels to out_key / out_idx in ARBITRARY order
 * and their number to scalars[7]; the caller sorts the pairs by key (the reference returns ascending key order).
 * Workspaces: ws_keys / ws_best [table_size] 8-byte words with table_size = pinb200_voxel_table_size(n), scalars
 * [8] i32, out_key / out_idx [>= number of voxels, n is always enough] i64.  Replaces torch.unique(return_inverse) +
 * scatter_reduce over the whole frame by a lock-free hash set (one atomicCAS + one atomicMin per point). */
int64_t pinb200_voxel_table_size(int64_t n);
int pinb200_voxel_downsample(const float* points, int64_t n, float voxel_size, const float* value, int64_t* ws_keys,
                             uint64_t* ws_best, int64_t table_size, int32_t* scalars, int64_t* out_key,
                             int64_t* out_idx, void* stream);

/* Window filter of the replay pool (utils/mapper.py:404-438): keeps the samples whose global coordinate lies within
 * sqrt(radius2) of `origin` (device, 3 x fp64; the reference's fp32 - fp64 difference is evaluated in fp64) and writes
 * them, ORDER PRESERVED, to the o_* arrays (a second arena: the call does not work in place).  counts (device, 2 x i64):
 * [0] samples kept, [1] samples kept among the last n_tail (the current frame's).  scratch: pinb200_pool_filter_scratch(n)
 * i32.  Replaces six boolean-mask indexings (six reallocations of multi-million-row tensors per frame). */
/* Local-map reset (model/neural_points.py:424-513 NeuralPoints.reset_local_map), split around the one host sync (the
   local point count shapes the local tensors).
   _select: keep_i = recent_i & near_i -> local_mask [n+1] (last entry 1: the padding row), counts = {recent points,
            local points} (device int64[2]); recent = travel-distance window (use_travel_dist) or time-stamp window around
            ts_create (or the truncated mean with ts_update: use_mid_ts), optionally only ts >= reboot_ts, everything if
            fewer than 100 are recent or temporal_on = 0; near = |p_i - sensor|^2 < radius2, evaluated in float64 when the
            sensor position is float64 (torch type promotion).  scratch: pinb200_local_map_scratch(n) int32.
   _gather: idx_pad [n_local+1] int64 (ascending global ids, then n), global2local [n+1] (local id | miss_value outside
            the local map | -1 for the padding entry), and the gathered positions / orientations / certainties /
            update stamps. */
int64_t pinb200_local_map_scratch(int64_t n);
int pinb200_local_map_select(const float* points, const int32_t* ts_create, const int32_t* ts_update, const float* travel_dist,
                             int64_t n, int32_t cur_ts, int32_t temporal_on, int32_t use_mid_ts, int32_t use_travel_dist,
                             int32_t diff_ts_local, int32_t reboot_map, int32_t reboot_ts, float diff_travel,
                             const void* sensor_pos, int32_t sensor_is_f64, double radius2, uint8_t* local_mask,
                             int32_t* scratch, int64_t* counts, void* stream);
int pinb200_local_map_gather(const float* points, const float* orient, const float* certainty, const int32_t* ts_update,
                             const uint8_t* local_mask, const int32_t* scratch, int64_t n, int64_t n_local, int32_t miss_value,
                             int64_t* idx_pad, int32_t* global2local, float* l_points, float* l_orient, float* l_certainty,
                             int32_t* l_ts_update, void* stream);

/* Per-ray training samples (utils/data_sampler.py:18-260 DataSampler.sample), ray-major output of
   total = 1 + n_surface + n_front + n_behind samples per point: the end point, Gaussian samples around it
   (z_surf [n_surface*n] standard-normal draws, element j*n + i belongs to point i), uniform samples in front
   (u_front [n_front*n]) and behind (u_behind [n_behind*n]); label = signed distance along the ray, weight with the
   reference's distance / drop-off terms and a negative sign for free-space samples; colours copied for the surface
   samples, 0 for free space.  The random draws are the caller's (torch generator of the reference). */
int pinb200_ray_samples(const float* points, const float* colors, int32_t color_channels, int64_t n, const float* z_surf,
                        const float* u_front, const float* u_behind, int32_t n_surface, int32_t n_front, int32_t n_behind,
                        float sigma, float free_begin_ratio, float free_end_dist, float max_range, int32_t dist_weight_on,
                        float dist_weight_scale, int32_t behind_dropoff_on, float* coord, float* label, float* weight,
                        float* color, void* stream);

/* Map growth (model/neural_points.py:311-392 NeuralPoints.update): tests the n voxel-down-sampled candidates [n,3]
   against the hash table (empty slot | owner farther than sqrt(3) voxels | owner not refreshed within `diff_travel` of
   travel distance when temporal_on; grow_all: every candidate, the first / reboot frame) and appends the passing ones, in
   candidate order, to the caller's arenas behind row n_points: points [cap,3], orient [cap,4] (identity), ts_create /
   ts_update [cap] (cur_ts), certainty [cap] (0).  The table is updated with the reference's sequential semantics (the
   last candidate of a slot decides its owner).  n_new (device int64) receives the number of appended points;
   scratch: pinb200_map_grow_scratch(n) int32 elements.  The feature rows are initialised by the caller (torch RNG
   stream of the reference). */
int64_t pinb200_map_grow_scratch(int64_t n);
int pinb200_map_grow(const float* cand, int64_t n, int32_t* table, int64_t buffer_size, float resolution, float* points,
                     float* orient, int32_t* ts_create, int32_t* ts_update, float* certainty, int64_t n_points,
                     int64_t capacity, const float* travel_dist, int32_t cur_ts, int32_t grow_all, int32_t temporal_on,
                     float diff_travel, float far2 /* 3 * resolution^2 */, int32_t* scratch, int64_t* n_new, void* stream);

/* Loop-closure map surgery: row i of xyz [N,3] (and of quat [N,4] wxyz, may be NULL) is moved by the correction of
   its frame t_i = ts_a[i] (or trunc((ts_a[i] + ts_b[i]) / 2) when ts_b is given: config.use_mid_ts):
     xyz_i <- R_t xyz_i + t_t,   quat_i <- dquat_t (x) quat_i,      tf3x4 [n_ts,12] = rows of [R | t], dquat [n_ts,4].
   Replaces model/neural_points.py:791-822 (adjust_map) and utils/mapper.py:527-531 (transform_data_pool). */
int pinb200_frame_transform(float* xyz, float* quat, const int32_t* ts_a, const int32_t* ts_b, const float* tf3x4,
                            const float* dquat, int64_t n, int32_t n_ts, void* stream);

int64_t pinb200_pool_filter_scratch(int64_t n);
int pinb200_pool_filter(const float* coord, const float* gcoord, const float* label, const float* weight,
                        const int32_t* ts, const float* color, int32_t color_channels, int64_t n, int64_t n_tail,
                        const double* origin, double radius2, float* o_coord, float* o_gcoord, float* o_label,
                        float* o_weight, int32_t* o_ts, float* o_color, int32_t* scratch, int64_t* counts, void* stream);

/* Batch assembly of one map-training iteration in ONE launch (utils/mapper.py:482-503 pool gathers +
 * :990-1002 the six +-eps shifted copies of every `decimation`-th sample):
 *   rows  [n + 6*ne, 3] = [ coord_pool[index] | x+e_x | x-e_x | x+e_y | x-e_y | x+e_z | x-e_z ],  ne = ceil(n/decimation)
 *   label [n], ts [n], weight [n] gathered with the same index; color [n,cc] if color_pool != NULL.
 * `index` are the int64 draws of torch.randint (the RNG stream stays the reference's). */
int pinb200_assemble_batch(const float* coord_pool, const float* label_pool, const int32_t* ts_pool,
                           const float* weight_pool, const float* color_pool, int32_t color_channels,
                           const int64_t* index, int64_t n, int32_t decimation, float eps, float* rows,
                           float* label, int32_t* ts, float* weight, float* color, void* stream);

/* Mesh extraction (DESIGN.md row f5; utils/mesher.py:369-397 skimage marching cubes, :443-456 / :631 Open3D clean-up).
   Grid: sdf fp32 / mask u8 (NULL: every cube) [nx*ny*nz], point p = (x*ny + y)*nz + z.  A corner is inside iff
   sdf < level; cube (i,j,k) is polygonised iff mask at its lowest corner.  Vertex keys: 3*p + axis for the crossing of
   the edge from grid point p along axis, at t = (level - a) / (b - a) (fp32); t exactly 0 or 1: 3*N + q for the grid
   point q it lands on.  Triangles come in cube order, table order within a cube, degenerate ones (two equal keys)
   dropped; right-hand normals point to sdf < level.
   _count: number of triangles -> n_tri (device int64) and the per-block offsets -> scratch
           (pinb200_mc_scratch_bytes(nx*ny*nz) bytes); _emit (same grid, same scratch): tri_keys [n_tri, 3] int64;
   _vertices: grid-index-space positions pos [n_keys, 3] fp64 (i + t along the edge) of vertex keys.
   pinb200_mesh_clusters: edge-connected triangle clusters.  edge_key [n_edges] ascending (one key per undirected
   triangle edge), edge_tri [n_edges] the triangle of each, parent [n_tri] scratch; on return root [n_tri] holds the
   smallest triangle id of each triangle's cluster and size [n_tri] the number of triangles of the cluster rooted there
   (0 elsewhere). */
int64_t pinb200_mc_scratch_bytes(int64_t n_points);
int pinb200_mc_count(const float* sdf, const uint8_t* mask, int64_t nx, int64_t ny, int64_t nz, float level, void* scratch,
                     int64_t* n_tri, void* stream);
int pinb200_mc_emit(const float* sdf, const uint8_t* mask, int64_t nx, int64_t ny, int64_t nz, float level,
                    const void* scratch, int64_t* tri_keys, void* stream);
int pinb200_mc_vertices(const float* sdf, int64_t nx, int64_t ny, int64_t nz, float level, const int64_t* keys,
                        int64_t n_keys, double* pos, void* stream);
int pinb200_mesh_clusters(const int64_t* edge_key, const int32_t* edge_tri, int64_t n_edges, int64_t n_tri,
                          int32_t* parent, int32_t* root, int32_t* size, void* stream);

/* Frame preparation (DESIGN.md row f6).
   pinb200_frame_crop replaces the gathers by the down-sampling index (dataset/slam_dataset.py:437-439), crop_frame
   (:1229-1248) and intrinsic_correct (:1251-1270): row j = index[i] of points [n, cols] (cols 3..7, fp32; the columns
   after xyz travel along) is kept iff min_range < r < max_range and min_z < z < max_z, r = |xyz| in fp32.  With
   correction_deg != 0, a = (float)(correction_deg / 180 * pi), v = asin(z / r), vc = v + a, x and y scale by
   cos(vc) / cos(v) and z = r sin(vc).  Survivors -> points_out [K, cols] and ts_out [K] (ts and ts_out both NULL or
   both set) in index order; K -> n_kept (device int64).  scratch: ceil(m / 1024) int32.
   pinb200_deskew replaces utils/tools.py:747-779 (roma.rotmat_slerp): in place on the xyz columns of n rows
   `row_stride` floats apart, p <- exp(s log R) p + s t with s = (ts - min ts) / (max ts - min ts) - ts_mid, pose
   T_last<-cur [4,4] fp32 row-major on the device, log R the shortest-arc rotation vector.  scratch: 2 floats.  No
   host synchronisation. */
int pinb200_frame_crop(const float* points, int64_t n, int32_t cols, const int64_t* index, int64_t m, const float* ts,
                       float min_z, float max_z, float min_range, float max_range, double correction_deg,
                       int32_t* scratch, int64_t scratch_len, int64_t* n_kept, float* points_out, float* ts_out,
                       void* stream);
int pinb200_deskew(float* points, int64_t n, int64_t row_stride, const float* ts, const float* pose, float ts_mid,
                   float* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PINB200_H */
