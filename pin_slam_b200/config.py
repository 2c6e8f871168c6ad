"""Minimal configuration object carrying the attributes the hot path reads from the
reference's `utils.config.Config` (utils/config.py:13-312), with the same names and
defaults.  The drop-in classes are duck-typed: they accept the reference Config
unchanged; this class exists so the hot path can be driven without the reference
checkout (tests, bench, smoke on the GPU box)."""
from dataclasses import dataclass

import torch


@dataclass
class HotPathConfig:
    device: str = "cuda"
    dtype: torch.dtype = torch.float32
    tran_dtype: torch.dtype = torch.float64
    silence: bool = True
    # neural points (config.py:92-104)
    voxel_size_m: float = 0.3
    weighted_first: bool = True
    layer_norm_on: bool = False
    num_nei_cells: int = 2
    query_nn_k: int = 6
    use_mid_ts: bool = False
    search_alpha: float = 0.2
    buffer_size: int = int(5e7)
    feature_dim: int = 8
    feature_std: float = 0.0
    color_on: bool = False
    color_channel: int = 0
    # local map (config.py:112-115, 559-560)
    diff_ts_local: float = 400.0
    local_map_travel_dist_ratio: float = 5.0
    local_map_radius: float = 50.0
    max_range: float = 60.0
    # decoder (config.py:138-158)
    mlp_bias_on: bool = True
    mlp_leaky_relu: bool = False
    geo_mlp_level: int = 1
    geo_mlp_hidden_dim: int = 64
    color_mlp_level: int = 1
    color_mlp_hidden_dim: int = 64
    use_gaussian_pe: bool = False
    pos_encoding_band: int = 0
    pos_input_dim: int = 3
    # loss (config.py:161-184)
    main_loss_type: str = "bce"
    sigma_sigmoid_m: float = 0.1
    logistic_gaussian_ratio: float = 0.55
    loss_weight_on: bool = False
    numerical_grad: bool = True
    gradient_decimation: int = 10
    num_grad_step_ratio: float = 0.2
    ekional_loss_on: bool = True
    ekional_add_to: str = "all"
    weight_e: float = 0.5
    weight_i: float = 1.0
    surface_sample_range_m: float = 0.25
    # optimiser (config.py:188-199)
    iters: int = 12
    bs: int = 16384
    lr: float = 0.01
    weight_decay: float = 0.0
    adam_eps: float = 1e-15
    opt_adam: bool = True
    bs_new_sample: int = 2048
    # tracker (config.py:213-233)
    track_on: bool = True
    photometric_loss_on: bool = False
    photometric_loss_weight: float = 0.01
    consist_wieght_on: bool = True
    reg_min_grad_norm: float = 0.5
    reg_max_grad_norm: float = 2.0
    track_mask_query_nn_k: int = 6
    max_sdf_ratio: float = 5.0
    max_sdf_std_ratio: float = 1.0
    reg_dist_div_grad_norm: bool = False
    reg_GM_dist_m: float = 0.3
    reg_GM_grad: float = 0.1
    reg_lm_lambda: float = 1e-4
    reg_iter_n: int = 50
    reg_term_thre_deg: float = 0.01
    reg_term_thre_m: float = 0.001
    eigenvalue_check: bool = True
    eigenvalue_ratio_thre: float = 0.005
    final_residual_ratio_thre: float = 0.6
    semantic_on: bool = False
    # sampler / pool / map management (config.py:105-136)
    surface_sample_n: int = 3
    free_sample_begin_ratio: float = 0.3
    free_sample_end_dist_m: float = 1.0
    free_front_n: int = 2
    free_behind_n: int = 1
    dist_weight_on: bool = True
    dist_weight_scale: float = 0.8
    behind_dropoff_on: bool = False
    from_sample_points: bool = True
    from_all_samples: bool = False
    map_surface_ratio: float = 0.5
    prune_map_on: bool = False
    max_prune_certainty: float = 3.0
    prune_freq_frame: int = 100
    window_radius: float = 50.0
    pool_capacity: int = int(1e7)
    new_certainty_thre: float = 1.0
    pool_filter_freq: int = 10
    adaptive_iters: bool = False
    new_sample_ratio_less: float = 0.02
    new_sample_ratio_more: float = 0.15
    new_sample_ratio_restart: float = 0.3
    freeze_after_frame: int = 40
    dynamic_filter_on: bool = False
    dynamic_certainty_thre: float = 1.0
    dynamic_sdf_ratio_thre: float = 0.5
    dynamic_min_grad_norm_thre: float = 0.25
    pgo_on: bool = False
    # mesh reconstruction (config.py:281-289)
    mc_res_m: float = 0.3
    pad_voxel: int = 3
    skip_top_voxel: int = 2
    mc_mask_on: bool = True
    mesh_min_nn: int = 8
    min_cluster_vertices: int = 300
    # frame preparation (config.py:48-68, :216)
    deskew: bool = False
    min_z: float = -5.0
    max_z: float = 80.0
    min_range: float = 2.5
    adaptive_range_on: bool = False
    kitti_correction_on: bool = False
    correction_deg: float = 0.0
    vox_down_m: float = 0.05
    source_vox_down_m: float = 0.8
    rand_downsample: bool = False
    rand_down_r: float = 1.0

    @property
    def infer_bs(self):
        return self.bs * 32

    @classmethod
    def kitti(cls, **kw):
        """config/lidar_slam/run_kitti.yaml of the reference (SURVEY.md App. C)."""
        d = dict(voxel_size_m=0.4, weighted_first=False, feature_dim=8, query_nn_k=6, track_mask_query_nn_k=6,
                 sigma_sigmoid_m=0.08, loss_weight_on=True, weight_e=0.5, max_range=80.0, local_map_radius=82.0,
                 surface_sample_range_m=0.25, reg_GM_dist_m=0.2, reg_GM_grad=0.1, reg_iter_n=100, bs_new_sample=1000,
                 surface_sample_n=4, free_front_n=2, free_behind_n=1, window_radius=80.0, pool_capacity=int(2e7),
                 pool_filter_freq=1)
        d.update(kw)
        return cls(**d)

    @classmethod
    def replica(cls, **kw):
        """config/rgbd_slam/run_replica.yaml of the reference (SURVEY.md App. C): RGB-D, colour head, photometric
        tracking, weighted_first (default)."""
        d = dict(voxel_size_m=0.05, weighted_first=True, feature_dim=8, query_nn_k=6, track_mask_query_nn_k=6,
                 color_on=True, color_channel=3, sigma_sigmoid_m=0.01, weight_e=0.2, surface_sample_range_m=0.03,
                 surface_sample_n=3, free_front_n=1, free_behind_n=1, free_sample_end_dist_m=0.1, bs_new_sample=4000,
                 pool_capacity=int(2e7), pool_filter_freq=10, photometric_loss_on=True, photometric_loss_weight=0.01,
                 eigenvalue_check=False, reg_min_grad_norm=0.4, reg_max_grad_norm=2.5, reg_GM_grad=0.3,
                 reg_GM_dist_m=0.05, reg_term_thre_deg=1e-3, reg_term_thre_m=1e-4, reg_iter_n=50, iters=20,
                 max_range=10.0, local_map_radius=12.0, window_radius=10.0)
        d.update(kw)
        return cls(**d)

    @classmethod
    def cfg2(cls, **kw):
        """BASELINE.json configs[1]: 32-d features, K=8, 2-layer decoder."""
        d = dict(voxel_size_m=0.4, weighted_first=True, feature_dim=32, query_nn_k=8, track_mask_query_nn_k=8,
                 geo_mlp_level=2)
        d.update(kw)
        return cls(**d)
