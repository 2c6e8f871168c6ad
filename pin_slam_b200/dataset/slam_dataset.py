"""Frame preparation of the reference's `dataset.slam_dataset.SLAMDataset` on the GPU (DESIGN.md row f6).

    import dataset.slam_dataset as sd
    from pin_slam_b200.dataset.slam_dataset import patch_reference_dataset
    patch_reference_dataset(sd)

replaces `SLAMDataset.preprocess_frame` (dataset/slam_dataset.py:359-505) and the module's `deskewing`
(utils/tools.py:747-779, which needs roma), so `update_odom_pose` and `write_merged_point_cloud` deskew through the
kernel without being copied.  The pose bookkeeping stays the reference's numpy; the point work is the voxel
down-sampling kernel, one crop / correction compaction (pinb200_frame_crop), the source down-sampling and gather, and
the in-place deskew (pinb200_deskew).  Host reads per frame: the two voxel counts, the crop count and, with
`adaptive_range_on`, the range bound.
"""
import torch

from .. import ops


def deskewing(points: torch.Tensor, ts, pose: torch.Tensor, ts_mid_pose=0.5):
    """utils/tools.py:747-779 on the GPU: points[:, :3] moved in place by the fraction of `pose` (T_last<-cur) at
    each point's normalised timestamp; returns `points`, unchanged when there are no timestamps."""
    if ts is None:
        return points
    return ops.deskew_(points, ts, pose, ts_mid_pose)


def range_bound(points: torch.Tensor, max_range: float):
    """crop_max_range of `adaptive_range_on` (slam_dataset.py:399-407): the smaller of max_range and twice the larger
    of the x and y half-extents seen from the sensor, with one host read.  Returns a Python float when max_range wins
    and a 0-dim fp32 CPU tensor otherwise, as the reference's min() of a float and a tensor does, so that the voxel
    sizes derived from it round as the reference's do."""
    lo, hi = torch.aminmax(points[:, :3], dim=0)
    half = torch.maximum(torch.minimum(hi[0].abs(), lo[0].abs()), torch.minimum(hi[1].abs(), lo[1].abs()))
    bound = 2.0 * half.cpu()
    return max_range if not bool(bound < max_range) else bound


def preprocess_frame(self):
    """SLAMDataset.preprocess_frame (dataset/slam_dataset.py:359-505) with the point work on the GPU."""
    if self.cur_sem_labels_torch is not None:
        raise NotImplementedError("pin_slam_b200: frame preparation with semantic labels (filter_sem_kitti) is not "
                                  "implemented")
    cfg = self.config
    frame_id = self.processed_frame
    cur_pose_init_guess = self.cur_pose_ref
    if frame_id == 0:
        if cfg.track_on:
            self.odom_poses[frame_id] = self.cur_pose_ref
        if cfg.pgo_on:
            self.pgo_poses[frame_id] = self.cur_pose_ref
        self.travel_dist[frame_id] = 0.0
        self.last_pose_ref = self.cur_pose_ref
    elif frame_id > 0:
        if cfg.uniform_motion_on and not self.lose_track:
            cur_pose_init_guess = self.last_pose_ref @ self.last_odom_tran  # T_world<-last @ T_last<-cur
        else:
            cur_pose_init_guess = self.last_pose_ref
        if not cfg.track_on and self.gt_pose_provided:
            cur_pose_init_guess = self.gt_poses[frame_id]
        self.cur_pose_guess_torch = torch.tensor(cur_pose_init_guess, dtype=torch.float64, device=self.device)

    cloud = self.cur_point_cloud_torch
    if cloud is None or cloud.shape[0] < 10:  # missing or nearly empty frame
        if cfg.track_on:
            self.odom_poses[frame_id] = cur_pose_init_guess
        if cfg.pgo_on:
            self.pgo_poses[frame_id] = cur_pose_init_guess
        return False
    if cloud.dtype != torch.float32:
        raise RuntimeError("pin_slam_b200: frame preparation runs on float32 point clouds")

    crop_max_range = range_bound(cloud, cfg.max_range) if cfg.adaptive_range_on else cfg.max_range
    train_voxel_m = float((crop_max_range / cfg.max_range) * cfg.vox_down_m)
    source_voxel_m = float((crop_max_range / cfg.max_range) * cfg.source_vox_down_m)

    n = cloud.shape[0]
    if cfg.rand_downsample:
        idx = torch.randint(0, n, (int(n * cfg.rand_down_r),), device=self.device)
    else:
        idx = ops.voxel_downsample(cloud[:, :3], train_voxel_m)
    ts = self.cur_point_ts_torch
    corr = cfg.correction_deg if cfg.kitti_correction_on else 0.0
    cloud = cloud.contiguous()
    points, ts_out = ops.frame_crop(cloud, idx, None if ts is None else ts.reshape(-1).contiguous(), cfg.min_z,
                                    cfg.max_z, cfg.min_range, float(crop_max_range), corr)
    self.cur_point_cloud_torch = points
    if ts is not None:
        ts_out = ts_out.view(-1, *ts.shape[1:])  # the reference keeps the [N, 1] of guessed timestamps
    self.cur_point_ts_torch = ts_out

    if frame_id > 0:  # source points for the registration
        idx = ops.voxel_downsample(points[:, :3], source_voxel_m)
        source = points[idx]
        self.cur_source_points = source[:, :3]
        if cfg.color_on:
            self.cur_source_colors = source[:, 3:]
        source_ts = None if ts_out is None else ts_out[idx]
        if cfg.deskew and not self.lose_track:
            self.cur_source_points = deskewing(
                self.cur_source_points, source_ts,
                torch.tensor(self.last_odom_tran, device=self.device, dtype=self.dtype))  # T_last<-cur
    return True


def patch_reference_dataset(module) -> None:
    """Route the reference's imported `dataset.slam_dataset` module through the frame-preparation kernels:
    `SLAMDataset.preprocess_frame` is replaced and the module global `deskewing` rebound."""
    module.SLAMDataset.preprocess_frame = preprocess_frame
    module.deskewing = deskewing

