#!/usr/bin/env python3
"""Generate tests/golden/prep_kitti.npz by running the UNMODIFIED reference's SLAMDataset.preprocess_frame
(dataset/slam_dataset.py:359-505 of PRBonn/PIN_SLAM, with the same optional-import stubs as make_golden.py) on seeded
64 x 1024 scans with an intensity column, CPU, fp32.  Run where a reference checkout exists:

    python tests/golden/make_golden_prep.py [--src /root/reference]

Two configurations, each at frame 0 and frame 1 (frame 1 also down-samples the registration source):
  kitti: run_kitti.yaml (kitti_correction_on, correct_deg 0.195), velodyne yaw timestamps (get_point_ts)
  run:   run.yaml with adaptive_range_on, Ouster-64 index timestamps [N, 1] (get_point_ts)
Deskew is off: the reference deskews with roma, which is not installed here.  The intensity column is a permutation
of k / 65536, so every output row names the input row it came from; with color_on the source rows are named the same
way.  To stay small the fixture keeps no clouds and no timestamps: `scan(seed)` regenerates the clouds (numpy's PCG64
stream; `cloud_sha256` pins their bytes) and `scan_ts` restates the guessed timestamps.  Per frame it keeps the kept
rows as a bit mask, the ordered survivors and source rows as sha256 digests of their int64 ids, and, for the
corrected KITTI configuration, the xyz of N_SAMPLE seeded output rows.  That outputs carry the intensity and
timestamps of their survivors is checked here.
"""
import argparse
import hashlib
import os
import sys
from unittest.mock import MagicMock

import numpy as np

F32 = np.float32

OUT = os.path.dirname(os.path.abspath(__file__))
N_BEAM, N_AZ = 64, 1024
N_SAMPLE = 4096  # corrected output rows whose coordinates the fixture keeps, per frame


def digest(a) -> str:
    """sha256 of an array's bytes (row ids as int64)."""
    a = np.asarray(a)
    return hashlib.sha256((a.astype(np.int64) if a.dtype.kind in "iu" else a).tobytes()).hexdigest()


def scan_ts(cloud, name):
    """The timestamps get_point_ts guesses for these clouds (slam_dataset.py:307-337) restated in numpy: Ouster-64
    column index [N, 1] for the `run` clouds, velodyne yaw [N] for the KITTI ones."""
    n = cloud.shape[0]
    if name == "run":
        return (np.floor(np.arange(n) / 64) / 1024).reshape(-1, 1).astype(np.float32)
    yaw = -np.arctan2(cloud[:, 1], cloud[:, 0])
    return (F32(0.5) * (yaw / F32(np.pi) + F32(1.0))).astype(np.float32)


def scan(seed, drop_rays):
    """A 64-beam ring scan of a room (walls at x = -26 / 31, y = -13 / 17), a ground plane at z = -1.73, a ceiling-free
    a few zero returns; `drop_rays` removes the rays without a return (KITTI-style clouds)."""
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(np.linspace(-24.8, 2.0, N_BEAM))
    az = np.linspace(np.pi, -np.pi, N_AZ, endpoint=False)
    A, E = np.meshgrid(az, elev, indexing="xy")  # [beam, az] ... order the cloud column-major like an Ouster
    A, E = A.T.reshape(-1), E.T.reshape(-1)
    d = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], 1)
    t = np.full(d.shape[0], 150.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        for axis, planes in ((0, (-26.0, 31.0)), (1, (-13.0, 17.0)), (2, (-1.73,))):
            for c in planes:
                tt = (c + rng.normal(0, 0.002)) / d[:, axis]
                t = np.where((tt > 0) & (tt < t), tt, t)
    t = t + rng.normal(0.0, 0.01, t.shape)
    p = d * t[:, None]
    p += rng.normal(0.0, 0.3, 3) * np.array([1.0, 1.0, 0.02])  # sensor offset between the frames
    p[rng.random(p.shape[0]) < 0.01] = 0.0  # no-return rays written as zeros
    if drop_rays:
        p = p[np.abs(p).sum(1) > 0]
    inten = rng.permutation(p.shape[0]).astype(np.float64) / 65536.0
    return np.concatenate([p, inten[:, None]], 1).astype(np.float32)


def main(src):
    for m in ["open3d", "matplotlib", "matplotlib.cm", "matplotlib.pyplot", "roma", "wandb", "natsort",
              "skimage", "skimage.measure", "pypose", "gtsam", "dtyper", "pyquaternion", "laspy", "evo"]:
        sys.modules[m] = MagicMock()
    sys.path.insert(0, src)
    import torch

    from dataset.slam_dataset import SLAMDataset
    from utils.config import Config

    out = {}
    for name, yaml, seed in (("kitti", "run_kitti.yaml", 11), ("run", "run.yaml", 21)):
        cfg = Config()
        cfg.load(os.path.join(src, "config", "lidar_slam", yaml))
        cfg.device, cfg.silence, cfg.track_on, cfg.pgo_on, cfg.color_on = "cpu", True, True, False, True
        if name == "run":
            cfg.adaptive_range_on = True
        cfg.setup_dtype()
        torch.set_default_dtype(cfg.dtype)
        for k in ("min_z", "max_z", "min_range", "max_range", "vox_down_m", "source_vox_down_m", "correction_deg"):
            out[f"{name}.cfg.{k}"] = np.float64(getattr(cfg, k))
        for k in ("kitti_correction_on", "adaptive_range_on"):
            out[f"{name}.cfg.{k}"] = np.bool_(getattr(cfg, k))
        ds = SLAMDataset.__new__(SLAMDataset)
        ds.config, ds.silence, ds.device, ds.dtype = cfg, True, "cpu", cfg.dtype
        ds.odom_poses, ds.pgo_poses, ds.travel_dist = np.zeros((4, 4, 4)), None, np.zeros(4)
        ds.gt_pose_provided, ds.lose_track, ds.cur_sem_labels_torch = False, False, None
        ds.last_odom_tran = np.eye(4)
        ds.cur_pose_ref = np.eye(4)
        for f in (0, 1):
            cloud = scan(seed + f, drop_rays=(name == "kitti"))
            assert (cloud.shape[0] == N_BEAM * N_AZ) == (name == "run")  # Ouster-64 timestamps vs velodyne yaw
            ds.processed_frame = f
            ds.cur_point_cloud_torch = torch.tensor(cloud)
            cfg.deskew, cfg.lidar_type_guess = True, "velodyne"
            ds.get_point_ts(None)
            cfg.deskew = False
            ts = ds.cur_point_ts_torch.numpy().copy()
            assert ds.preprocess_frame()
            pts = ds.cur_point_cloud_torch.numpy()
            key = f"{name}.f{f}."
            row_of = np.argsort(np.rint(cloud[:, 3].astype(np.float64) * 65536.0).astype(np.int64))
            surv = row_of[np.rint(pts[:, 3].astype(np.float64) * 65536.0).astype(np.int64)]
            assert np.array_equal(pts[:, 3], cloud[surv, 3])
            assert np.array_equal(ds.cur_point_ts_torch.numpy().reshape(-1), ts.reshape(-1)[surv])
            assert np.allclose(scan_ts(cloud, name), ts, rtol=0, atol=1e-6)
            out[key + "cloud_sha256"] = np.array(digest(cloud))
            out[key + "kept"] = np.packbits(np.isin(np.arange(cloud.shape[0]), surv))
            out[key + "survivors_sha256"] = np.array(digest(surv))
            if cfg.kitti_correction_on:
                pick = np.sort(np.random.default_rng(seed + f).choice(pts.shape[0], N_SAMPLE, replace=False))
                out[key + "sample"], out[key + "sample_xyz"] = pick.astype(np.int32), pts[pick, :3].copy()
            else:
                assert np.array_equal(pts, cloud[surv])
            if f > 0:  # color_on: cur_source_colors is the intensity column of the source rows
                src_rows = row_of[np.rint(ds.cur_source_colors.numpy()[:, 0].astype(np.float64) * 65536.0)
                                  .astype(np.int64)]
                assert np.isin(src_rows, surv).all()
                out[key + "source_sha256"] = np.array(digest(src_rows))
            ds.last_odom_tran = np.eye(4)
            ds.last_odom_tran[:3, 3] = [0.8, 0.05, 0.0]
            ds.last_pose_ref = ds.cur_pose_ref
    path = os.path.join(OUT, "prep_kitti.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items() if v.ndim})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default="/root/reference")
    main(ap.parse_args().src)
