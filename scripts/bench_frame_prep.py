#!/usr/bin/env python3
"""Device time per stage and host synchronisations of the frame preparation (DESIGN.md row f6): the reference's
SLAMDataset.preprocess_frame + the mapping deskew of update_odom_pose in torch CUDA (oracle/_ref, with
oracle/frame_oracle.py's torch slerp standing in for roma), then the same object patched by patch_reference_dataset.

    python scripts/bench_frame_prep.py [--iters 50] [--out bench_frame_prep.json]

Scans are seeded 64 x 1024 and 128 x 2048 rings (intensity column, Ouster index timestamps), with the KITTI crop
and correction settings and deskew on.  Prints one table and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import frame_oracle as fo  # noqa: E402


def ring_scan(beams, cols, seed):
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(np.linspace(-22.5, 22.5, beams))
    az = np.linspace(np.pi, -np.pi, cols, endpoint=False)
    A, E = (g.T.reshape(-1) for g in np.meshgrid(az, elev, indexing="xy"))
    d = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], 1)
    t = rng.uniform(2.0, 90.0, d.shape[0])
    with np.errstate(divide="ignore"):
        tz = -1.73 / d[:, 2]
    t = np.where((tz > 0) & (tz < t), tz, t)
    p = d * t[:, None] + rng.normal(0, 0.01, d.shape)
    inten = rng.random(p.shape[0])
    ts = (np.floor(np.arange(p.shape[0]) / beams) / cols).reshape(-1, 1)
    return np.concatenate([p, inten[:, None]], 1).astype(np.float32), ts.astype(np.float32)


def make_dataset(sd, cloud, ts):
    from utils.config import Config

    cfg = Config()
    cfg.device, cfg.silence, cfg.track_on, cfg.pgo_on = "cuda", True, True, False
    cfg.kitti_correction_on, cfg.correction_deg, cfg.deskew = True, 0.195, True
    cfg.min_range, cfg.max_range, cfg.min_z, cfg.vox_down_m, cfg.source_vox_down_m = 3.0, 80.0, -3.5, 0.08, 0.6
    cfg.setup_dtype()
    ds = sd.SLAMDataset.__new__(sd.SLAMDataset)
    ds.config, ds.silence, ds.device, ds.dtype = cfg, True, "cuda", cfg.dtype
    ds.odom_poses, ds.pgo_poses, ds.travel_dist = np.zeros((3, 4, 4)), None, np.zeros(3)
    ds.gt_pose_provided, ds.lose_track, ds.cur_sem_labels_torch = False, False, None
    ds.stop_count, ds.consecutive_lose_track_frame = 0, 0
    ds.cur_pose_ref, ds.last_pose_ref = np.eye(4), np.eye(4)
    motion = np.eye(4)
    c, s = np.cos(0.03), np.sin(0.03)
    motion[:2, :2] = [[c, -s], [s, c]]
    motion[:3, 3] = [1.2, 0.05, 0.01]
    ds.last_odom_tran, ds.processed_frame = motion, 1
    ds.cur_cloud_np, ds.cur_ts_np = cloud, ts
    return ds


def run_frame(ds, tracked):
    ds.cur_point_cloud_torch = torch.from_numpy(ds.cur_cloud_np).cuda()
    ds.cur_point_ts_torch = torch.from_numpy(ds.cur_ts_np).cuda()
    ds.last_pose_ref = np.eye(4)
    ds.preprocess_frame()
    ds.update_odom_pose(tracked)


class Stages:
    """CUDA-event time per named stage, accumulated over calls (wraps module attributes)."""

    def __init__(self):
        self.ms, self.calls = {}, {}

    def wrap(self, owner, attr, name):
        fn = getattr(owner, attr)

        def timed(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **k)
            e1.record()
            self.pending.append((name, e0, e1))
            return out

        setattr(owner, attr, timed)
        return fn

    def start(self):
        self.pending = []

    def collect(self):
        torch.cuda.synchronize()
        for name, e0, e1 in self.pending:
            self.ms[name] = self.ms.get(name, 0.0) + e0.elapsed_time(e1)
            self.calls[name] = self.calls.get(name, 0) + 1


def measure(ds, tracked, iters, stages):
    for _ in range(5):  # warm-up: module loads, allocator, library picks
        stages.start()
        run_frame(ds, tracked)
        stages.collect()
    stages.ms, stages.calls = {}, {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(iters):
        stages.start()
        e0.record()
        run_frame(ds, tracked)
        e1.record()
        stages.collect()
        total += e0.elapsed_time(e1)
    torch.cuda.set_sync_debug_mode("warn")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        run_frame(ds, tracked)
    torch.cuda.set_sync_debug_mode(0)
    syncs = sum("synchroniz" in str(x.message) for x in w)
    return dict(frame_ms=total / iters, syncs=syncs,
                stages={k: v / iters for k, v in stages.ms.items()})


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_prep: needs a CUDA device")
    if not fo.reference_dataset_available():
        raise SystemExit("bench_frame_prep: oracle/_ref has no dataset/slam_dataset.py (build() makes it)")
    sd = fo.load_reference_dataset()
    import utils.tools as tools

    from pin_slam_b200 import ops
    from pin_slam_b200.dataset import slam_dataset as drop

    tracked = torch.tensor(np.eye(4), device="cuda")
    tracked[:3, 3] = torch.tensor([1.0, 0.02, 0.0])
    card = gpu_info()
    rows = []
    for beams, cols in ((64, 1024), (128, 2048)):
        cloud, ts = ring_scan(beams, cols, beams)
        res = {}
        # reference formulation (torch CUDA)
        st = Stages()
        orig = [(sd, "voxel_down_sample_torch", st.wrap(sd, "voxel_down_sample_torch", "voxel down-sampling")),
                (sd, "crop_frame", st.wrap(sd, "crop_frame", "crop")),
                (sd, "intrinsic_correct", st.wrap(sd, "intrinsic_correct", "correction")),
                (sd, "deskewing", st.wrap(sd, "deskewing", "deskew"))]
        pre = sd.SLAMDataset.preprocess_frame
        res["reference"] = measure(make_dataset(sd, cloud, ts), tracked, a.iters, st)
        for owner, attr, fn in orig:
            setattr(owner, attr, fn)
        # drop-in
        drop.patch_reference_dataset(sd)
        st = Stages()
        orig = [(ops, "voxel_downsample", st.wrap(ops, "voxel_downsample", "voxel down-sampling")),
                (ops, "frame_crop", st.wrap(ops, "frame_crop", "crop + correction")),
                (ops, "deskew_", st.wrap(ops, "deskew_", "deskew"))]
        res["drop-in"] = measure(make_dataset(sd, cloud, ts), tracked, a.iters, st)
        for owner, attr, fn in orig:
            setattr(owner, attr, fn)
        sd.SLAMDataset.preprocess_frame, sd.deskewing = pre, tools.deskewing
        rows.append(dict(scan=f"{beams}x{cols}", points=int(cloud.shape[0]), **res))
    print(f"card: {card}")
    print(f"{'scan':>9} {'impl':>9} {'frame ms':>9} {'syncs':>6}  stages (ms per frame)")
    for r in rows:
        for impl in ("reference", "drop-in"):
            x = r[impl]
            st = ", ".join(f"{k} {v:.3f}" for k, v in x["stages"].items())
            print(f"{r['scan']:>9} {impl:>9} {x['frame_ms']:9.3f} {x['syncs']:6d}  {st}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(dict(card=card, rows=rows), open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
