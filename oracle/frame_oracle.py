"""Frame preparation (DESIGN.md row f6) restated in numpy: the crop and intrinsic correction of
dataset/slam_dataset.py:1229-1270 in fp32, as the reference computes them, the preparation chain of
SLAMDataset.preprocess_frame (:399-500), and the deskewing of utils/tools.py:747-779 in fp64.

The reference deskews with roma.rotmat_slerp(I, R, s) = exp(s log R) with log R on the shortest arc.  Here that is
the quaternion logarithm of R followed by Rodrigues' formula, pinned against scipy's
Rotation.from_rotvec(s * Rotation.from_matrix(R).as_rotvec()) by tests/test_frame_prep.py.  No run of roma has
checked it: roma is not installed where the fixtures are made.
"""
import math
import os
import sys
import types
from unittest.mock import MagicMock

import numpy as np
import torch

F32 = np.float32
REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def crop_mask(xyz: np.ndarray, min_z, max_z, min_range, max_range) -> np.ndarray:
    """crop_frame's test in fp32: min_range < |xyz| < max_range and min_z < z < max_z, |xyz| = sqrt((x*x + y*y) + z*z)
    with every product and sum rounded on its own."""
    x, y, z = (xyz[:, a].astype(F32) for a in range(3))
    r = np.sqrt((x * x + y * y) + z * z)
    return (r > F32(min_range)) & (r < F32(max_range)) & (z > F32(min_z)) & (z < F32(max_z))


def correction_angle(correction_deg: float) -> np.float32:
    """The Python scalar correct_deg / 180 * pi, rounded once to fp32 when added to the fp32 angles."""
    return F32(correction_deg / 180.0 * math.pi)


def intrinsic_correct(points: np.ndarray, correction_deg: float) -> np.ndarray:
    """slam_dataset.py:1251-1270 in fp32 on a copy of `points`."""
    p = points.astype(F32, copy=True)
    if correction_deg == 0.0:
        return p
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r = np.sqrt((x * x + y * y) + z * z)
    v = np.arcsin(z / r)
    vc = v + correction_angle(correction_deg)
    s = np.cos(vc) / np.cos(v)
    p[:, 0] = x * s
    p[:, 1] = y * s
    p[:, 2] = r * np.sin(vc)
    return p


def frame_crop(points, index, ts, min_z, max_z, min_range, max_range, correction_deg=0.0):
    """points[index] (and ts[index]) cropped and corrected: (points_out, ts_out or None, kept rows of `points`)."""
    index = np.asarray(index, np.int64)
    keep = crop_mask(points[index, :3], min_z, max_z, min_range, max_range)
    rows = index[keep]
    out = intrinsic_correct(points[rows], correction_deg)
    return out, None if ts is None else np.asarray(ts, F32).reshape(-1)[rows], rows


def rotation_log(R: np.ndarray) -> np.ndarray:
    """Shortest-arc rotation vector of a (nearly orthonormal) rotation matrix, fp64: the quaternion by the largest of
    (trace, diagonal), normalised, w >= 0, then 2 atan2(|v|, w) v / |v|."""
    R = np.asarray(R, np.float64)
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    if tr >= R[0, 0] and tr >= R[1, 1] and tr >= R[2, 2]:
        s = 2.0 * math.sqrt(1.0 + tr)
        q = [0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    elif R[0, 0] >= R[1, 1] and R[0, 0] >= R[2, 2]:
        s = 2.0 * math.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2])
        q = [(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s]
    elif R[1, 1] >= R[2, 2]:
        s = 2.0 * math.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2])
        q = [(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s]
    else:
        s = 2.0 * math.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1])
        q = [(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s]
    q = np.array(q) / np.linalg.norm(q)
    if q[0] < 0:
        q = -q
    vn = np.linalg.norm(q[1:])
    return q[1:] * (2.0 * math.atan2(vn, q[0]) / vn) if vn > 0 else np.zeros(3)


def rotation_exp(phi: np.ndarray) -> np.ndarray:
    """Rotation matrices [n, 3, 3] of rotation vectors [n, 3] (Rodrigues, with the series below 1e-4 rad)."""
    phi = np.asarray(phi, np.float64).reshape(-1, 3)
    th2 = (phi * phi).sum(1)
    th = np.sqrt(th2)
    small = th < 1e-4
    ths = np.where(small, 1.0, th)
    a = np.where(small, 1.0 - th2 / 6.0 * (1.0 - th2 / 20.0), np.sin(ths) / ths)
    b = np.where(small, 0.5 - th2 / 24.0 * (1.0 - th2 / 30.0), 2.0 * np.sin(0.5 * ths) ** 2 / ths ** 2)
    K = np.zeros((phi.shape[0], 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -phi[:, 2], phi[:, 1], -phi[:, 0]
    K[:, 1, 0], K[:, 2, 0], K[:, 2, 1] = phi[:, 2], -phi[:, 1], phi[:, 0]
    return np.eye(3) + a[:, None, None] * K + b[:, None, None] * (K @ K)


def deskew_fraction(ts: np.ndarray, ts_mid: float = 0.5) -> np.ndarray:
    """s = (ts - min) / (max - min) - ts_mid in fp32, as torch computes it (all-equal ts: 0/0 = NaN)."""
    ts = np.asarray(ts, F32).reshape(-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (ts - ts.min()) / (ts.max() - ts.min()) - F32(ts_mid)


def deskew(points: np.ndarray, ts: np.ndarray, pose: np.ndarray, ts_mid: float = 0.5) -> np.ndarray:
    """utils/tools.py:747-779 in fp64: p' = exp(s log R) p + s t for the xyz of `points` (fp32 pose, as the reference
    rounds it); returns the deskewed xyz [n, 3] fp64."""
    pose = np.asarray(pose, F32).astype(np.float64)
    s = deskew_fraction(ts, ts_mid).astype(np.float64)
    Rs = rotation_exp(s[:, None] * rotation_log(pose[:3, :3])[None, :])
    p = np.asarray(points, F32)[:, :3].astype(np.float64)
    return np.einsum("nij,nj->ni", Rs, p) + s[:, None] * pose[:3, 3][None, :]


def range_bound(points: np.ndarray, max_range: float):
    """crop_max_range of adaptive_range_on (slam_dataset.py:399-407): a Python float when max_range wins, else fp32."""
    xyz = np.asarray(points, F32)[:, :3]
    hi, lo = xyz.max(0), xyz.min(0)
    b = F32(2.0) * max(min(abs(hi[0]), abs(lo[0])), min(abs(hi[1]), abs(lo[1])))
    return max_range if not b < max_range else b


def voxel_down_sample(points: np.ndarray, voxel: float) -> np.ndarray:
    """The reference's voxel_down_sample_torch in its torch CPU form (pinned by the golden fixtures)."""
    from pin_slam_b200.model.neural_points import voxel_down_sample as vds

    return vds(torch.from_numpy(np.ascontiguousarray(points[:, :3], F32)), voxel).numpy()


def prepare_frame(cloud, ts, cfg, frame_id, last_odom_tran=None, lose_track=False):
    """SLAMDataset.preprocess_frame's point work (no semantic labels); for frame_id > 0 the source points, deskewed
    with `last_odom_tran` (T_last<-cur) when cfg.deskew is on.  `cfg` carries the reference's names.  Returns a dict:
    points, ts, rows (rows of `cloud` kept, in order) and, for frame_id > 0, source [n, 3] fp64 and source_rows (their
    rows of `cloud`)."""
    cloud = np.asarray(cloud, F32)
    crop_max_range = range_bound(cloud, cfg.max_range) if cfg.adaptive_range_on else cfg.max_range
    if isinstance(crop_max_range, np.floating):  # fp32 tensor arithmetic of the reference
        ratio = F32(crop_max_range) / F32(cfg.max_range)
        train_voxel_m, source_voxel_m = float(ratio * F32(cfg.vox_down_m)), float(ratio * F32(cfg.source_vox_down_m))
    else:
        train_voxel_m, source_voxel_m = cfg.vox_down_m, cfg.source_vox_down_m
    idx = voxel_down_sample(cloud, train_voxel_m)
    corr = cfg.correction_deg if cfg.kitti_correction_on else 0.0
    pts, ts_out, rows = frame_crop(cloud, idx, ts, cfg.min_z, cfg.max_z, cfg.min_range, float(crop_max_range), corr)
    out = dict(points=pts, ts=ts_out, rows=rows)
    if frame_id > 0:
        sidx = voxel_down_sample(pts, source_voxel_m)
        src = pts[sidx, :3].astype(np.float64)
        if cfg.deskew and not lose_track and ts_out is not None:
            src = deskew(pts[sidx], ts_out[sidx], last_odom_tran)
        out["source"], out["source_rows"] = src, rows[sidx]
    return out


def rotmat_slerp_torch(R0: torch.Tensor, R1: torch.Tensor, steps: torch.Tensor) -> torch.Tensor:
    """roma.rotmat_slerp(R0, R1, steps) in torch, [n, 3, 3] in the dtype of R1: R0 exp(steps log(R0^T R1)), the log
    on the shortest arc (rotation_log, one host read of the 3x3) and one rotation matrix per step, as roma builds."""
    w = torch.as_tensor(rotation_log((R0.transpose(0, 1) @ R1).double().cpu().numpy()), dtype=R1.dtype,
                        device=R1.device)
    phi = steps.reshape(-1, 1) * w
    th2 = (phi * phi).sum(1, keepdim=True)
    th = th2.sqrt()
    small = th < 1e-4
    ths = torch.where(small, torch.ones_like(th), th)
    a = torch.where(small, 1.0 - th2 / 6.0, torch.sin(ths) / ths).unsqueeze(-1)
    b = torch.where(small, 0.5 - th2 / 24.0, 2.0 * torch.sin(0.5 * ths) ** 2 / ths ** 2).unsqueeze(-1)
    z = torch.zeros_like(phi[:, 0])
    K = torch.stack([z, -phi[:, 2], phi[:, 1], phi[:, 2], z, -phi[:, 0], -phi[:, 1], phi[:, 0], z], 1).view(-1, 3, 3)
    return R0 @ (torch.eye(3, dtype=R1.dtype, device=R1.device) + a * K + b * (K @ K))


def reference_dataset_available() -> bool:
    return os.path.isfile(os.path.join(REF, "dataset", "slam_dataset.py"))


def load_reference_dataset(root: str = REF):
    """Import the reference's unmodified `dataset.slam_dataset` from `root` (oracle/_ref, see oracle/make_ref_frame.py)
    with its GUI / IO dependencies stubbed, and give its `utils.tools` rotmat_slerp_torch in place of roma."""
    for m in ["open3d", "matplotlib", "matplotlib.cm", "matplotlib.pyplot", "roma", "wandb", "natsort", "skimage",
              "skimage.measure", "pypose", "gtsam", "dtyper", "pyquaternion", "laspy", "evo"]:
        sys.modules.setdefault(m, MagicMock())
    for m in ["dataset", "dataset.slam_dataset"]:  # oracle/ref_arm.py stubs these
        if isinstance(sys.modules.get(m), MagicMock):
            del sys.modules[m]
    if root not in sys.path:
        sys.path.insert(0, root)
    import dataset.slam_dataset as sd
    import utils.tools as tools

    tools.roma = types.SimpleNamespace(rotmat_slerp=rotmat_slerp_torch)
    return sd
