"""Frame preparation (DESIGN.md row f6): crop, intrinsic correction and deskewing.  CPU tests pin the numpy oracle
(oracle/frame_oracle.py) against the reference's own preprocess_frame (tests/golden/prep_kitti.npz) and its deskew
rotation against scipy; GPU tests compare the kernels of pin_slam_b200/csrc/frame and the patched reference
SLAMDataset (oracle/_ref) with the oracle."""
import os
import re
import types

import numpy as np
import pytest
import torch

from oracle import frame_oracle as fo
from tests.golden.make_golden_prep import digest, scan, scan_ts
from tests.helpers import kernels_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FRAME_CSRC = os.path.join(ROOT, "pin_slam_b200", "csrc", "frame")
FIXTURE = os.path.join(ROOT, "tests", "golden", "prep_kitti.npz")
SEEDS = {"kitti": 11, "run": 21}  # tests/golden/make_golden_prep.py

# kernel ledger of the frame module (pin_slam_b200/csrc/frame): every __global__ kernel there is named by a test of
# this file, and that test checks that it launched it
FRAME_KERNEL_LEDGER = {
    "crop_count_kernel": "test_crop_matches_oracle",
    "crop_scan_kernel": "test_crop_matches_oracle",
    "crop_scatter_kernel": "test_crop_matches_oracle",
    "deskew_minmax_kernel": "test_deskew_matches_fp64_oracle",
    "deskew_apply_kernel": "test_deskew_matches_fp64_oracle",
}


def assert_launched(fn, test, tries=3):
    """fn() launches every kernel the ledger gives to `test`.  The profiler now and then drops the first kernels of a
    trace, so a torch kernel opens each window and the kernel names of up to `tries` runs of fn() are pooled."""
    want = [k for k, v in FRAME_KERNEL_LEDGER.items() if v == test]
    assert want
    names = set()
    for _ in range(tries):
        names |= kernels_run(lambda: (torch.ones(1, device="cuda").add_(1), fn()))[1]
        missing = [k for k in want if not any(re.search(rf"\bpinb::{k}\b", n) for n in names)]
        if not missing:
            return
    assert not missing, (missing, sorted(n for n in names if "pinb::" in n))


def fixture_frame(fx, name, f):
    """(cloud, ts, config namespace) of one fixture frame; the cloud is regenerated and checked against its hash."""
    cloud = scan(SEEDS[name] + f, drop_rays=(name == "kitti"))
    assert digest(cloud) == str(fx[f"{name}.f{f}.cloud_sha256"])
    pre = f"{name}.cfg."
    cfg = types.SimpleNamespace(**{k[len(pre):]: fx[k].item() for k in fx.files if k.startswith(pre)})
    cfg.deskew = False
    return cloud, scan_ts(cloud, name), cfg


def rows_of(cloud, out):
    """Rows of `cloud` that the output rows came from: the intensity column is a permutation of k / 65536."""
    key = lambda a: np.rint(np.asarray(a, np.float64) * 65536.0).astype(np.int64)  # noqa: E731
    return np.argsort(key(cloud[:, 3]))[key(out)]


def assert_matches_fixture(fx, name, f, cloud, ts, rows, points, ts_out, source_rows=None):
    """One prepared frame against prep_kitti.npz: the kept rows (bit mask, with the ordered ids by digest), the
    timestamps and extra columns that travel with them, the coordinates (exact without correction, 1e-6 relative on
    the sampled rows with it) and the source rows (digest)."""
    key = f"{name}.f{f}."
    kept = np.unpackbits(fx[key + "kept"])[: cloud.shape[0]].astype(bool)
    assert np.array_equal(np.isin(np.arange(cloud.shape[0]), rows), kept), "kept rows differ"
    assert rows.shape[0] == kept.sum() and digest(rows) == str(fx[key + "survivors_sha256"]), "survivor order differs"
    assert np.array_equal(np.asarray(ts_out).reshape(-1), ts.reshape(-1)[rows])
    assert np.array_equal(points[:, 3:], cloud[rows, 3:])
    if key + "sample" in fx.files:
        ref = fx[key + "sample_xyz"]
        got = points[fx[key + "sample"], :3]
        assert rel_err(got, ref, np.linalg.norm(ref, axis=1, keepdims=True)).max() <= 1e-6
        assert not np.array_equal(got, cloud[rows[fx[key + "sample"]], :3])  # the correction moved them
    else:
        assert np.array_equal(points, cloud[rows])
    if f:
        assert digest(source_rows) == str(fx[key + "source_sha256"]), "source rows differ"


def rel_err(a, b, scale):
    return np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) / np.maximum(scale, 1e-30)


# --------------------------------------------------------------------------------------
# CPU
# --------------------------------------------------------------------------------------
def test_frame_kernel_ledger():
    """Every kernel defined in pin_slam_b200/csrc/frame is in FRAME_KERNEL_LEDGER, named by a test of this file that
    exists, and the ledger names no kernel that is gone (the library-wide ledger parser, pointed at the module)."""
    from tests import test_map_kernels as tmk

    old = tmk.CSRC
    tmk.CSRC = FRAME_CSRC
    try:
        found = tmk.global_kernels()
    finally:
        tmk.CSRC = old
    assert found == set(FRAME_KERNEL_LEDGER), (sorted(found - set(FRAME_KERNEL_LEDGER)),
                                               sorted(set(FRAME_KERNEL_LEDGER) - found))
    src = open(os.path.abspath(__file__)).read()
    for kernel, test in FRAME_KERNEL_LEDGER.items():
        assert re.search(rf"^def {test}\(", src, re.M), (kernel, test)


@pytest.mark.parametrize("name", ["kitti", "run"])
@pytest.mark.parametrize("f", [0, 1])
def test_oracle_matches_reference_preprocess_frame(name, f):
    fx = np.load(FIXTURE)
    cloud, ts, cfg = fixture_frame(fx, name, f)
    got = fo.prepare_frame(cloud, ts, cfg, f)
    assert got["rows"].shape[0] > 40000
    assert_matches_fixture(fx, name, f, cloud, ts, got["rows"], got["points"], got["ts"], got.get("source_rows"))


@pytest.mark.parametrize("angle", [1e-9, 1e-3, 1.0, 3.0])
def test_deskew_oracle_matches_scipy(angle):
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(int(angle * 1e3) + 5)
    axis = rng.normal(size=3)
    R = Rotation.from_rotvec(angle * axis / np.linalg.norm(axis)).as_matrix()
    # the logarithm and the exponential on an orthonormal matrix
    w = fo.rotation_log(R)
    assert np.abs(w - Rotation.from_matrix(R).as_rotvec()).max() <= 1e-14 + 1e-12 * angle
    s = np.linspace(-0.5, 0.5, 101)
    assert np.abs(fo.rotation_exp(s[:, None] * w) - Rotation.from_rotvec(s[:, None] * w).as_matrix()).max() <= 1e-15
    # end to end with the fp32 pose the reference passes; it is orthonormal to ~1e-7 only, and scipy projects it onto
    # a rotation in its own way
    pose = np.eye(4)
    pose[:3, :3], pose[:3, 3] = R, [0.7, -0.2, 0.05]
    pose = pose.astype(np.float32)
    n = 4096
    p = rng.uniform(-60, 60, (n, 3)).astype(np.float32)
    ts = rng.random(n).astype(np.float32)
    got = fo.deskew(p, ts, pose)
    s = fo.deskew_fraction(ts).astype(np.float64)
    assert s.min() == -0.5 and s.max() == 0.5
    P = pose.astype(np.float64)
    rots = Rotation.from_rotvec(s[:, None] * Rotation.from_matrix(P[:3, :3]).as_rotvec()[None, :])
    ref = rots.apply(p.astype(np.float64)) + s[:, None] * P[:3, 3]
    assert np.abs(got - ref).max() <= 1e-8 * 60


def test_patch_reference_dataset_rebinds_and_rejects_semantic_labels():
    from pin_slam_b200.dataset import slam_dataset as ds

    class SLAMDataset:
        def preprocess_frame(self):
            return "reference"

    mod = types.SimpleNamespace(SLAMDataset=SLAMDataset, deskewing=lambda *a: "reference")
    ds.patch_reference_dataset(mod)
    assert mod.SLAMDataset.preprocess_frame is ds.preprocess_frame and mod.deskewing is ds.deskewing
    frame = SLAMDataset()
    frame.cur_sem_labels_torch = torch.zeros(3, dtype=torch.int64)
    with pytest.raises(NotImplementedError):
        frame.preprocess_frame()
    pts = torch.ones(4, 3)
    assert ds.deskewing(pts, None, torch.eye(4)) is pts  # no timestamps: unchanged, as the reference


# --------------------------------------------------------------------------------------
# GPU
# --------------------------------------------------------------------------------------
def crop_inputs(n, seed, cols=5):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-90, 90, (n, cols)).astype(np.float32)
    pts[:, 2] = rng.uniform(-6, 12, n).astype(np.float32)
    if n >= 8:  # rows on the bounds (min_range 5, min_z -3.5, max_z 10): all excluded
        pts[0, :3] = (3, 4, 0)
        pts[1, :3] = (6, 0, -3.5)
        pts[2, :3] = (6, 0, 10)
        pts[3, :3] = (0, 0, 0)
        pts[4, :3] = (6, 0, 0)  # kept
    m = n + n // 3
    index = np.concatenate([np.arange(n), rng.integers(0, n, m - n)]) if n else np.zeros(0, np.int64)
    rng.shuffle(index[8:])
    ts = rng.random(n).astype(np.float32)
    return pts, index.astype(np.int64), ts


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 65536, 262144, 3_000_000])
def test_crop_matches_oracle(n):
    from pin_slam_b200 import ops

    pts, index, ts = crop_inputs(n, n + 1)
    bounds = dict(min_z=-3.5, max_z=10.0, min_range=5.0, max_range=80.0)
    P, I, T = torch.from_numpy(pts).cuda(), torch.from_numpy(index).cuda(), torch.from_numpy(ts).cuda()
    for deg in (0.0, 0.195):
        out, ts_out = ops.frame_crop(P, I, T, correction_deg=deg, **bounds)
        ref, ref_ts, rows = fo.frame_crop(pts, index, ts, correction_deg=deg, **bounds)
        out, ts_out = out.cpu().numpy(), ts_out.cpu().numpy()
        assert out.shape == ref.shape and np.array_equal(ts_out, ref_ts)
        assert np.array_equal(out[:, 3:], ref[:, 3:])  # the extra columns travel: equal rows in equal order
        if n >= 8:
            assert not np.isin([0, 1, 2, 3], rows).any() and 4 in rows
        r = np.linalg.norm(ref[:, :3].astype(np.float64), axis=1, keepdims=True)
        if deg == 0.0:
            assert np.array_equal(out, ref)
        elif n:
            assert rel_err(out[:, :3], ref[:, :3], r).max() <= 1e-6
        if n == 3_000_000:
            assert_launched(lambda: ops.frame_crop(P, I, T, correction_deg=deg, **bounds), "test_crop_matches_oracle")
        # without timestamps
        out2, none = ops.frame_crop(P, I, None, correction_deg=deg, **bounds)
        assert none is None and np.array_equal(out2.cpu().numpy(), out)


@pytest.mark.gpu
def test_deskew_matches_fp64_oracle():
    from scipy.spatial.transform import Rotation

    from pin_slam_b200 import ops

    rng = np.random.default_rng(3)
    n = 200_000
    base = rng.uniform(-80, 80, (n, 4)).astype(np.float32)
    ts = rng.random(n).astype(np.float32)
    T = torch.from_numpy(ts).cuda()
    for angle in (1e-9, 1e-3, 0.05, 1.0, 3.0):
        axis = rng.normal(size=3)
        pose = np.eye(4)
        pose[:3, :3] = Rotation.from_rotvec(angle * axis / np.linalg.norm(axis)).as_matrix()
        pose[:3, 3] = rng.normal(0, 1.5, 3)
        pose = pose.astype(np.float32)
        P = torch.from_numpy(base).cuda()
        view = P[:, :3]  # the reference deskews the view cloud[:, :3] in place
        ops.deskew_(view, T, torch.from_numpy(pose).cuda())
        got = P.cpu().numpy()
        ref = fo.deskew(base, ts, pose)
        bound = 1e-6 * (np.linalg.norm(base[:, :3].astype(np.float64), axis=1) + np.linalg.norm(pose[:3, 3])) + 1e-7
        err = np.linalg.norm(got[:, :3] - ref, axis=1)
        assert (err <= bound).all(), (angle, float((err / bound).max()))
        assert np.array_equal(got[:, 3], base[:, 3])  # column 3 untouched
    pose_t = torch.from_numpy(pose).cuda()
    assert_launched(lambda: ops.deskew_(torch.from_numpy(base).cuda()[:, :3], T, pose_t), "test_deskew_matches_fp64_oracle")
    # the identity pose leaves the points bit-identical
    P = torch.from_numpy(base).cuda()
    ops.deskew_(P[:, :3], T, torch.eye(4, device="cuda"))
    assert np.array_equal(P.cpu().numpy(), base)
    # all-equal timestamps: s = 0/0 = NaN, as torch gives
    P = torch.from_numpy(base[:1000]).cuda()
    ops.deskew_(P[:, :3], torch.full((1000, 1), 0.25, device="cuda"), torch.eye(4, device="cuda"))
    assert torch.isnan(P[:, :3]).all() and torch.equal(P[:, 3].cpu(), torch.from_numpy(base[:1000, 3]))


def bare_dataset(sd, cfg_values, name):
    """A reference SLAMDataset without a data loader, as tests/golden/make_golden_prep.py builds it."""
    from utils.config import Config

    cfg = Config()
    for k, v in cfg_values.items():
        setattr(cfg, k, v)
    cfg.device, cfg.silence, cfg.track_on, cfg.pgo_on, cfg.deskew = "cuda", True, True, False, False
    cfg.color_on = True  # cur_source_colors names the source rows (intensity column)
    cfg.setup_dtype()
    ds = sd.SLAMDataset.__new__(sd.SLAMDataset)
    ds.config, ds.silence, ds.device, ds.dtype = cfg, True, "cuda", cfg.dtype
    ds.odom_poses, ds.pgo_poses, ds.travel_dist = np.zeros((4, 4, 4)), None, np.zeros(4)
    ds.gt_pose_provided, ds.lose_track, ds.cur_sem_labels_torch = False, False, None
    ds.last_odom_tran, ds.cur_pose_ref = np.eye(4), np.eye(4)
    ds.stop_count, ds.consecutive_lose_track_frame = 0, 0
    return ds


def load_frame(ds, cloud, ts, f):
    ds.processed_frame = f
    ds.cur_point_cloud_torch = torch.from_numpy(cloud).cuda()
    ds.cur_point_ts_torch = torch.from_numpy(ts).cuda()


@pytest.mark.gpu
@pytest.mark.skipif(not fo.reference_dataset_available(), reason="oracle/_ref has no dataset/slam_dataset.py")
@pytest.mark.parametrize("name", ["kitti", "run"])
def test_patched_reference_chain(name):
    """The reference's own SLAMDataset with the drop-in preprocess_frame and deskewing: with deskew off it reproduces
    prep_kitti.npz; with deskew on, the source points (frame 1) and the mapping points of the reference's
    update_odom_pose equal the oracle chain, and lose_track leaves both undeskewed."""
    sd = fo.load_reference_dataset()
    from pin_slam_b200.dataset.slam_dataset import patch_reference_dataset

    patch_reference_dataset(sd)
    assert sd.deskewing.__module__ == "pin_slam_b200.dataset.slam_dataset"
    fx = np.load(FIXTURE)
    frames = [fixture_frame(fx, name, f) for f in (0, 1)]
    cfg_values = vars(frames[0][2]).copy()
    # deskew off: the fixture
    ds = bare_dataset(sd, cfg_values, name)
    for f, (cloud, ts, _) in enumerate(frames):
        load_frame(ds, cloud, ts, f)
        assert ds.preprocess_frame()
        got = ds.cur_point_cloud_torch.cpu().numpy()
        assert ds.cur_point_ts_torch.shape[1:] == ts.shape[1:]
        source_rows = rows_of(cloud, ds.cur_source_colors.cpu().numpy()[:, 0]) if f else None
        assert_matches_fixture(fx, name, f, cloud, ts, rows_of(cloud, got[:, 3]), got,
                               ds.cur_point_ts_torch.cpu().numpy(), source_rows)
        ds.last_odom_tran = np.eye(4)
        ds.last_odom_tran[:3, 3] = [0.8, 0.05, 0.0]
        ds.last_pose_ref = ds.cur_pose_ref
    # deskew on: frame 0, frame 1 (source deskewed with the motion guess), update_odom_pose (mapping points deskewed
    # with the tracked pose); then the same frame with lose_track
    motion = np.eye(4)
    motion[:3, :3] = fo_rot(0.04)
    motion[:3, 3] = [1.1, 0.1, 0.02]
    tracked = np.eye(4)
    tracked[:3, :3] = fo_rot(-0.03)
    tracked[:3, 3] = [0.9, -0.05, 0.01]
    for lose in (False, True):
        cv = dict(cfg_values, deskew=True)
        ds = bare_dataset(sd, cv, name)
        ds.config.deskew = True
        cfg = types.SimpleNamespace(**cv)
        load_frame(ds, *frames[0][:2], 0)
        assert ds.preprocess_frame()
        ds.last_odom_tran, ds.lose_track = motion, lose
        load_frame(ds, *frames[1][:2], 1)
        assert ds.preprocess_frame()
        ref = fo.prepare_frame(frames[1][0], frames[1][1], cfg, 1, motion, lose)
        pts = ds.cur_point_cloud_torch.cpu().numpy()
        assert np.array_equal(pts[:, 3], frames[1][0][ref["rows"], 3])
        src = ds.cur_source_points.cpu().numpy()
        assert src.shape == ref["source"].shape
        scale = np.linalg.norm(ref["source"], axis=1) + np.linalg.norm(motion[:3, 3])
        assert (np.linalg.norm(src - ref["source"], axis=1) <= 1e-6 * scale + 1e-7).all()
        ds.update_odom_pose(torch.tensor(ds.last_pose_ref @ tracked, device="cuda"))
        mapped = ds.cur_point_cloud_torch.cpu().numpy()
        if lose:
            assert np.array_equal(mapped, pts)
        else:
            T32 = torch.tensor(ds.last_odom_tran, dtype=torch.float32).numpy()
            want = fo.deskew(pts, ds.cur_point_ts_torch.cpu().numpy(), T32)
            scale = np.linalg.norm(pts[:, :3].astype(np.float64), axis=1) + np.linalg.norm(T32[:3, 3])
            assert (np.linalg.norm(mapped[:, :3] - want, axis=1) <= 1e-6 * scale + 1e-7).all()
            assert np.array_equal(mapped[:, 3], pts[:, 3])


def fo_rot(yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
