#!/usr/bin/env python3
"""Recipe for the frame-preparation part of oracle/_ref: the UNMODIFIED reference `dataset/slam_dataset.py` and the
modules it imports, copied next to what oracle/make_ref.py copies, so that scripts/bench_frame_prep.py and the GPU
tests of tests/test_frame_prep.py can run the reference's own `SLAMDataset.preprocess_frame` / `update_odom_pose`
(oracle/frame_oracle.py: load_reference_dataset) where no reference checkout exists.

    python oracle/make_ref_frame.py [--src /root/reference]

`__graft_entry__.build()` runs it after oracle/make_ref.py whenever the reference checkout is present.
"""
import argparse
import os
import shutil

DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")  # as in oracle/make_ref.py

FILES = ["dataset/slam_dataset.py", "dataset/dataloaders/__init__.py", "eval/eval_traj_utils.py",
         "utils/semantic_kitti_utils.py"]


def make(src="/root/reference"):
    if not os.path.isdir(src):
        return False
    for rel in FILES:
        s, d = os.path.join(src, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        if (not os.path.exists(d)) or os.path.getmtime(s) > os.path.getmtime(d) or os.path.getsize(s) != os.path.getsize(d):
            shutil.copyfile(s, d)
    return True


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default="/root/reference")
    a = ap.parse_args()
    print("oracle/_ref frame preparation ready" if make(a.src) else f"{a.src} not found: not (re)built")
