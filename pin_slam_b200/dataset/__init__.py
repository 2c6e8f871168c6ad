"""Drop-in frame preparation for the reference's `dataset.slam_dataset` (see slam_dataset.py)."""
