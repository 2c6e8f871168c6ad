"""Make the reference's own import statements resolve to the CUDA drop-ins.

`pin_slam.py` (and utils/tracker.py, utils/mapper.py, utils/mesher.py ...) of the
reference import `from model.neural_points import NeuralPoints` and
`from model.decoder import Decoder`.  Calling `install()` before those imports
registers this package's modules under those names, so the reference driver runs
unchanged on top of the CUDA hot path (INTEGRATION.md)."""
import importlib
import sys


def install(tracker_and_mapper: bool = False) -> None:
    """Register the drop-in `model.neural_points` / `model.decoder` modules.

    tracker_and_mapper=True additionally registers the fused `utils.tracker` / `utils.mapper` modules under the
    reference's names, so `from utils.tracker import Tracker` / `from utils.mapper import Mapper` in the reference
    driver pick up the kernels' Tracker / Mapper (the other `utils.*` modules stay the reference's own)."""
    np_mod = importlib.import_module("pin_slam_b200.model.neural_points")
    dec_mod = importlib.import_module("pin_slam_b200.model.decoder")
    sys.modules["model.neural_points"] = np_mod
    sys.modules["model.decoder"] = dec_mod
    if "model" in sys.modules:
        sys.modules["model"].neural_points = np_mod
        sys.modules["model"].decoder = dec_mod
    if tracker_and_mapper:
        trk = importlib.import_module("pin_slam_b200.utils.tracker")
        mpr = importlib.import_module("pin_slam_b200.utils.mapper")
        sys.modules["utils.tracker"] = trk
        sys.modules["utils.mapper"] = mpr
        if "utils" in sys.modules:
            sys.modules["utils"].tracker = trk
            sys.modules["utils"].mapper = mpr
