import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def pytest_terminal_summary(terminalreporter, exitstatus, config):
    """How much of the gradient-parity allowances (fp64 slack, ReLU-kink rows; tests/test_cuda_parity.py) the run on
    THIS device actually used: written to gpurun_out/parity_slack.json and summarised on the terminal."""
    try:
        from tests import helpers
    except Exception:  # noqa: BLE001
        return
    log = helpers.PARITY_SLACK
    if not log:
        return
    import json

    agg = {}
    for e in log:
        a = agg.setdefault(e["test"], {"checks": 0, "elements": 0, "over_tight_bound": 0, "needed_fp64_slack": 0,
                                       "kink_rows_used": 0, "kink_rows_allowed": 0, "worst_err_over_tight_bound": 0.0})
        a["checks"] += 1
        for k in ("elements", "over_tight_bound", "needed_fp64_slack", "kink_rows_used", "kink_rows_allowed"):
            a[k] += e[k]
        a["worst_err_over_tight_bound"] = max(a["worst_err_over_tight_bound"], e["max_err_over_tight_bound"])
    terminalreporter.write_line("parity allowances used (elements over the tight bound / needing the fp64 slack / kink rows):")
    for name, a in sorted(agg.items()):
        terminalreporter.write_line(f"  {name}: {a['over_tight_bound']} / {a['needed_fp64_slack']} / "
                                    f"{a['kink_rows_used']} (allowed {a['kink_rows_allowed']}) of {a['elements']} elements, "
                                    f"worst err = {a['worst_err_over_tight_bound']:.2f} x tight bound")
    out = os.path.join(ROOT, "gpurun_out")
    if os.path.isdir(out):
        json.dump(agg, open(os.path.join(out, "parity_slack.json"), "w"), indent=1)
