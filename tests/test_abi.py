"""CPU-side checks of the C-ABI boundary: the library loads, exports every symbol
include/pinb200.h declares, and the ctypes mirror agrees with the header."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "pinb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pinb200_[a-z0-9_]+)\s*\(", src)))


def header_struct_fields(name):
    src = open(os.path.join(ROOT, "include", "pinb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        m = re.search(r"([A-Za-z_][A-Za-z0-9_]*)\s*(\[[A-Z0-9_]+\])?$", decl)
        fields.append(m.group(1))
    return fields


def test_library_exports_every_declared_symbol():
    from pin_slam_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    lib = _lib.load()
    names = header_functions()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/pinb200.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes prototype"
    assert sorted(_lib.SIGNATURES) == names
    assert lib.pinb200_version() == 200


@pytest.mark.parametrize("cname,pyname", [("pinb200_map_view", "MapView"), ("pinb200_decoder_view", "DecoderView"),
                                          ("pinb200_query_opts", "QueryOpts"), ("pinb200_query_out", "QueryOut"),
                                          ("pinb200_gn_opts", "GnOpts"), ("pinb200_map_train_opts", "MapTrainOpts")])
def test_ctypes_structs_mirror_header(cname, pyname):
    from pin_slam_b200 import _lib

    py = [f[0] for f in getattr(_lib, pyname)._fields_]
    assert py == header_struct_fields(cname)


def test_struct_sizes_match_c_compiler(tmp_path):
    """Compile a tiny C program against the header and compare sizeof() with ctypes."""
    import subprocess

    from pin_slam_b200 import _lib

    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "pinb200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n",'
                   "sizeof(pinb200_map_view),sizeof(pinb200_decoder_view),sizeof(pinb200_query_opts),"
                   "sizeof(pinb200_query_out),sizeof(pinb200_gn_opts),sizeof(pinb200_map_train_opts));return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).split()
    sizes = [int(x) for x in out]
    assert sizes == [ctypes.sizeof(_lib.MapView), ctypes.sizeof(_lib.DecoderView), ctypes.sizeof(_lib.QueryOpts),
                     ctypes.sizeof(_lib.QueryOut), ctypes.sizeof(_lib.GnOpts), ctypes.sizeof(_lib.MapTrainOpts)]


def test_no_cpu_fallback():
    """The product path must refuse CPU tensors instead of silently computing on the host."""
    import torch

    from pin_slam_b200 import ops

    with pytest.raises(RuntimeError):
        ops._ptr(torch.zeros(3))


def test_install_registers_reference_module_names():
    """install() makes the reference's import statements resolve to the drop-in classes (INTEGRATION.md)."""
    import subprocess
    import sys

    code = ("import sys; sys.path.insert(0, %r); import pin_slam_b200.install as i; i.install(tracker_and_mapper=True); "
            "import importlib as il; "
            "from model.neural_points import NeuralPoints; from model.decoder import Decoder; "
            "T = il.import_module('utils.tracker').Tracker; M = il.import_module('utils.mapper').Mapper; "
            "print(NeuralPoints.__module__, Decoder.__module__, T.__module__, M.__module__)") % ROOT
    out = subprocess.check_output([sys.executable, "-c", code]).decode().split()
    assert out == ["pin_slam_b200.model.neural_points", "pin_slam_b200.model.decoder", "pin_slam_b200.utils.tracker",
                   "pin_slam_b200.utils.mapper"]


def test_run_time_options_split_rule_and_workspace_sizes():
    """pinb200_set_option / ops.uses_split (no GPU needed: host-side state only): known options are accepted and
    mirrored in ops, unknown ones and out-of-range values fail loudly, workspace sizes cover stash + seeds."""
    from pin_slam_b200 import _lib, ops

    lib = _lib.load()
    assert ops.uses_split(2048, True) and not ops.uses_split(512, True)
    assert not ops.uses_split(20000, False) and ops.uses_split(40000, False)
    assert not ops.uses_split(20000, True, training_mode=True)  # mapper batches keep the general threshold
    ops.set_option("split_min_queries", 64)
    try:
        assert ops.uses_split(64, True) and ops.uses_split(64, False)
    finally:
        ops.set_option("split_min_queries", 0)
    assert ops.SPLIT_MIN_QUERIES == 32768 and ops.SPLIT_MIN_QUERIES_WF == 1024
    ops.set_option("split_min_queries_wf", 4096)
    assert not ops.uses_split(2048, True)
    ops.set_option("split_min_queries_wf", 0)
    with pytest.raises(RuntimeError):
        ops.set_option("decode_variant", 1)  # one decode per configuration: no option selects it
    with pytest.raises(RuntimeError):
        ops.set_option("no_such_option", 1)
    # 32 queries per tile: stash (1536 floats) + forward-mode seeds (1056 floats)
    assert lib.pinb200_query_workspace_bytes(1) == (1536 + 1056) * 4
    assert lib.pinb200_query_workspace_bytes(33) == 2 * (1536 + 1056) * 4
    assert lib.pinb200_map_grow_scratch(1000) >= 3 * 1000 + 4
