"""A/B of the two decode variants of the split pipeline at BASELINE cfg2 (200k queries): python scripts/exp_decode.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pin_slam_b200 import ops
from pin_slam_b200.config import HotPathConfig
from pin_slam_b200.model import Decoder
from pin_slam_b200.synthetic import build_map, surface_queries

dev = torch.device("cuda:0")
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
cfg = HotPathConfig.cfg2(device=str(dev), feature_std=0.1, local_map_radius=1e4)
npm = build_map(cfg, n_surface=3_000_000, seed=0, extent=80.0)
torch.manual_seed(42)
dec = Decoder(cfg, cfg.geo_mlp_hidden_dim, cfg.geo_mlp_level, 1)
q = surface_queries(npm, 200000, seed=1, sigma=0.1)
ref = None


def timed(fn, n=10):
    ts = []
    for it in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts = sorted(ts[3:])
    return ts[len(ts) // 2], ts[0]


for variant in [int(a) for a in sys.argv[1:]] or [0, 1]:
    ops.set_option("decode_variant", variant)
    out = {}
    ts = []
    for it in range(10):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        npm.query_sdf(q, dec, out=out)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts = sorted(ts[3:])
    line = f"variant {variant}: K1 (search + decode) cold-L2 median {ts[len(ts) // 2]:.4f} ms, min {ts[0]:.4f} ms"
    if ref is None:
        ref = {k: v.clone() for k, v in out.items() if torch.is_tensor(v) and not k.startswith("_")}
    else:
        ds = (out["sdf"] - ref["sdf"]).abs().max().item()
        dg = (out["grad"] - ref["grad"]).abs().max().item()
        line += f"; vs first variant: max |d sdf| {ds:.3e}, max |d grad| {dg:.3e} (|grad| mean {ref['grad'].abs().mean().item():.3e})"
    print(line, flush=True)
    o2 = {}
    med, mn = timed(lambda: npm.query_sdf(q, dec, need_grad=False, out=o2))
    print(f"variant {variant}: value-only (need_grad=False) cold-L2 median {med:.4f} ms, min {mn:.4f} ms", flush=True)

# per-warp phase cycle counters of the warp-specialised decode (one profiled launch)
import numpy as np
from pin_slam_b200 import _lib
ops.set_option("decode_variant", 1)
ops.set_option("ws_profile", 1)
npm.query_sdf(q, dec, out=out)
torch.cuda.synchronize()
ops.set_option("ws_profile", 0)
buf = np.zeros(132 * 16 * 8, dtype=np.uint64)
_lib.check(_lib.load().pinb200_debug_read(b"ws_profile", buf.ctypes.data, buf.size), "debug_read")
prof = buf.reshape(132, 16, 8).astype(np.float64)
names = {"E": ["wait_mma0", "epi0", "-", "wait_mma1", "epi1", "outputs"], "M": ["wait_A1", "wait_D1free", "issue_L1", "wait_Atile", "issue_L0"], "G": ["wait_A_free", "wait_meta", "issue_loads", "reduce+store", "pos+fence"],
         "L": ["wait_meta_free", "stash_loads", "seeds+store"]}
for role, ws in (("E", range(0, 8)), ("G", range(8, 16)), ("L", range(16, 18)), ("M", range(18, 20))):
    med = np.median(prof[:, list(ws), :], axis=0)  # [warps, slots] median over CTAs
    print(role, "median cycles per warp over the launch (", ", ".join(names[role]), "):")
    for w, row in zip(ws, med):
        print(f"  warp {w:2d}: " + "  ".join(f"{int(v):8d}" for v in row[:len(names[role])]) + f"   total {int(row.sum()):8d}")
