"""Where the time of K1 (search launch + decode launch) goes at BASELINE cfg2 (200k queries, K = 8, F = 32, 2 x 64
decoder, d sdf / dq), the headline workload of bench.py:

  1. K1 time with d/dq and value-only, library defaults (CUDA events, L2 flushed before every step)
  2. per-kernel device time per step (torch.profiler with CUDA activities, a run of its own); with --out DIR the trace
     goes to DIR/exp_decode_trace.json
  3. per-role cycle table of wsq_decode_kernel: per warp, clock deltas of the phases of its role, summed over one
     profiled launch (ws_profile); the role of every warp is read from the counters, so the table follows the kernel

Section 2 counts the launches of the in-library spatial sort (histogram memset, sort_key_kernel, the scan's kernels,
sort_scatter_kernel) with K1.
With --presorted it also runs with the sort off (sort_min_queries 0), on the bench's random queries and on the same
queries pre-permuted in Python into Morton order of their 0.4 m cells: the best that sorting inside the library
could reach, without its cost.  --sort-sweep times K1 with the sort off and on over batch sizes (CUDA events, L2
flushed before every step), to place the default of sort_min_queries.

python scripts/exp_decode.py [--steps N] [--out DIR] [--presorted] [--sort-sweep]"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from pin_slam_b200 import _lib, ops
from pin_slam_b200.config import HotPathConfig
from pin_slam_b200.model import Decoder
from pin_slam_b200.synthetic import build_map, surface_queries

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20, help="steps of the profiled run")
ap.add_argument("--out", default=None, help="directory for the profiler trace")
ap.add_argument("--presorted", action="store_true",
                help="also profile, with the sort off, the queries pre-permuted into Morton order of their cells")
ap.add_argument("--sort-sweep", action="store_true", help="K1 time with the sort off / on over batch sizes")
args = ap.parse_args()

dev = torch.device("cuda:0")
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
cfg = HotPathConfig.cfg2(device=str(dev), feature_std=0.1, local_map_radius=1e4)
npm = build_map(cfg, n_surface=3_000_000, seed=0, extent=80.0)
torch.manual_seed(42)
dec = Decoder(cfg, cfg.geo_mlp_hidden_dim, cfg.geo_mlp_level, 1)
q = surface_queries(npm, 200000, seed=1, sigma=0.1)


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


# ---- 1. K1 with d/dq and value-only
o1 = {}
med, mn = timed(lambda: npm.query_sdf(q, dec, out=o1))
print(f"K1 (search + decode) cold-L2 median {med:.4f} ms, min {mn:.4f} ms", flush=True)
med, mn = timed(lambda: npm.query_sdf(q, dec, need_grad=False, out=o1))
print(f"value-only (need_grad=False) cold-L2 median {med:.4f} ms, min {mn:.4f} ms", flush=True)

# ---- 2. per-kernel device time
from torch.profiler import ProfilerActivity, profile

def morton_presort(x, cell=0.4):
    """x[argsort(key)], key = 30-bit Morton interleave of floor(x / cell) (10 bits per axis, wrapped)."""
    c = torch.floor(x / cell).long() & 1023
    key = torch.zeros(x.shape[0], dtype=torch.long, device=x.device)
    for b in range(10):
        for a in range(3):
            key |= ((c[:, a] >> b) & 1) << (3 * b + a)
    return x[torch.argsort(key)].contiguous()


def kernel_table(qq, label, trace_name):
    out = {}
    for _ in range(3):
        npm.query_sdf(qq, dec, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as tp:
        for _ in range(args.steps):
            flush.zero_()
            npm.query_sdf(qq, dec, out=out)
        torch.cuda.synchronize()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        tp.export_chrome_trace(os.path.join(args.out, trace_name))
    rows = []
    for e in tp.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            rows.append((t / args.steps, e.count / args.steps, e.key))
    print(f"{label}: device time per step over {args.steps} profiled steps (flush = the L2 flush between steps, "
          "not part of K1):")
    k1 = 0.0
    for t, n, name in sorted(rows, reverse=True):
        tag = "K1" if any(k in name for k in K1_KERNELS) else "flush"
        if tag == "K1":
            k1 += t
        print(f"  {t:9.1f} us  {n:5.2f} launches  [{tag:5s}] {name[:110]}")
    print(f"  {k1:9.1f} us  K1 kernels per step (sum)", flush=True)
    return out


K1_KERNELS = ("search_kernel", "wsq_decode_kernel", "sort_key_kernel", "DeviceScan", "sort_scatter_kernel", "Memset")
out = kernel_table(q, "random queries, library defaults", "exp_decode_trace.json")
if args.presorted:
    ops.set_option("sort_min_queries", 0)
    kernel_table(q, "random queries, sort off", "exp_decode_trace_unsorted.json")
    kernel_table(morton_presort(q), "Morton-presorted queries, sort off", "exp_decode_trace_presorted.json")
    ops.set_option("sort_min_queries", ops.SORT_MIN_QUERIES)
if args.sort_sweep:
    print("K1 cold-L2 time over batch sizes, sort off vs on (best of 3 alternating medians of 12 steps):")
    for n in (1024, 2048, 4096, 8192, 16384, 32768, 65536, 200000):
        qn = q[:n].contiguous()
        o3 = {}
        res = {0: [], 1: []}
        for rep in range(3):
            for on in (0, 1):
                ops.set_option("sort_min_queries", 1 if on else 0)
                res[on].append(timed(lambda: npm.query_sdf(qn, dec, out=o3), 15)[0])
        off, on = min(res[0]), min(res[1])
        print(f"  n {n:7d}: off {1e3 * off:8.1f} us  on {1e3 * on:8.1f} us  ({100 * (on / off - 1):+.1f} %)", flush=True)
    ops.set_option("sort_min_queries", ops.SORT_MIN_QUERIES)

# ---- 3. per-role cycle table of one profiled launch of wsq_decode_kernel<32, true, true>
# role codes as written by wsq.cu (WS_ROLE_*) -> (name, slot names, indices of the slots that are waits)
ROLES = {
    1: ("C consumer", ["wait_A", "layer0", "layer1", "last+out"], {0}),
    2: ("C consumer, adjoint schedule", ["wait_A", "value_rows", "adjoint", "tangents+out"], {0}),
    4: ("G gather + meta refill", ["wait_A_free", "wait_meta", "issue_loads", "reduce+store", "pos+fence",
                                   "meta_refill", "wait_search"], {0, 1, 6}),
}
N_CTA, N_WARP, N_SLOT = 132, 16, 8
ops.set_option("ws_profile", 1)
npm.query_sdf(q, dec, out=out)
torch.cuda.synchronize()
ops.set_option("ws_profile", 0)
buf = np.zeros(N_CTA * N_WARP * N_SLOT, dtype=np.uint64)
_lib.check(_lib.load().pinb200_debug_read(b"ws_profile", buf.ctypes.data, buf.size), "debug_read")
prof = buf.reshape(N_CTA, N_WARP, N_SLOT)
ran = prof[:, :, N_SLOT - 1].max(axis=1) > 0  # CTAs of the launch (grid <= SM count)
role_of = prof[ran][0, :, N_SLOT - 1].astype(int)
cyc = prof[ran][:, :, : N_SLOT - 1].astype(np.float64)
med = np.median(cyc, axis=0)  # [warp, slot] median over CTAs
launch = med.sum(axis=1).max()
print(f"wsq_decode_kernel per-warp cycles, median over {int(ran.sum())} CTAs; longest warp {int(launch)} cycles")
for code in sorted(set(role_of.tolist())):
    name, slots, waits = ROLES[code]
    ws = [w for w in range(N_WARP) if role_of[w] == code]
    print(f"{name}: warps {ws[0]}-{ws[-1]}  ({', '.join(slots)})")
    for w in ws:
        row = med[w, : len(slots)]
        print(f"  warp {w:2d}: " + "  ".join(f"{int(v):9d}" for v in row) + f"   total {int(row.sum()):9d}")
    tot = med[ws, : len(slots)].sum(axis=0)
    share = tot / tot.sum()
    busy = 1.0 - sum(share[s] for s in waits)
    print("  share:   " + "  ".join(f"{100 * s:8.1f}%" for s in share) +
          f"   busy (not waiting on another role) {100 * busy:.1f}%", flush=True)
