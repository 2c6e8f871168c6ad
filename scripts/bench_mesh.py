"""Stage times of the device mesh path (DESIGN.md row f5) on the map of the KITTI-shaped synthetic frame loop.

    python scripts/bench_mesh.py [--frames 30] [--res 0.2] [--reps 5]

Builds the map with FrameLoop (run_kitti.yaml settings), then times with CUDA events around synchronised windows:
the dense grid query (Mesher.get_query_from_bbx + query_points), marching cubes (count / scan / emit, key unique,
vertex positions), the small-cluster filter (edge sort + union-find), and the whole Mesher.recon_aabb_mesh (with the
filter, normals and the host copy of the mesh).  It also times the float64 device-to-host copy of the grid that the
reference's path makes before skimage runs: a floor under the reference's cost, since skimage and Open3D are not
part of this project.  Prints one JSON line with the card's name and power limit beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True).strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, subprocess.CalledProcessError, ValueError):
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, reps):
    """Median ms of `fn` over `reps` runs after one warm-up, each between a synchronise and device events."""
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--res", type=float, default=0.2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh.py needs a CUDA device")

    from pin_slam_b200.frame_loop import FrameLoop
    from pin_slam_b200.utils.mesher import Mesher, marching_cubes, triangle_clusters

    loop = FrameLoop(device="cuda")
    loop.step(0, timed=False, map_iters=50)
    for f in range(1, args.frames):
        loop.step(f, timed=False)
    cfg = loop.cfg
    mesher = Mesher(cfg, loop.neural_points, {"sdf": loop.sdf_mlp, "semantic": None, "color": None})
    pts = loop.neural_points.neural_points.cpu().numpy().astype(np.float64)
    bbx = types.SimpleNamespace(get_min_bound=lambda: pts.min(0), get_max_bound=lambda: pts.max(0))
    min_nn = cfg.mesh_min_nn

    state = {}

    def query():
        coord, dims, origin = mesher.get_query_from_bbx(bbx, args.res, cfg.pad_voxel, cfg.skip_top_voxel)
        sdf, _, _, mask = mesher.query_points(coord, cfg.infer_bs, True, False, False, cfg.mc_mask_on, False, min_nn,
                                              out_torch=True)
        state.update(dims=dims, sdf=sdf, mask=mask)

    def mc():
        sdf, _, _, mask = mesher.assign_to_bbx(state["sdf"], None, None, state["mask"], state["dims"])
        state["verts"], state["faces"] = marching_cubes(sdf, mask)

    def clusters():
        _, size = triangle_clusters(state["faces"])
        state["keep"] = size >= cfg.min_cluster_vertices

    def d2h_f64():  # what the reference's query_points(out_torch=False) hands to skimage
        state["host"] = (state["sdf"].cpu().numpy().astype(np.float64), state["mask"].cpu().numpy().astype(np.float64))

    def recon():
        state["mesh"] = mesher.recon_aabb_mesh(bbx, args.res, None, False, False, False, True, True, True, min_nn)

    t_query = timed(query, args.reps)
    t_mc = timed(mc, args.reps)
    t_cl = timed(clusters, args.reps)
    t_copy = timed(d2h_f64, args.reps)
    t_total = timed(recon, args.reps)
    name, power = card()
    mesh = state["mesh"]
    print(json.dumps({
        "card": name, "power_limit": power, "frames": args.frames, "mc_res_m": args.res,
        "grid": [int(d) for d in state["dims"]], "grid_points": int(np.prod(state["dims"])),
        "masked_in": int(state["mask"].sum()), "map_points": int(pts.shape[0]),
        "triangles_mc": int(state["faces"].shape[0]), "vertices_mc": int(state["verts"].shape[0]),
        "triangles_kept": int(mesh.triangles.shape[0]), "vertices_kept": int(mesh.vertices.shape[0]),
        "ms": {"grid_query": round(t_query, 3), "marching_cubes": round(t_mc, 3), "cluster_filter": round(t_cl, 3),
               "recon_aabb_mesh": round(t_total, 3), "reference_f64_d2h_copy": round(t_copy, 3)},
        "reps": args.reps, "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
