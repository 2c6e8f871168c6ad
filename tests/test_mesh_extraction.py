"""Mesh extraction (DESIGN.md row f5): the marching-cubes rules and the small-cluster filter restated by
oracle/mesh_oracle.py (CPU tests), and the CUDA kernels behind the drop-in Mesher against that oracle with `==`
(GPU tests)."""
import os
import re
import types

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from tests.helpers import kernels_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MESH_CSRC = os.path.join(ROOT, "pin_slam_b200", "csrc", "mesh")

# kernel ledger of the mesh module (pin_slam_b200/csrc/mesh): every __global__ kernel there is named by a test of this
# file, and that test checks that it launched it
MESH_KERNEL_LEDGER = {
    "mc_count_kernel": "test_large_quantised_field_with_random_mask_matches_oracle",
    "mc_scan_kernel": "test_large_quantised_field_with_random_mask_matches_oracle",
    "mc_emit_kernel": "test_large_quantised_field_with_random_mask_matches_oracle",
    "mc_vertex_kernel": "test_large_quantised_field_with_random_mask_matches_oracle",
    "uf_init_kernel": "test_cluster_filter_matches_oracle",
    "uf_union_kernel": "test_cluster_filter_matches_oracle",
    "uf_root_kernel": "test_cluster_filter_matches_oracle",
}


def assert_launched(names, test):
    want = [k for k, v in MESH_KERNEL_LEDGER.items() if v == test]
    assert want
    missing = [k for k in want if not any(re.search(rf"\bpinb::{k}\b", n) for n in names)]
    assert not missing, (missing, sorted(n for n in names if "pinb::" in n))


def ball(n, center, radius):
    g = np.indices((n, n, n)).astype(np.float64)
    return (np.sqrt(((g - np.reshape(center, (3, 1, 1, 1))) ** 2).sum(0)) - radius).astype(np.float32)


def torus(n, center, big, small):
    g = np.indices((n, n, n)).astype(np.float64) - np.reshape(center, (3, 1, 1, 1))
    q = np.sqrt(g[0] ** 2 + g[1] ** 2) - big
    return (np.sqrt(q ** 2 + g[2] ** 2) - small).astype(np.float32)


def euler(verts, faces):
    e = np.unique(np.sort(faces[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2), 1), axis=0).shape[0]
    return verts.shape[0] - e + faces.shape[0]


def face_normals(verts, faces):
    v = verts[faces]
    return np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])


def quantised_field(n, seed, step=0.25):
    """Smooth seeded field rounded to multiples of `step`: many corners exactly 0."""
    rng = np.random.default_rng(seed)
    x = np.linspace(0.0, 6.0, n, dtype=np.float64)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    a = rng.uniform(0.5, 1.5, 6)
    f = np.sin(a[0] * X + a[1]) * np.cos(a[2] * Y) + np.sin(a[3] * Z + a[4] * X) + 0.3 * np.cos(a[5] * (X + Y + Z))
    return (np.round(f * 4.0 / (4.0 * step)) * step).astype(np.float32)


# --------------------------------------------------------------------------------------
# CPU: the oracle pins the rules
# --------------------------------------------------------------------------------------
def test_mesh_kernel_ledger():
    """Every kernel defined in pin_slam_b200/csrc/mesh is in MESH_KERNEL_LEDGER, named by a test of this file that
    exists, and the ledger names no kernel that is gone (the parser of the library-wide kernel ledger, pointed at the
    mesh module)."""
    from tests import test_map_kernels as tmk

    old = tmk.CSRC
    tmk.CSRC = MESH_CSRC
    try:
        found = tmk.global_kernels()
    finally:
        tmk.CSRC = old
    assert found == set(MESH_KERNEL_LEDGER), (sorted(found - set(MESH_KERNEL_LEDGER)),
                                              sorted(set(MESH_KERNEL_LEDGER) - found))
    src = open(os.path.abspath(__file__)).read()
    for kernel, test in MESH_KERNEL_LEDGER.items():
        assert re.search(rf"^def {test}\(", src, re.M), (kernel, test)


def test_kernel_table_is_the_face_rule_table():
    src = open(os.path.join(MESH_CSRC, "mcubes.cu")).read()
    body = re.search(r"MC_TRI\[256\]\[16\] = \{(.*?)\n\};", src, flags=re.S).group(1)
    table = np.array([int(v) for v in re.findall(r"-?\d+", body)], np.int64).reshape(256, 16)
    ref = mo.mc_triangle_table()
    assert np.array_equal(table, ref)
    n_tri = (ref >= 0).sum(1) // 3
    assert int((n_tri > 0).sum()) == 254 and int(n_tri.max()) == 5
    assert np.all(ref[:, 15] == -1) and np.all((ref[:, 0:15:3] < 0) == (ref[:, 1:15:3] < 0))


@pytest.mark.parametrize("seed", range(4))
def test_random_fields_give_closed_consistently_oriented_surfaces(seed):
    n = 14
    sdf = np.random.default_rng(seed).standard_normal((n, n, n)).astype(np.float32)
    verts, faces, _ = mo.marching_cubes(sdf)
    assert faces.shape[0] > 1000
    directed = faces[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2)
    assert np.unique(directed, axis=0).shape[0] == directed.shape[0]  # every directed edge exactly once
    und, cnt = np.unique(np.sort(directed, 1), axis=0, return_counts=True)
    a, b = verts[und[:, 0]], verts[und[:, 1]]
    on_boundary = np.any(((a == 0) & (b == 0)) | ((a == n - 1) & (b == n - 1)), axis=1)
    assert np.all(cnt[~on_boundary] == 2)
    assert np.all(cnt[on_boundary] == 1)


def test_sphere_and_torus_topology_area_and_winding():
    r = 20.3
    c = np.array([24.4, 23.7, 24.1])
    verts, faces, _ = mo.marching_cubes(ball(50, c, r))
    assert euler(verts, faces) == 2
    fn = face_normals(verts, faces)
    area = 0.5 * np.linalg.norm(fn, axis=1).sum()
    assert abs(area / (4 * np.pi * r * r) - 1) < 0.01
    # right-hand normals point toward decreasing sdf (into the ball)
    assert np.all(np.einsum("ij,ij->i", fn, verts[faces].mean(1) - c) < 0)
    tv, tf, _ = mo.marching_cubes(torus(48, [23.6, 24.2, 23.9], 13.0, 5.2))
    assert euler(tv, tf) == 0


def test_exact_zero_corners_weld_and_leave_no_degenerate_triangle():
    sdf = np.round(ball(30, [14.5, 14.2, 14.7], 9.6) * 2.0) / 2.0  # many corners exactly 0 (and -0)
    sdf = sdf.astype(np.float32)
    assert (sdf == 0).sum() > 100
    verts, faces, keys = mo.marching_cubes(sdf)
    n = sdf.size
    assert np.all((faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2]))
    assert np.unique(verts, axis=0).shape[0] == verts.shape[0]  # one vertex per position
    on_grid = keys >= 3 * n
    assert on_grid.sum() > 100
    q = keys[on_grid] - 3 * n
    assert np.all(sdf.reshape(-1)[q] == 0)
    assert np.array_equal(verts[on_grid], np.stack(np.unravel_index(q, sdf.shape), 1).astype(np.float64))
    # the welded mesh of the quantised ball is still one closed surface
    assert euler(verts, faces) == 2


def test_mask_is_read_at_the_lowest_corner_of_each_cube():
    sdf = np.ones((3, 3, 3), np.float32)
    sdf[1, 1, 1] = -1.0  # inside corner shared by all eight cubes
    assert mo.marching_cubes(sdf)[1].shape[0] == 8
    for at, n_tri in (((0, 0, 0), 1), ((1, 1, 1), 1), ((0, 1, 0), 1), ((2, 2, 2), 0), ((1, 2, 1), 0)):
        mask = np.zeros((3, 3, 3), bool)
        mask[at] = True
        verts, faces, keys = mo.marching_cubes(sdf, mask)
        assert faces.shape[0] == n_tri, at
        if n_tri:  # the one triangle is on the three edges of (1,1,1) inside cube `at`
            assert np.all(np.abs(verts - 1.0).sum(1) == 0.5)
    sdf[1, 1, 1] = 0.0  # exactly the level: outside
    assert mo.marching_cubes(sdf)[1].shape[0] == 0


def strips(sizes, seed):
    """Triangle strips (i, i+1, i+2) of the given triangle counts, vertex-disjoint, triangles shuffled."""
    faces, base = [], 0
    for s in sizes:
        i = np.arange(s)
        faces.append(np.stack([i, i + 1, i + 2], 1) + base)
        base += s + 2
    f = np.concatenate(faces)
    # two triangles touching at one vertex only: two clusters
    f = np.concatenate([f, [[base, base + 1, base + 2], [base + 2, base + 3, base + 4]]])
    return f[np.random.default_rng(seed).permutation(f.shape[0])]


def flood_fill_clusters(faces):
    edge_tris = {}
    for t, f in enumerate(faces):
        for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
            edge_tris.setdefault((min(a, b), max(a, b)), []).append(t)
    nbr = [[] for _ in range(len(faces))]
    for ts in edge_tris.values():
        for t in ts:
            nbr[t] += ts
    lab = -np.ones(len(faces), np.int64)
    k = 0
    for s in range(len(faces)):
        if lab[s] >= 0:
            continue
        stack, lab[s] = [s], k
        while stack:
            for u in nbr[stack.pop()]:
                if lab[u] < 0:
                    lab[u] = k
                    stack.append(u)
        k += 1
    return lab


def test_mesh_clusters_match_flood_fill():
    rng = np.random.default_rng(3)
    faces = strips(list(rng.integers(1, 30, 60)) + [300, 299], 4)
    sdf = np.random.default_rng(5).standard_normal((9, 9, 9)).astype(np.float32)
    _, mc_faces, _ = mo.marching_cubes(sdf)
    for f in (faces, mc_faces):
        lab, size = mo.mesh_clusters(f)
        ref = flood_fill_clusters(f)
        assert np.array_equal(lab, ref)
        assert np.array_equal(size, np.bincount(ref))
    assert sorted(mo.mesh_clusters(faces)[1])[-2:] == [299, 300]


def read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    assert head[1] == "format binary_little_endian 1.0"
    types_ = {"double": "<f8", "uchar": "u1", "int": "<i4", "float": "<f4"}
    elems, cur = [], None
    for line in head:
        w = line.split()
        if w and w[0] == "element":
            cur = [w[1], int(w[2]), []]
            elems.append(cur)
        elif w and w[0] == "property" and w[1] != "list":
            cur[2].append((w[2], types_[w[1]]))
    vname, nv, vfields = elems[0]
    vert = np.frombuffer(data, dtype=vfields, count=nv, offset=end)
    face = np.frombuffer(data, dtype=[("n", "u1"), ("v", "<i4", (3,))], count=elems[1][1], offset=end + vert.nbytes)
    assert np.all(face["n"] == 3)
    return vert, face["v"]


def test_ply_round_trip(tmp_path):
    from pin_slam_b200.utils.mesher import TriangleMesh, write_ply

    verts, faces, _ = mo.marching_cubes(ball(16, [7.3, 7.6, 7.4], 5.1))
    mesh = TriangleMesh(verts * 0.1 + np.array([1.0, -2.0, 3.0]), faces)
    mesh.vertex_colors = np.random.default_rng(0).random(verts.shape)
    mesh.compute_vertex_normals()
    path = str(tmp_path / "m.ply")
    write_ply(path, mesh)
    vert, tri = read_ply(path)
    assert np.array_equal(np.stack([vert["x"], vert["y"], vert["z"]], 1), mesh.vertices)
    assert np.array_equal(np.stack([vert["nx"], vert["ny"], vert["nz"]], 1), mesh.vertex_normals)
    rgb = np.stack([vert["red"], vert["green"], vert["blue"]], 1)
    assert np.array_equal(rgb, np.round(mesh.vertex_colors * 255).astype(np.uint8))
    assert np.array_equal(tri, faces)
    # normals of the ball point inward (decreasing sdf) and are unit length
    assert np.allclose(np.linalg.norm(mesh.vertex_normals, axis=1), 1.0)
    assert np.all(np.einsum("ij,ij->i", mesh.vertex_normals, verts - [7.3, 7.6, 7.4]) < 0)


def test_mesh_merge_and_triangle_selection():
    from pin_slam_b200.utils.mesher import TriangleMesh

    a = TriangleMesh([[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 1, 2]])
    b = TriangleMesh([[1, 0, 0], [0, 1, 0], [1, 1, 0], [5, 5, 5]], [[0, 2, 1]])
    a.vertex_colors = np.full((3, 3), 0.25)
    b.vertex_colors = np.full((4, 3), 0.75)
    a += b
    a.remove_duplicated_vertices()
    assert np.array_equal(a.vertices, [[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [5, 5, 5]])
    assert np.array_equal(a.triangles, [[0, 1, 2], [1, 3, 2]])
    assert np.array_equal(a.vertex_colors[:, 0], [0.25, 0.25, 0.25, 0.75, 0.75])  # first occurrence wins
    a.select_triangles([False, True])
    assert np.array_equal(a.vertices, [[1, 0, 0], [0, 1, 0], [1, 1, 0]])
    assert np.array_equal(a.triangles, [[0, 2, 1]]) and a.vertex_colors.shape == (3, 3)


def test_install_registers_the_mesher():
    import subprocess
    import sys

    code = ("import sys; sys.path.insert(0, %r); import pin_slam_b200.install as i; i.install(mesher=True); "
            "import importlib as il; print(il.import_module('utils.mesher').Mesher.__module__)") % ROOT
    assert subprocess.check_output([sys.executable, "-c", code]).decode().split() == ["pin_slam_b200.utils.mesher"]


# --------------------------------------------------------------------------------------
# GPU: kernels against the oracle
# --------------------------------------------------------------------------------------
def fixture_mesher(name, **cfg_kw):
    from pin_slam_b200 import ops
    from pin_slam_b200.config import HotPathConfig
    from pin_slam_b200.utils.mesher import Mesher
    from tests.helpers import decoder_from_fixture, decoder_handle_from_oracle, load_npz, map_from_fixture, map_handle_from_oracle

    fx = load_npz(name)
    m = map_from_fixture(fx)
    color = "mesh.color" in fx
    k, wf = int(fx["cfg.query_nn_k"]), bool(fx["cfg.weighted_first"])
    mh = map_handle_from_oracle(m, False)
    dh = decoder_handle_from_oracle(decoder_from_fixture(fx, "sdf_mlp"))
    ch = decoder_handle_from_oracle(decoder_from_fixture(fx, "color_mlp"), sigmoid_out=True) if color else None

    class _Points:  # the members Mesher touches
        neural_points = mh.keep["points"]

        @staticmethod
        def query_sdf(q, sdf_dec, query_locally=False, need_grad=False, color_decoder=None, out=None):
            return ops.query_sdf(mh, dh, q, nn_k=k, weighted_first=wf, need_grad=False, color_dec=color_decoder, out=out)

    cfg = HotPathConfig(device="cuda", color_on=color, color_channel=3 if color else 0, **cfg_kw)
    bbx = types.SimpleNamespace(get_min_bound=lambda: fx["grid"].min(0).astype(np.float64),
                                get_max_bound=lambda: fx["grid"].max(0).astype(np.float64))
    return Mesher(cfg, _Points, {"sdf": None, "semantic": None, "color": ch}), bbx


def assert_kernel_matches_oracle(sdf, mask, level=0.0):
    from pin_slam_b200 import ops
    from pin_slam_b200.utils.mesher import marching_cubes

    keys = ops.mc_triangle_keys(sdf, mask, level)
    verts, faces = marching_cubes(sdf, mask, level)
    torch.cuda.synchronize()
    rv, rf, rk = mo.marching_cubes(sdf.cpu().numpy(), None if mask is None else mask.cpu().numpy(), level)
    assert np.array_equal(keys.cpu().numpy(), rk[rf].reshape(-1, 3))
    assert np.array_equal(faces.cpu().numpy(), rf)
    assert np.array_equal(verts.cpu().numpy(), rv)  # float64 positions, bit for bit
    return rv, rf


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mesh_kitti_nwf", "mesh_replica_wf_color"])
def test_fixture_grids_match_oracle(name):
    mesher, bbx = fixture_mesher(name)
    coord, dims, _ = mesher.get_query_from_bbx(bbx, 0.1, 0, 0)
    sdf, _, _, mask = mesher.query_points(coord, 4096, True, False, False, True, mask_min_nn_count=4, out_torch=True)
    sdf, _, _, mask = mesher.assign_to_bbx(sdf, None, None, mask, dims)
    assert int(mask.sum()) > 1000 and int((sdf == 0).sum()) > 0
    sdf, mask = sdf.contiguous(), mask.contiguous()
    assert_kernel_matches_oracle(sdf, mask)
    assert_kernel_matches_oracle(sdf, None)
    # the KITTI fixture's decoder is positive everywhere inside the mask: also cut every map at its median masked sdf
    level = float(sdf[mask].median())
    for m in (mask, None):
        rv, rf = assert_kernel_matches_oracle(sdf, m, level)
        assert rf.shape[0] > 1000
    if name == "mesh_replica_wf_color":
        assert assert_kernel_matches_oracle(sdf, mask)[1].shape[0] > 1000


@pytest.mark.gpu
def test_large_quantised_field_with_random_mask_matches_oracle():
    n = 257  # 2^24 cubes: the block-sum scan runs over ~8200 blocks in 9 passes
    sdf = quantised_field(n, 7)
    assert (sdf == 0).mean() > 0.02
    mask = np.random.default_rng(8).random(sdf.shape) < 0.9
    sdf, mask = torch.from_numpy(sdf).cuda(), torch.from_numpy(mask).cuda()
    (rv, rf), names = kernels_run(lambda: assert_kernel_matches_oracle(sdf, mask))
    assert rf.shape[0] > 100000
    assert_launched(names, "test_large_quantised_field_with_random_mask_matches_oracle")


@pytest.mark.gpu
def test_degenerate_grids_give_empty_meshes():
    from pin_slam_b200.utils.mesher import marching_cubes

    ball_sdf = torch.from_numpy(ball(20, [9.5, 9.3, 9.6], 6.2)).cuda()
    cases = [(torch.ones(16, 16, 16, device="cuda"), None),  # no crossing
             (ball_sdf, torch.zeros(20, 20, 20, dtype=torch.bool, device="cuda")),  # everything masked out
             (ball_sdf[:, :, 9:10].contiguous(), None),  # one layer: no cube
             (torch.zeros(0, 4, 4, device="cuda"), None)]
    for sdf, mask in cases:
        verts, faces = marching_cubes(sdf, mask)
        torch.cuda.synchronize()
        assert verts.shape == (0, 3) and faces.shape == (0, 3)
    assert marching_cubes(ball_sdf)[1].shape[0] > 0


@pytest.mark.gpu
def test_full_size_sphere_is_closed_oriented_genus_zero():
    from pin_slam_b200.utils.mesher import marching_cubes

    n, r = 632, 300.37  # 631^3 = 2.5e8 cubes
    c = torch.tensor([315.61, 315.28, 315.83], dtype=torch.float64)
    x = torch.arange(n, dtype=torch.float32, device="cuda")
    d2 = ((x - float(c[0])) ** 2).view(-1, 1, 1) + ((x - float(c[1])) ** 2).view(1, -1, 1)
    sdf = d2 + ((x - float(c[2])) ** 2).view(1, 1, -1)
    del d2
    sdf.sqrt_().sub_(r)
    verts, faces = marching_cubes(sdf)
    del sdf
    torch.cuda.synchronize()
    f = faces.long()
    nv = verts.shape[0]
    directed = f[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2)
    dkey = torch.sort(directed[:, 0] * nv + directed[:, 1])[0]
    assert bool((dkey[1:] != dkey[:-1]).all())  # each directed edge once ...
    rkey = torch.sort(directed[:, 1] * nv + directed[:, 0])[0]
    assert bool((rkey == dkey).all())  # ... and its reverse once: closed and consistently oriented
    n_edges = directed.shape[0] // 2
    assert nv - n_edges + f.shape[0] == 2
    v = verts[f]
    cr = torch.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0], dim=1)
    area = 0.5 * float(cr.norm(dim=1).sum())
    assert abs(area / (4 * np.pi * r * r) - 1) < 1e-3
    volume = float((cr * (v[:, 0] - c.cuda())).sum()) / 6.0  # negative: normals point into the ball
    assert abs(-volume / (4.0 / 3.0 * np.pi * r ** 3) - 1) < 1e-3


@pytest.mark.gpu
def test_cluster_filter_matches_oracle():
    from pin_slam_b200.utils.mesher import TriangleMesh, triangle_clusters

    m = 300
    rng = np.random.default_rng(11)
    faces = strips(list(rng.integers(1, 80, 3000)) + [m, m - 1, m + 40], 12)
    _, mc_faces, _ = mo.marching_cubes(np.random.default_rng(13).standard_normal((40, 40, 40)).astype(np.float32))
    for f in (faces, mc_faces):
        lab, size = mo.mesh_clusters(f)
        (root, tri_size), names = kernels_run(lambda: triangle_clusters(torch.from_numpy(f).int().cuda()))
        assert_launched(names, "test_cluster_filter_matches_oracle")
        min_id = np.full(size.shape[0], f.shape[0])
        np.minimum.at(min_id, lab, np.arange(f.shape[0]))
        assert np.array_equal(root.cpu().numpy(), min_id[lab])
        assert np.array_equal(tri_size.cpu().numpy(), size[lab])
    mesher, _ = fixture_mesher("mesh_kitti_nwf")
    mesh = TriangleMesh(np.random.default_rng(1).random((faces.max() + 1, 3)), faces)
    kept = mesher.filter_isolated_vertices(mesh, m)
    lab, size = mo.mesh_clusters(faces)
    keep = size[lab] >= m
    assert kept.triangles.shape[0] == int(keep.sum())
    assert sorted(np.unique(mo.mesh_clusters(kept.triangles)[1])) == sorted(np.unique(size[size >= m]))
    assert m in mo.mesh_clusters(kept.triangles)[1] and m - 1 not in mo.mesh_clusters(kept.triangles)[1]
    assert kept.vertices.shape[0] == np.unique(kept.triangles).shape[0]  # unreferenced vertices compacted


@pytest.mark.gpu
def test_recon_mesh_vertex_colours_are_the_colour_query(tmp_path):
    from tests.test_mesh_extraction import read_ply

    mesher, bbx = fixture_mesher("mesh_replica_wf_color", pad_voxel=0, skip_top_voxel=0, min_cluster_vertices=20)
    path = str(tmp_path / "replica.ply")
    mesh = mesher.recon_aabb_mesh(bbx, 0.1, path, estimate_color=True, filter_isolated_mesh=True, mesh_min_nn=4)
    assert mesh.triangles.shape[0] > 1000 and mesh.has_vertex_colors() and mesh.has_vertex_normals()
    q = torch.from_numpy(mesh.vertices).float().cuda()
    _, _, col, _ = mesher.query_points(q, 4096, False, False, True, False, out_torch=True)
    np.testing.assert_allclose(mesh.vertex_colors, col.double().cpu().numpy(), rtol=1e-6, atol=1e-7)
    vert, tri = read_ply(path)
    assert np.array_equal(np.stack([vert["x"], vert["y"], vert["z"]], 1), mesh.vertices)
    assert np.array_equal(tri, mesh.triangles)
    # the 0.2 m drop-in call of the reference driver writes a mesh too
    mesh2 = mesher.recon_aabb_mesh(bbx, 0.2, str(tmp_path / "r2.ply"))
    assert mesh2.triangles.shape[0] > 0 and os.path.getsize(str(tmp_path / "r2.ply")) > 0


@pytest.mark.gpu
def test_collections_mesh_merges_overlapping_chunks():
    mesher, bbx = fixture_mesher("mesh_replica_wf_color")
    lo, hi = bbx.get_min_bound(), bbx.get_max_bound()
    mid = lo + 0.5 * (hi - lo)
    a = types.SimpleNamespace(get_min_bound=lambda: lo, get_max_bound=lambda: np.array([mid[0] + 1.0, hi[1], hi[2]]))
    b = types.SimpleNamespace(get_min_bound=lambda: np.array([mid[0] - 1.0, lo[1], lo[2]]), get_max_bound=lambda: hi)
    ma = mesher.recon_aabb_mesh(a, 0.1)
    mb = mesher.recon_aabb_mesh(b, 0.1)
    merged = mesher.recon_aabb_collections_mesh([a, b], 0.1)
    assert merged.vertices.shape[0] > 0
    assert np.unique(merged.vertices, axis=0).shape[0] == merged.vertices.shape[0]
    assert merged.vertices.shape[0] <= ma.vertices.shape[0] + mb.vertices.shape[0]
    assert merged.triangles.shape[0] == ma.triangles.shape[0] + mb.triangles.shape[0]
    assert merged.vertex_normals.shape == merged.vertices.shape
