"""The reference's mesher (utils/mesher.py of PRBonn/PIN_SLAM) on the GPU, without skimage or Open3D.

* `Mesher.query_points` (SURVEY.md section 8 row f3, utils/mesher.py:40-164): the per-batch `query_feature ->
  Decoder.sdf -> IDW sum` chain is ONE launch of K1 in global-map, no-gradient mode per chunk.
* `Mesher.recon_aabb_mesh` / `recon_aabb_collections_mesh` (DESIGN.md row f5, utils/mesher.py:507-649): the grid
  query, marching cubes (pinb200_mc_*), vertex colours and the small-cluster filter (pinb200_mesh_clusters) stay on the
  device; only the final mesh crosses to the host.  The result is a `TriangleMesh` with Open3D's legacy attribute names
  (`vertices`, `triangles`, `vertex_colors`, `vertex_normals`) and is written as binary little-endian PLY.
"""
import numpy as np
import torch

from .. import ops


class TriangleMesh:
    """Host mesh: vertices [V,3] float64, triangles [T,3] int32, vertex_colors / vertex_normals [V,3] float64 (or
    empty), the attributes of Open3D's legacy TriangleMesh that pin_slam.py and the GUI read."""

    def __init__(self, vertices=None, triangles=None):
        self.vertices = np.zeros((0, 3)) if vertices is None else np.asarray(vertices, np.float64).reshape(-1, 3)
        self.triangles = (np.zeros((0, 3), np.int32) if triangles is None
                          else np.asarray(triangles, np.int32).reshape(-1, 3))
        self.vertex_colors = np.zeros((0, 3))
        self.vertex_normals = np.zeros((0, 3))

    def has_triangles(self):
        return self.triangles.shape[0] > 0

    def has_vertex_colors(self):
        return self.vertex_colors.shape[0] > 0 and self.vertex_colors.shape[0] == self.vertices.shape[0]

    def has_vertex_normals(self):
        return self.vertex_normals.shape[0] > 0 and self.vertex_normals.shape[0] == self.vertices.shape[0]

    def compute_vertex_normals(self):
        self.vertex_normals = vertex_normals(torch.from_numpy(self.vertices),
                                             torch.from_numpy(self.triangles.astype(np.int64))).numpy()
        return self

    def transform(self, tf):
        tf = np.asarray(tf, np.float64)
        self.vertices = self.vertices @ tf[:3, :3].T + tf[:3, 3]
        if self.has_vertex_normals():
            n = self.vertex_normals @ tf[:3, :3].T
            norm = np.linalg.norm(n, axis=1, keepdims=True)
            self.vertex_normals = np.where(norm > 0, n / np.where(norm > 0, norm, 1.0), 0.0)
        return self

    def __iadd__(self, other):
        """Concatenation; per-vertex attributes survive only when both meshes (or an empty one) carry them."""
        nv = self.vertices.shape[0]
        for name in ("vertex_colors", "vertex_normals"):
            a, b = getattr(self, name), getattr(other, name)
            ok_a, ok_b = a.shape[0] == nv, b.shape[0] == other.vertices.shape[0]
            setattr(self, name, np.concatenate([a, b]) if ok_a and ok_b else np.zeros((0, 3)))
        self.vertices = np.concatenate([self.vertices, other.vertices])
        self.triangles = np.concatenate([self.triangles, other.triangles + nv]).astype(np.int32)
        return self

    def remove_duplicated_vertices(self):
        """Merge vertices with equal float64 positions, keeping the first occurrence and its attributes (Open3D's
        remove_duplicated_vertices)."""
        if self.vertices.shape[0] == 0:
            return self
        _, first, inv = np.unique(self.vertices, axis=0, return_index=True, return_inverse=True)
        order = np.argsort(first)
        new_id = np.empty_like(order)
        new_id[order] = np.arange(order.shape[0])
        self._take_vertices(first[order], new_id[inv.reshape(-1)])
        return self

    def select_triangles(self, keep):
        """Keep the triangles where `keep` is true and the vertices they still reference (Open3D's
        remove_triangles_by_mask keeps unreferenced vertices; this drops them)."""
        self.triangles = self.triangles[np.asarray(keep, bool)]
        used = np.zeros(self.vertices.shape[0], bool)
        used[self.triangles.reshape(-1)] = True
        idx = np.nonzero(used)[0]
        new_id = np.cumsum(used) - 1
        self._take_vertices(idx, new_id)
        return self

    def _take_vertices(self, idx, new_id):
        nv = self.vertices.shape[0]
        for name in ("vertex_colors", "vertex_normals"):
            a = getattr(self, name)
            if a.shape[0] == nv:
                setattr(self, name, a[idx])
        self.vertices = self.vertices[idx]
        self.triangles = new_id[self.triangles].astype(np.int32).reshape(-1, 3)


def vertex_normals(verts: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """Normalised area-weighted sums of the face normals (x1 - x0) x (x2 - x0) (Open3D's compute_vertex_normals);
    float64, on the tensors' device."""
    f = faces.long()
    v = verts[f]
    fn = torch.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0], dim=1)
    n = torch.zeros_like(verts).index_add_(0, f.reshape(-1), fn.repeat_interleave(3, 0))
    return torch.nn.functional.normalize(n, dim=1, eps=1e-300)


def write_ply(path, mesh: TriangleMesh) -> None:
    """Binary little-endian PLY: float64 positions, float64 normals and uchar colours when present, int32 faces."""
    nv, nt = mesh.vertices.shape[0], mesh.triangles.shape[0]
    fields = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {nv}"] + [f"property double {c}" for c in "xyz"]
    if mesh.has_vertex_normals():
        fields += [("nx", "<f8"), ("ny", "<f8"), ("nz", "<f8")]
        head += [f"property double {c}" for c in ("nx", "ny", "nz")]
    if mesh.has_vertex_colors():
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        head += [f"property uchar {c}" for c in ("red", "green", "blue")]
    head += [f"element face {nt}", "property list uchar int vertex_indices", "end_header"]
    vert = np.empty(nv, dtype=fields)
    for a, c in enumerate("xyz"):
        vert[c] = mesh.vertices[:, a]
    if mesh.has_vertex_normals():
        for a, c in enumerate(("nx", "ny", "nz")):
            vert[c] = mesh.vertex_normals[:, a]
    if mesh.has_vertex_colors():
        rgb = np.round(np.clip(mesh.vertex_colors, 0.0, 1.0) * 255.0).astype(np.uint8)
        for a, c in enumerate(("red", "green", "blue")):
            vert[c] = rgb[:, a]
    face = np.empty(nt, dtype=[("n", "u1"), ("v", "<i4", (3,))])
    face["n"] = 3
    face["v"] = mesh.triangles
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(vert.tobytes())
        f.write(face.tobytes())


def marching_cubes(sdf: torch.Tensor, mask=None, level: float = 0.0):
    """Welded marching-cubes mesh of a device grid sdf [nx,ny,nz] fp32 (mask: bool grid or None): vertices [V,3]
    float64 in grid-index space, numbered in ascending key order, and triangles [T,3] int64, both on the device
    (include/pinb200.h states the rules; oracle/mesh_oracle.py restates them)."""
    keys = ops.mc_triangle_keys(sdf, mask, level)
    uniq, inv = torch.unique(keys.reshape(-1), sorted=True, return_inverse=True)
    return ops.mc_vertices(sdf, uniq, level), inv.reshape(-1, 3)


def triangle_clusters(faces: torch.Tensor):
    """Edge-connected clusters of device triangles [T,3]: (root [T] int32 = smallest triangle id of the cluster,
    cluster size [T] int64 per triangle)."""
    t = faces.shape[0]
    if t == 0:
        return torch.zeros(0, dtype=torch.int32, device=faces.device), torch.zeros(0, dtype=torch.int64, device=faces.device)
    e = faces[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2).long()
    lo, hi = torch.minimum(e[:, 0], e[:, 1]), torch.maximum(e[:, 0], e[:, 1])
    key, order = torch.sort(lo * (int(faces.max()) + 1) + hi)
    root, size = ops.mesh_clusters(key, (order // 3).int(), t)
    return root, size.long()[root.long()]


class Mesher:
    # queries per launch: large enough to fill the GPU many times over, small enough to bound the output buffers
    CHUNK = 1 << 22

    def __init__(self, config, neural_points, decoders: dict):
        self.config = config
        self.silence = config.silence
        self.neural_points = neural_points
        self.sdf_mlp = decoders["sdf"]
        self.sem_mlp = decoders.get("semantic")
        self.color_mlp = decoders.get("color")
        self.device = config.device
        self.cur_device = self.device
        self.dtype = config.dtype
        self.global_transform = np.eye(4)

    def query_points(self, coord, bs, query_sdf=True, query_sem=False, query_color=False, query_mask=True,
                     query_locally=False, mask_min_nn_count: int = 4, out_torch: bool = False):
        """Returns (sdf_pred, sem_pred, color_pred, mc_mask) like the reference; `bs` is accepted for
        compatibility (it only sets a lower bound on the chunk size, the kernel takes millions of points per
        launch)."""
        if query_sem:
            raise NotImplementedError("semantic head is outside the CUDA hot path")
        n = coord.shape[0]
        dev = self.neural_points.neural_points.device
        chunk = max(int(bs), self.CHUNK)
        sdf_pred = torch.zeros(n, device=dev) if query_sdf else None
        color_pred = torch.zeros((n, self.config.color_channel), device=dev) if query_color else None
        mc_mask = torch.zeros(n, dtype=torch.bool, device=dev) if query_mask else None
        work = {}
        for head in range(0, n, chunk):
            tail = min(head + chunk, n)
            q = coord[head:tail].to(device=dev, dtype=torch.float32).contiguous()
            o = self.neural_points.query_sdf(q, self.sdf_mlp, query_locally=query_locally, need_grad=False,
                                             color_decoder=self.color_mlp if query_color else None, out=work)
            if query_sdf:
                # rows without any neighbour are never decoded by the reference: they keep sdf 0 (mesher.py:118-131)
                sdf_pred[head:tail] = torch.where(o["nn_count"] >= 1, o["sdf"], torch.zeros_like(o["sdf"]))
            if query_color:
                color_pred[head:tail] = o["color"]
            if query_mask:
                mc_mask[head:tail] = o["nn_count"] >= mask_min_nn_count
        if out_torch:
            return sdf_pred, None, color_pred, mc_mask
        return (None if sdf_pred is None else sdf_pred.cpu().numpy().astype(np.float64), None,
                None if color_pred is None else color_pred.cpu().numpy().astype(np.float64),
                None if mc_mask is None else mc_mask.cpu().numpy().astype(np.float64))

    def get_query_from_bbx(self, bbx, voxel_size, pad_voxel=0, skip_top_voxel=0):
        """Grid points of a bounding box (any object with get_min_bound() / get_max_bound()) as the reference builds
        them (utils/mesher.py:166-209): (coord [N,3] on the device, voxel_num_xyz, voxel_origin), or (None,)*3 above
        5e8 points.  Point index (x*ny + y)*nz + z."""
        min_bound = np.asarray(bbx.get_min_bound(), np.float64)
        max_bound = np.asarray(bbx.get_max_bound(), np.float64)
        voxel_num_xyz = (np.ceil((max_bound - min_bound) / voxel_size) + pad_voxel * 2).astype(np.int_)
        voxel_origin = min_bound - pad_voxel * voxel_size
        voxel_origin[2] -= voxel_size  # one more voxel underground keeps the ground closed
        voxel_num_xyz[2] += 1
        voxel_num_xyz[2] -= skip_top_voxel
        if voxel_num_xyz[0] * voxel_num_xyz[1] * voxel_num_xyz[2] > 5e8:
            print("too many query points, use smaller chunks")
            return None, None, None
        ax = [torch.arange(int(n), dtype=torch.int16, device=self.cur_device) for n in voxel_num_xyz]
        x, y, z = torch.meshgrid(*ax, indexing="ij")
        coord = torch.stack((x.flatten(), y.flatten(), z.flatten())).transpose(0, 1).float()
        coord *= voxel_size
        coord += torch.tensor(voxel_origin, dtype=self.dtype, device=self.cur_device)
        return coord, voxel_num_xyz, voxel_origin

    def assign_to_bbx(self, sdf_pred, sem_pred, color_pred, mc_mask, voxel_num_xyz):
        """Reshape the flat grid outputs to [nx,ny,nz] (utils/mesher.py:334-367)."""
        shape = tuple(int(n) for n in voxel_num_xyz)
        return tuple(None if a is None else a.reshape(shape) for a in (sdf_pred, sem_pred, color_pred, mc_mask))

    def mc_mesh(self, mc_sdf, mc_mask, voxel_size, mc_origin):
        """Marching cubes at level 0 on the device (utils/mesher.py:369-397 with skimage's mask= / allow_degenerate=
        False): (world-space vertices [V,3] float64, triangles [T,3] int64), both device tensors; vertices are
        origin + v * voxel_size in float64."""
        if not self.silence:
            print("Marching cubes ...")
        dev = self.neural_points.neural_points.device
        sdf = torch.as_tensor(mc_sdf).to(device=dev, dtype=torch.float32).contiguous()
        mask = None if mc_mask is None else torch.as_tensor(mc_mask).to(device=dev, dtype=torch.bool).contiguous()
        verts, faces = marching_cubes(sdf, mask, 0.0)
        origin = torch.as_tensor(np.asarray(mc_origin, np.float64), device=dev)
        return origin + verts * float(voxel_size), faces

    def estimate_vertices_color(self, mesh, verts):
        """Vertex colours from the colour head at the world-space vertices (utils/mesher.py:423-441)."""
        if len(verts) == 0:
            return mesh
        q = torch.as_tensor(verts).to(device=self.neural_points.neural_points.device, dtype=self.dtype)
        _, _, col, _ = self.query_points(q, self.config.infer_bs, False, False, True, False, out_torch=True)
        col = col.double().cpu().numpy()
        if self.config.color_channel == 1:
            col = np.repeat(col * 2.0, 3, axis=1)
        mesh.vertex_colors = col
        return mesh

    def filter_isolated_vertices(self, mesh, filter_cluster_min_tri=300):
        """Drop the edge-connected triangle clusters of fewer than `filter_cluster_min_tri` triangles
        (utils/mesher.py:443-456), then the vertices no triangle references any more."""
        if not mesh.has_triangles():
            return mesh
        faces = torch.as_tensor(mesh.triangles, device=self.neural_points.neural_points.device)
        _, size = triangle_clusters(faces)
        return mesh.select_triangles((size >= int(filter_cluster_min_tri)).cpu().numpy())

    def recon_aabb_mesh(self, bbx, voxel_size, mesh_path=None, query_locally=False, estimate_sem=False,
                        estimate_color=False, mesh_normal=True, filter_isolated_mesh=False,
                        filter_free_space_vertices=True, mesh_min_nn=10, use_torch_mc=False):
        """Mesh of one bounding box (utils/mesher.py:558-649).  `use_torch_mc` is accepted and ignored: every path
        is the device one."""
        if estimate_sem:
            raise NotImplementedError("semantic head is outside the CUDA hot path")
        cfg = self.config
        coord, voxel_num_xyz, voxel_origin = self.get_query_from_bbx(bbx, voxel_size, cfg.pad_voxel, cfg.skip_top_voxel)
        if coord is None:
            return None
        sdf, _, _, mask = self.query_points(coord, cfg.infer_bs, True, False, False, cfg.mc_mask_on, query_locally,
                                            mesh_min_nn, out_torch=True)
        del coord
        mc_sdf, _, _, mc_mask = self.assign_to_bbx(sdf, None, None, mask, voxel_num_xyz)
        verts, faces = self.mc_mesh(mc_sdf, mc_mask, voxel_size, voxel_origin)
        mesh = TriangleMesh(verts.cpu().numpy(), faces.int().cpu().numpy())
        if estimate_color:
            mesh = self.estimate_vertices_color(mesh, verts)
        if mesh_normal:
            mesh.vertex_normals = vertex_normals(verts, faces).cpu().numpy()
        if filter_isolated_mesh:
            mesh = self.filter_isolated_vertices(mesh, cfg.min_cluster_vertices)
        if not np.array_equal(self.global_transform, np.eye(4)):
            mesh.transform(self.global_transform)
        if mesh_path is not None:
            write_ply(mesh_path, mesh)
            if not self.silence:
                print("save the mesh to %s\n" % (mesh_path))
        return mesh

    def recon_aabb_collections_mesh(self, aabbs, voxel_size, mesh_path=None, query_locally=False, estimate_sem=False,
                                    estimate_color=False, mesh_normal=True, filter_isolated_mesh=False,
                                    filter_free_space_vertices=True, mesh_min_nn=10, use_torch_mc=False):
        """Meshes of several bounding boxes, concatenated, with vertices of equal positions merged
        (utils/mesher.py:507-556)."""
        merged = TriangleMesh()
        for bbx in aabbs:
            cur = self.recon_aabb_mesh(bbx, voxel_size, None, query_locally, estimate_sem, estimate_color, mesh_normal,
                                       filter_isolated_mesh, filter_free_space_vertices, mesh_min_nn, use_torch_mc)
            if cur is not None:
                merged += cur
        merged.remove_duplicated_vertices()
        if mesh_normal:
            merged.compute_vertex_normals()
        if mesh_path is not None:
            write_ply(mesh_path, merged)
            if not self.silence:
                print("save the mesh to %s\n" % (mesh_path))
        return merged


def patch_reference_mesher(mesher_cls) -> None:
    """Route the reference's own `utils.mesher.Mesher` (marching cubes, mesh IO untouched) through the fused
    grid query:  `from utils.mesher import Mesher; patch_reference_mesher(Mesher)`."""
    mesher_cls.query_points = Mesher.query_points
    if not hasattr(mesher_cls, "CHUNK"):
        mesher_cls.CHUNK = Mesher.CHUNK
