"""CPU oracle of the mesh extraction (DESIGN.md row f5)  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates, in vectorised numpy / scipy, the specification pin_slam_b200/csrc/mesh/mcubes.cu implements: the
marching-cubes triangle table derived from one rule on cube faces, the welded marching-cubes mesh of a masked SDF grid
(the reference's skimage.measure.marching_cubes(mask=...) + Open3D remove_duplicated_vertices, utils/mesher.py:369-397,
:631), and the edge-connected triangle clusters of utils/mesher.py:443-456 (Open3D cluster_connected_triangles).
Only tests/ import it.
"""

# --------------------------------------------------------------------------
# mesh extraction (DESIGN.md row f5): marching cubes + small-cluster filter, the spec of csrc/mesh/mcubes.cu
# --------------------------------------------------------------------------
# corner c of a cube sits at (c & 1, c >> 1 & 1, c >> 2 & 1); edge e = 4 * axis + m runs along `axis` from the m-th
# corner (ascending) whose `axis` bit is clear to that corner with the bit set
MC_EDGES = [(c, c | (1 << a), a) for a in range(3) for c in range(8) if not (c >> a) & 1]


def mc_triangle_table():
    """The 256 x 16 triangle table (edge ids, -1 padded) derived from one rule on cube faces: a face with two
    crossing edges gets one segment; an ambiguous face (four crossing edges) cuts off each inside corner with its own
    segment.  Segments are directed so that (outward face normal) x (segment) points to the inside corner(s) of the
    face; every crossing edge then has one successor and one predecessor.  Each loop (in order from its smallest edge)
    is fanned from its first edge whose diagonals all cross the cube's interior: a diagonal joining two edges of one
    face could be drawn by the cube on the other side of that face too, and the surface would no longer be a closed
    2-manifold.  The right-hand normal of every triangle points to the inside (sdf < level)."""
    import numpy as np

    corner = np.array([(c & 1, c >> 1 & 1, c >> 2 & 1) for c in range(8)], np.float64)
    mid = np.array([corner[lo] + 0.5 * np.eye(3)[a] for lo, _, a in MC_EDGES])
    table = np.full((256, 16), -1, np.int64)
    # the two faces (axis, side) each edge lies on
    face_of = [{(b, lo >> b & 1) for b in range(3) if b != a} for lo, _, a in MC_EDGES]
    for ci in range(256):
        inside = [(ci >> c) & 1 for c in range(8)]
        succ = {}
        for a in range(3):
            for s in (0, 1):
                n = (2.0 * s - 1.0) * np.eye(3)[a]
                fc = [c for c in range(8) if (c >> a) & 1 == s]
                fe = [e for e, (lo, hi, ax) in enumerate(MC_EDGES) if ax != a and (lo >> a) & 1 == s]
                cross = [e for e in fe if inside[MC_EDGES[e][0]] != inside[MC_EDGES[e][1]]]
                if len(cross) == 2:
                    segs = [(cross[0], cross[1], next(c for c in fc if inside[c]))]
                elif len(cross) == 4:
                    segs = []
                    for c in fc:
                        if inside[c]:
                            p, q = [e for e in fe if c in MC_EDGES[e][:2]]
                            segs.append((p, q, c))
                else:
                    segs = []
                for p, q, c in segs:
                    d = mid[q] - mid[p]
                    if np.dot(np.cross(n, d), corner[c] - 0.5 * (mid[p] + mid[q])) < 0:
                        p, q = q, p
                    assert p not in succ
                    succ[p] = q
        assert sorted(succ) == sorted(succ.values())
        tris, seen = [], set()
        for e0 in sorted(succ):
            if e0 in seen:
                continue
            loop = [e0]
            while succ[loop[-1]] != e0:
                loop.append(succ[loop[-1]])
            seen.update(loop)
            # fan apex: the first loop edge none of whose diagonals joins two edges of one cube face (such a diagonal
            # could be drawn by the neighbouring cube too, and the surface would not close)
            apex = next(r for r in range(len(loop)) if not any(
                face_of[loop[r]] & face_of[loop[(r + i) % len(loop)]] for i in range(2, len(loop) - 1)))
            loop = loop[apex:] + loop[:apex]
            tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
        assert len(tris) <= 5
        table[ci, :3 * len(tris)] = np.array(tris, np.int64).reshape(-1)
    return table


def marching_cubes(sdf, mask=None, level=0.0, chunk=1 << 21):
    """Vectorised numpy restatement of the marching-cubes kernel (pin_slam_b200/csrc/mesh/mcubes.cu).
    sdf [nx,ny,nz] float32 (grid point p = (x*ny + y)*nz + z), mask [nx,ny,nz] bool or None.
      * a corner is inside iff sdf < level; cube (i,j,k) is polygonised iff mask[i,j,k] (its lowest corner)
      * one vertex per grid edge whose corners differ: t = (level - a) / (b - a) in float32 from the lower corner a to
        the upper corner b, key 3*p + axis (p: lower corner); t == 0 or 1 puts it on the grid point q, key 3*N + q
      * triangles in cube order, table order within a cube; a triangle with two equal keys is dropped
      * vertices numbered in ascending key order, positions in grid-index space (float64 i + t)
    Returns (verts [V,3] float64, faces [T,3] int64, keys [V] int64)."""
    import numpy as np

    sdf = np.ascontiguousarray(sdf, np.float32)
    nx, ny, nz = sdf.shape
    n = sdf.size
    stride = np.array([ny * nz, nz, 1], np.int64)
    empty = (np.zeros((0, 3)), np.zeros((0, 3), np.int64), np.zeros(0, np.int64))
    if min(nx, ny, nz) < 2:
        return empty
    table = mc_triangle_table()
    lvl = np.float32(level)
    flat = sdf.reshape(-1)
    ci = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, c >> 1 & 1, c >> 2 & 1
        ci |= (sdf[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz] < lvl).astype(np.int64) << c
    sel = (ci > 0) & (ci < 255)
    if mask is not None:
        sel &= np.asarray(mask, bool)[:-1, :-1, :-1]
    ii, jj, kk = np.nonzero(sel)  # ascending cube index
    cube_ci = ci[ii, jj, kk]
    cube_p = (ii * ny + jj) * nz + kk
    corner_off = np.array([(c & 1) * stride[0] + (c >> 1 & 1) * stride[1] + (c >> 2 & 1) for c in range(8)], np.int64)
    out = []
    with np.errstate(divide="ignore", invalid="ignore"):
        for h in range(0, cube_p.shape[0], chunk):
            p, cc = cube_p[h:h + chunk], cube_ci[h:h + chunk]
            keys = np.empty((p.shape[0], 12), np.int64)
            for e, (lo, hi, a) in enumerate(MC_EDGES):
                q = p + corner_off[lo]
                va, vb = flat[q], flat[p + corner_off[hi]]
                t = (lvl - va) / (vb - va)
                keys[:, e] = np.where(t == 0, 3 * n + q, np.where(t == 1, 3 * n + q + stride[a], 3 * q + a))
            e15 = table[cc, :15]  # [m,15]
            k = np.take_along_axis(keys, np.maximum(e15, 0), 1).reshape(-1, 5, 3)
            ok = (e15[:, ::3] >= 0) & (k[..., 0] != k[..., 1]) & (k[..., 1] != k[..., 2]) & (k[..., 0] != k[..., 2])
            out.append(k[ok])  # cube-major, table order within a cube
    tri_keys = np.concatenate(out) if out else np.zeros((0, 3), np.int64)
    if tri_keys.shape[0] == 0:
        return empty
    uniq, inv = np.unique(tri_keys.reshape(-1), return_inverse=True)
    return mc_vertex_positions(sdf, uniq, level), inv.reshape(-1, 3).astype(np.int64), uniq


def mc_vertex_positions(sdf, keys, level=0.0):
    """Grid-index-space positions (float64) of vertex keys (see marching_cubes)."""
    import numpy as np

    nx, ny, nz = sdf.shape
    n = sdf.size
    flat = np.ascontiguousarray(sdf, np.float32).reshape(-1)
    stride = np.array([ny * nz, nz, 1], np.int64)
    on_grid = keys >= 3 * n
    q = np.where(on_grid, keys - 3 * n, keys // 3)
    a = np.where(on_grid, 0, keys % 3)
    pos = np.stack([q // stride[0], q // nz % ny, q % nz], 1).astype(np.float64)
    e = ~on_grid
    with np.errstate(divide="ignore", invalid="ignore"):
        va, vb = flat[q[e]], flat[q[e] + stride[a[e]]]
        t = (np.float32(level) - va) / (vb - va)
    pos[np.nonzero(e)[0], a[e]] += t.astype(np.float64)
    return pos


def mesh_clusters(faces, n_verts=None):
    """Open3D's cluster_connected_triangles restated: triangles are connected when they share an (undirected) edge.
    Returns (label [T] int64, cluster size in triangles [n_clusters] int64), labels numbered by first triangle."""
    import numpy as np
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components

    f = np.asarray(faces, np.int64)
    t = f.shape[0]
    if t == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    e = np.sort(f[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2), 1)
    key = e[:, 0] * (int(f.max()) + 1) + e[:, 1]
    order = np.argsort(key, kind="stable")
    tri = order // 3
    same = key[order][1:] == key[order][:-1]
    g = sp.coo_matrix((np.ones(int(same.sum())), (tri[1:][same], tri[:-1][same])), shape=(t, t))
    _, lab = connected_components(g, directed=False)
    _, first, lab = np.unique(lab, return_index=True, return_inverse=True)
    rank = np.argsort(np.argsort(first))
    lab = rank[lab]
    return lab, np.bincount(lab)
