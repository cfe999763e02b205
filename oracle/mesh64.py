"""Float64 restatement of the mesh extractor (DESIGN §3.15), written from the statement of open3d's legacy TSDF
integration and extraction, and of LaRa's postprocess (tools/meshExtractor.py:116-134).  numpy only; the marching-cubes
triangles come from the generated table's source, tools/gen_mc_table.py.

Inputs are the float32 values the kernels receive (images, camera records, voxel_size, sdf_trunc), widened to float64.
"""
from __future__ import annotations

import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FX, FY, CX, CY, DT = 16, 17, 18, 19, 20
NEAR_PX = 1e-4


def mc_table():
    """The 256 cases' triangles (lists of local edge triples) and the local edges' (start corner, axis)."""
    spec = importlib.util.spec_from_file_location("gen_mc_table", os.path.join(ROOT, "tools", "gen_mc_table.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    edges = [(s, (t ^ s).bit_length() - 1) for s, t in mod.EDGES]
    return mod.table(), edges


def integrate(n, voxel_size, sdf_trunc, depth, acc, image, cams, alpha_thres, state=None):
    """Fuse V views into the voxels n [M,3] (integer indices).  depth, acc [V,H,W], image [V,3,H,W], cams [V,24].
    Returns (tsdf [M], weight [M], color [M,3], near [M]): ``near`` marks voxels whose u_f or v_f lies within 1e-4 px of
    an integer or of a bound in some view, or whose sdf lies within 1e-5 (|z| + d) of -sdf_trunc: there an fp32
    evaluation may pick another pixel or another branch."""
    n = np.asarray(n, dtype=np.float64)
    M = len(n)
    vs, st = float(np.float32(voxel_size)), float(np.float32(sdf_trunc))
    at = np.float32(alpha_thres)
    if state is None:
        tsdf, w, col = np.zeros(M), np.zeros(M), np.zeros((M, 3))
    else:
        tsdf, w, col = (np.array(x, dtype=np.float64) for x in state)
    near = np.zeros(M, dtype=bool)
    p = (n + 0.5) * vs
    V, H, W = depth.shape
    for v in range(V):
        r = np.asarray(cams[v], dtype=np.float64)
        E = r[:16].reshape(4, 4)
        fx, fy, cx, cy, dt = r[FX], r[FY], r[CX], r[CY], r[DT]
        q = p @ E[:3, :3].T + E[:3, 3]
        z = q[:, 2]
        front = z > 0
        zs = np.where(front, z, 1.0)
        uf = q[:, 0] * fx / zs + cx + 0.5
        vf = q[:, 1] * fy / zs + cy + 0.5
        for f, size in ((uf, W), (vf, H)):
            near |= front & ((np.abs(f - np.round(f)) < NEAR_PX) | (np.abs(f - 1e-4) < NEAR_PX)
                             | (np.abs(f - (size - 1e-4)) < NEAR_PX))
        inside = front & (uf >= 1e-4) & (uf < W - 1e-4) & (vf >= 1e-4) & (vf < H - 1e-4)
        u = np.where(inside, uf, 0).astype(np.int64)
        vv = np.where(inside, vf, 0).astype(np.int64)
        a = acc[v][vv, u]
        d = depth[v][vv, u].astype(np.float64)
        d = np.where((a < at) | (d > np.float64(np.float32(dt))), 0.0, d)
        ok = inside & (d > 0)
        mult = np.sqrt(1 + ((u - cx) / fx) ** 2 + ((vv - cy) / fy) ** 2)
        sdf = (d - z) * mult
        near |= ok & (np.abs(sdf + st) < 1e-5 * (np.abs(z) + d))
        upd = ok & (sdf > -st)
        t = np.minimum(1.0, sdf / st)
        rgb = np.trunc(np.stack([image[v, c][vv, u] for c in range(3)], -1).astype(np.float32) * np.float32(255))
        w1 = w + 1
        tsdf = np.where(upd, (tsdf * w + t) / w1, tsdf)
        col = np.where(upd[:, None], (col * w[:, None] + rgb.astype(np.float64)) / w1[:, None], col)
        w = np.where(upd, w1, w)
    return tsdf, w, col, near


def grid_voxels(n0, dims):
    """Integer indices [N,3] of a block's voxels in linear order (x fastest)."""
    k, j, i = np.meshgrid(*(np.arange(d) for d in dims[::-1]), indexing="ij")
    return np.stack((i.reshape(-1) + n0[0], j.reshape(-1) + n0[1], k.reshape(-1) + n0[2]), -1)


def extract(n0, dims, voxel_size, tsdf, weight, color):
    """Marching cubes on a block (tsdf, weight [nz,ny,nx], color [3,nz,ny,nx] or [nz,ny,nx,3]): (vertices [Nv,3],
    triangles [Nt,3], colors [Nv,3]) in the canonical order, vertices by (owning voxel, axis), triangles by (cube,
    table order)."""
    tab, edges = mc_table()
    vs = float(np.float32(voxel_size))
    nx, ny, nz = dims
    T = np.asarray(tsdf, np.float64).reshape(nz, ny, nx)
    Wt = np.asarray(weight, np.float64).reshape(nz, ny, nx)
    C = np.asarray(color, np.float64)
    C = C.reshape(3, nz, ny, nx) if C.shape[0] == 3 and C.ndim != 2 else C.reshape(nz, ny, nx, 3).transpose(3, 0, 1, 2)
    cx_, cy_, cz_ = nx - 1, ny - 1, nz - 1
    if min(cx_, cy_, cz_) <= 0:
        return np.zeros((0, 3)), np.zeros((0, 3), np.int64), np.zeros((0, 3))

    def corner(a, c):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        return a[dz:dz + cz_, dy:dy + cy_, dx:dx + cx_]
    valid = np.ones((cz_, cy_, cx_), dtype=bool)
    case = np.zeros((cz_, cy_, cx_), dtype=np.int64)
    for c in range(8):
        valid &= corner(Wt, c) > 0
        case |= (corner(T, c) < 0).astype(np.int64) << c
    case = np.where(valid, case, 0)
    flags = np.zeros((nz, ny, nx, 3), dtype=bool)
    for s, axis in edges:
        cross = ((case >> s) & 1) != ((case >> (s | (1 << axis))) & 1)
        dx, dy, dz = s & 1, (s >> 1) & 1, (s >> 2) & 1
        flags[dz:dz + cz_, dy:dy + cy_, dx:dx + cx_, axis] |= cross
    flat = flags.reshape(-1)
    ids = np.cumsum(flat) - 1
    e = np.nonzero(flat)[0]
    vox, axis = e // 3, e % 3
    n = grid_voxels(n0, dims)[vox].astype(np.float64)
    step = np.array([1, nx, nx * ny])[axis]
    t0, t1 = T.reshape(-1)[vox], T.reshape(-1)[vox + step]
    f0, f1 = np.abs(t0), np.abs(t1)
    verts = (n + 0.5) * vs
    verts[np.arange(len(e)), axis] += f0 / (f0 + f1) * vs
    Cf = C.reshape(3, -1)
    cols = ((f1[:, None] * Cf[:, vox].T + f0[:, None] * Cf[:, vox + step].T) / (f0 + f1)[:, None]) / 255.0
    # triangles, by (cube linear index, slot)
    cz, cy, cx = np.nonzero(case)
    cs = case[cz, cy, cx]
    cube = cx + nx * (cy + ny * cz)
    tris, keys = [], []
    maxt = max(len(t) for t in tab)
    cnt = np.array([len(t) for t in tab])
    arr = np.zeros((256, maxt, 3), np.int64)
    for c, t in enumerate(tab):
        if t:
            arr[c, :len(t)] = t
    es, ea = np.array([x[0] for x in edges]), np.array([x[1] for x in edges])
    for slot in range(maxt):
        has = cnt[cs] > slot
        if not has.any():
            continue
        tri = np.zeros((int(has.sum()), 3), np.int64)
        for m in range(3):
            le = arr[cs[has], slot, m]
            s, ax = es[le], ea[le]
            g = cube[has] + (s & 1) + ((s >> 1) & 1) * nx + ((s >> 2) & 1) * nx * ny
            tri[:, m] = ids[3 * g + ax]
        tris.append(tri)
        keys.append(np.stack((cube[has], np.full(int(has.sum()), slot)), -1))
    if not tris:
        return verts, np.zeros((0, 3), np.int64), cols
    tris, keys = np.concatenate(tris), np.concatenate(keys)
    order = np.lexsort((keys[:, 1], keys[:, 0]))
    return verts, tris[order], cols


def filter_mesh(vertices, triangles, colors, aabb, keep=10):
    """LaRa's postprocess: aabb cut (any vertex outside drops the triangle), edge-connected clusters through a
    triangle-edge incidence matrix, keep counts >= the min(#clusters, keep)-th largest, drop unreferenced vertices."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components
    tris = np.asarray(triangles, np.int64).reshape(-1, 3)
    v = np.asarray(vertices, np.float64)
    if aabb is not None and len(tris):
        a = np.asarray(aabb, np.float64).reshape(2, 3)
        bad = ~((v >= a[0]).all(-1) & (v <= a[1]).all(-1))
        tris = tris[~bad[tris].any(-1)]
    if len(tris):
        und = np.sort(np.stack((tris, np.roll(tris, -1, axis=1)), -1).reshape(-1, 2), axis=1)
        _, edge_id = np.unique(und, axis=0, return_inverse=True)
        edge_id = edge_id.reshape(-1)
        inc = csr_matrix((np.ones(len(edge_id)), (np.repeat(np.arange(len(tris)), 3), edge_id)))
        _, lab = connected_components(inc @ inc.T, directed=False)
        cnt = np.bincount(lab)
        thr = np.sort(cnt)[-min(len(cnt), keep)]
        tris = tris[cnt[lab] >= thr]
    used = np.unique(tris.reshape(-1))
    remap = np.full(len(v), -1, np.int64)
    remap[used] = np.arange(len(used))
    return np.asarray(vertices)[used], remap[tris], np.asarray(colors)[used]
