"""GPU mesh extraction for LaRa's ``tools/meshExtractor.py`` (DESIGN §3.15): TSDF fusion of the rendered camera path
and marching cubes in CUDA (``csrc/mesh.cu``, C ABI ``include/surfel_mesh.h``), without open3d.

LaRa's ``MeshExtractor.extract`` renders 48 views, copies each to the host and fuses it into open3d's CPU
``ScalableTSDFVolume``, then runs open3d's marching cubes and a cluster filter.  Here the forward-only renders are fused
on the device as the fused epilogue leaves them, the mesh is extracted and filtered (edge-connected clusters, as LaRa
filters them) on the device, and only the filtered mesh is copied to the host for the file write:

    vol = tsdf_volume(depth, acc, records, voxel_size, sdf_trunc, alpha_thres, aabb)
    integrate(vol, depth, acc, image, records, alpha_thres)
    vertices, triangles, colors = filter_mesh_device(extract_triangle_mesh(vol), aabb)
    write_obj(path, vertices, triangles, colors)

``filter_mesh`` is the same filter on the host (numpy and scipy), equal to ``filter_mesh_device`` element for element.

``MeshExtractor`` wraps these behind LaRa's class, with the camera list in place of ``uni_mesh_path``'s arguments.
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

CAM_FX, CAM_FY, CAM_CX, CAM_CY, CAM_DEPTH_TRUNC = 16, 17, 18, 19, 20      # include/surfel_mesh.h SRF_MESH_CAM_*


@dataclass
class TSDFVolume:
    """A dense block of voxels n0 + (i, j, k) on the world-aligned grid of ``voxel_size``: tsdf and weight
    [dims[2], dims[1], dims[0]], color [3, dims[2], dims[1], dims[0]] (0..255), i.e. x fastest."""
    n0: Tuple[int, int, int]
    dims: Tuple[int, int, int]
    voxel_size: float
    sdf_trunc: float
    tsdf: torch.Tensor
    weight: torch.Tensor
    color: torch.Tensor

    @property
    def empty(self) -> bool:
        return min(self.dims) <= 0


def camera_records64(cams, aabb_center=None, radius=None, depth_trunc: float = 10.0) -> np.ndarray:
    """[V, 24] float64 integration records of MiniCam-like cameras, computed as LaRa's extract computes open3d's
    arguments (meshExtractor.py:77-82, 95-97, 108): w2c = world_view_transform^T, fx = W / (2 tan(FoVx / 2)),
    cx = W / 2, and with an aabb (its centre and radius given) depth_trunc = |camera_center - centre| + radius."""
    rec = np.zeros((len(cams), _lib.MESH_CAM_FLOATS), dtype=np.float64)
    for v, cam in enumerate(cams):
        W, H = int(cam.image_width), int(cam.image_height)
        rec[v, :16] = cam.world_view_transform.detach().cpu().numpy().T.reshape(16)
        rec[v, CAM_FX] = W / (2 * math.tan(cam.FoVx / 2.0))
        rec[v, CAM_FY] = H / (2 * math.tan(cam.FoVy / 2.0))
        rec[v, CAM_CX], rec[v, CAM_CY] = W / 2, H / 2
        if aabb_center is not None:
            campos = cam.camera_center.detach().cpu().numpy()
            rec[v, CAM_DEPTH_TRUNC] = np.linalg.norm(campos - aabb_center, axis=-1) + radius
        else:
            rec[v, CAM_DEPTH_TRUNC] = depth_trunc
    return rec


def camera_records(cams, device, aabb_center=None, radius=None, depth_trunc: float = 10.0) -> torch.Tensor:
    """:func:`camera_records64` as the float32 device tensor the kernel reads."""
    return torch.from_numpy(camera_records64(cams, aabb_center, radius, depth_trunc)).to(torch.float32).to(device)


def mesh_settings(aabb: Optional[np.ndarray], voxel_size: float, sdf_trunc: float):
    """(voxel_size, sdf_trunc, aabb centre, aabb radius) of LaRa's extract (meshExtractor.py:54-58): an aabb (the x1.1
    box) overrides the arguments with radius / 256 and twice that."""
    if aabb is None:
        return voxel_size, sdf_trunc, None, None
    center = aabb.mean(0)
    radius = np.linalg.norm(aabb[1] - aabb[0]) * 0.5
    voxel_size = radius / 256
    return voxel_size, voxel_size * 2, center, radius


def _check_views(depth, acc, image, cams):
    for name, t in (("depth", depth), ("acc", acc), ("image", image), ("cams", cams)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda:
            raise RuntimeError(f"mesh: {name} must be a float32 CUDA tensor")
        if t.device != depth.device:
            raise RuntimeError(f"mesh: {name} must be on {depth.device}, got {t.device}")
        if not t.is_contiguous():
            raise RuntimeError(f"mesh: {name} must be contiguous (the planar [V,C,H,W] buffers of the epilogue)")
    if depth.ndim != 3:
        raise RuntimeError(f"mesh: depth must be [V,H,W], got {tuple(depth.shape)}")
    V, H, W = (int(s) for s in depth.shape)
    for name, t, shape in (("acc", acc, (V, H, W)), ("image", image, (V, 3, H, W)),
                           ("cams", cams, (V, _lib.MESH_CAM_FLOATS))):
        if tuple(t.shape) != shape:
            raise RuntimeError(f"mesh: {name} must be {shape}, got {tuple(t.shape)}")
    return V, H, W


def _index_range(lo: np.ndarray, hi: np.ndarray, vs: float):
    """Voxel indices whose centres (n + 0.5) vs cover [lo, hi], plus one voxel on each side."""
    return np.floor(lo / vs - 0.5).astype(np.int64) - 1, np.ceil(hi / vs - 0.5).astype(np.int64) + 1


def tsdf_volume(depth: torch.Tensor, acc: torch.Tensor, cams: torch.Tensor, voxel_size: float, sdf_trunc: float,
                alpha_thres: float, aabb: Optional[np.ndarray] = None) -> TSDFVolume:
    """Choose and allocate (cleared) the block for these views (DESIGN §3.15): every voxel whose TSDF any view can make
    negative lies within  sdf_trunc sqrt(1 + sx^2 + sy^2) + d_max / 2 sqrt(1/fx^2 + 1/fy^2)  of a back-projected valid
    pixel (sx, sy the largest |x/z|, |y/z| of the image, d_max its largest valid depth); the block is their bounding box
    grown by that margin and one voxel, so that it holds every cube with a negative corner.  With ``aabb`` (the x1.1
    box, [2,3]) it is clipped to the aabb grown by one voxel, which holds every cube of a triangle the aabb filter
    keeps.  The result then equals an unbounded volume's after the filter."""
    V, H, W = (int(s) for s in depth.shape)
    vs = float(np.float32(voxel_size))
    lo, hi, margin = np.full(3, np.inf), np.full(3, -np.inf), 0.0
    rec = cams.detach().cpu().to(torch.float64)
    v_, u_ = torch.meshgrid(torch.arange(H, device=depth.device, dtype=torch.float64),
                            torch.arange(W, device=depth.device, dtype=torch.float64), indexing="ij")
    for v in range(V):
        r = rec[v]
        fx, fy, cx, cy, dt = (float(r[k]) for k in (CAM_FX, CAM_FY, CAM_CX, CAM_CY, CAM_DEPTH_TRUNC))
        d = depth[v].to(torch.float64)
        ok = (acc[v] >= alpha_thres) & (depth[v] > 0) & (depth[v] <= np.float32(dt))
        if not bool(ok.any()):
            continue
        d = d[ok]
        pc = torch.stack(((u_[ok] - cx) / fx * d, (v_[ok] - cy) / fy * d, d), dim=-1)
        E = r[:16].reshape(4, 4).to(depth.device)
        pw = (pc - E[:3, 3]) @ torch.linalg.inv(E[:3, :3]).T
        lo = np.minimum(lo, pw.amin(0).cpu().numpy())
        hi = np.maximum(hi, pw.amax(0).cpu().numpy())
        sx, sy = (max(cx, W - cx) + 0.5) / fx, (max(cy, H - cy) + 0.5) / fy
        margin = max(margin, sdf_trunc * math.sqrt(1 + sx * sx + sy * sy)
                     + 0.5 * float(d.max()) * math.sqrt(1 / fx ** 2 + 1 / fy ** 2))
    dev = depth.device
    if not np.isfinite(lo).all():
        n_lo, n_hi = np.zeros(3, np.int64), np.full(3, -1, np.int64)
    else:
        n_lo, n_hi = _index_range(lo - margin, hi + margin, vs)
        if aabb is not None:
            a_lo, a_hi = _index_range(np.asarray(aabb[0], np.float64), np.asarray(aabb[1], np.float64), vs)
            n_lo, n_hi = np.maximum(n_lo, a_lo), np.minimum(n_hi, a_hi)
    dims = tuple(int(max(x, 0)) for x in n_hi - n_lo + 1)
    shape = (dims[2], dims[1], dims[0])
    return TSDFVolume(tuple(int(x) for x in n_lo), dims, vs, float(np.float32(sdf_trunc)),
                      torch.zeros(shape, dtype=torch.float32, device=dev),
                      torch.zeros(shape, dtype=torch.float32, device=dev),
                      torch.zeros((3,) + shape, dtype=torch.float32, device=dev))


def integrate(volume: TSDFVolume, depth: torch.Tensor, acc: torch.Tensor, image: torch.Tensor, cams: torch.Tensor,
              alpha_thres: float) -> None:
    """Fuse the views depth [V,H,W], acc [V,H,W], image [V,3,H,W] (planar, as the fused epilogue writes them) with
    the records ``cams`` [V,24] into ``volume`` in place, in view order."""
    V, H, W = _check_views(depth, acc, image, cams)
    if volume.empty or V == 0:
        return
    _lib.launch("srf_tsdf_integrate", depth.device, _lib.int3(volume.n0), _lib.int3(volume.dims), volume.voxel_size,
                volume.sdf_trunc, volume.tsdf.data_ptr(), volume.weight.data_ptr(), volume.color.data_ptr(), V, H, W,
                depth.data_ptr(), acc.data_ptr(), image.data_ptr(), cams.data_ptr(), float(alpha_thres))


def extract_triangle_mesh(volume: TSDFVolume):
    """Marching cubes on the device: (vertices [Nv,3] float32, triangles [Nt,3] int32, colors [Nv,3] float32 in
    0..1), vertices ordered by (owning voxel, axis), triangles by (cube, table order).  One host read of the totals."""
    dev = volume.tsdf.device
    if volume.empty:
        return (torch.empty((0, 3), dtype=torch.float32, device=dev), torch.empty((0, 3), dtype=torch.int32, device=dev),
                torch.empty((0, 3), dtype=torch.float32, device=dev))
    dims = _lib.int3(volume.dims)
    ws = torch.empty(_lib.mesh_workspace_bytes(_lib.load(), volume.dims), dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int32, device=dev)
    _lib.launch("srf_mesh_count", dev, dims, volume.tsdf.data_ptr(), volume.weight.data_ptr(), ws.data_ptr(),
                totals.data_ptr())
    Nv, Nt = (int(x) for x in totals.cpu())
    vertices = torch.empty((Nv, 3), dtype=torch.float32, device=dev)
    colors = torch.empty((Nv, 3), dtype=torch.float32, device=dev)
    triangles = torch.empty((Nt, 3), dtype=torch.int32, device=dev)
    _lib.launch("srf_mesh_emit", dev, _lib.int3(volume.n0), dims, volume.voxel_size, volume.tsdf.data_ptr(),
                volume.color.data_ptr(), ws.data_ptr(), Nv, Nt, vertices.data_ptr(), colors.data_ptr(),
                triangles.data_ptr())
    return vertices, triangles, colors


def _numpy(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def filter_mesh(mesh, aabb: Optional[np.ndarray], keep: int = 10):
    """LaRa's postprocess (meshExtractor.py:116-134) on the host: drop the triangles with a vertex outside ``aabb``
    ([2,3], inclusive), keep the edge-connected components whose triangle count is at least the min(#components,
    keep)-th largest (ties keep more), drop unreferenced vertices (order kept).  Returns numpy (vertices, triangles,
    colors)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    vertices, triangles, colors = (_numpy(x) for x in mesh)
    triangles = triangles.astype(np.int64).reshape(-1, 3)
    if aabb is not None and len(triangles):
        a = np.asarray(aabb, dtype=np.float64).reshape(2, 3)
        v64 = vertices.astype(np.float64)
        outside = ~((v64 >= a[0]).all(-1) & (v64 <= a[1]).all(-1))
        triangles = triangles[~outside[triangles].any(-1)]
    if len(triangles):
        nt = len(triangles)
        # triangles that share an undirected edge are adjacent: sort the 3 nt edges and link equal neighbours
        e = np.sort(triangles[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2), axis=1)
        owner = np.repeat(np.arange(nt), 3)
        order = np.lexsort((e[:, 1], e[:, 0]))
        es, os_ = e[order], owner[order]
        same = (es[1:] == es[:-1]).all(-1)
        g = coo_matrix((np.ones(int(same.sum())), (os_[:-1][same], os_[1:][same])), shape=(nt, nt))
        _, labels = connected_components(g, directed=False)
        counts = np.bincount(labels)
        n_cluster = np.sort(counts)[-min(len(counts), keep)]
        triangles = triangles[counts[labels] >= n_cluster]
    used = np.zeros(len(vertices), dtype=bool)
    used[triangles.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    return (np.ascontiguousarray(vertices[used]), remap[triangles].astype(np.int32).reshape(-1, 3),
            np.ascontiguousarray(colors[used]))


def _check_mesh(vertices, triangles, colors):
    for name, t, dtype in (("vertices", vertices, torch.float32), ("triangles", triangles, torch.int32),
                           ("colors", colors, torch.float32)):
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_cuda:
            raise RuntimeError(f"filter_mesh_device: {name} must be a {dtype} CUDA tensor")
        if t.device != vertices.device:
            raise RuntimeError(f"filter_mesh_device: {name} must be on {vertices.device}, got {t.device}")
        if t.ndim != 2 or t.shape[1] != 3:
            raise RuntimeError(f"filter_mesh_device: {name} must be [N,3], got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise RuntimeError(f"filter_mesh_device: {name} must be contiguous")
    if colors.shape[0] != vertices.shape[0]:
        raise RuntimeError(f"filter_mesh_device: colors must be {tuple(vertices.shape)}, got {tuple(colors.shape)}")
    return int(vertices.shape[0]), int(triangles.shape[0])


def filter_mesh_device(mesh, aabb: Optional[np.ndarray] = None, keep: int = 10):
    """:func:`filter_mesh` on the device (``srf_mesh_filter_count`` / ``_emit``): the same crop to ``aabb`` ([2,3]
    float64, inclusive, each float32 coordinate compared as a float64), edge-connected clusters, the cut at the
    min(#clusters, keep)-th largest count and the compaction, equal to it element for element.  ``mesh`` is
    (vertices [Nv,3] float32, triangles [Nt,3] int32, colors [Nv,3] float32) on one CUDA device, e.g. the output of
    :func:`extract_triangle_mesh`; returns the filtered three as CUDA tensors on that device.  Runs on torch's current
    stream with one host read of the counts; an index outside [0, Nv) raises ``RuntimeError`` before any output is
    written."""
    vertices, triangles, colors = mesh
    Nv, Nt = _check_mesh(vertices, triangles, colors)
    dev = vertices.device
    box = None
    if aabb is not None:
        box = (ctypes.c_double * 6)(*np.asarray(aabb, dtype=np.float64).reshape(6).tolist())
    lib = _lib.load()
    ws = torch.empty(_lib.mesh_filter_workspace_bytes(lib, Nv, Nt), dtype=torch.uint8, device=dev)
    totals = torch.empty(4, dtype=torch.int32, device=dev)
    _lib.launch("srf_mesh_filter_count", dev, Nv, Nt, vertices.data_ptr(), triangles.data_ptr(), box,
                min(int(keep), 2**31 - 1), ws.data_ptr(), totals.data_ptr())
    nv, nt, _clusters, invalid = (int(x) for x in totals.cpu())
    if invalid:
        raise RuntimeError(f"filter_mesh_device: {invalid} triangles have an index outside [0, {Nv})")
    out_v = torch.empty((nv, 3), dtype=torch.float32, device=dev)
    out_c = torch.empty((nv, 3), dtype=torch.float32, device=dev)
    out_t = torch.empty((nt, 3), dtype=torch.int32, device=dev)
    _lib.launch("srf_mesh_filter_emit", dev, Nv, Nt, vertices.data_ptr(), colors.data_ptr(), triangles.data_ptr(),
                ws.data_ptr(), nv, nt, out_v.data_ptr(), out_c.data_ptr(), out_t.data_ptr())
    return out_v, out_t, out_c


def write_obj(path: str, vertices, triangles, colors) -> None:
    """``v x y z r g b`` lines (9 significant digits: float32 values read back exactly) and 1-based ``f a b c``."""
    v, t, c = _numpy(vertices), _numpy(triangles), _numpy(colors)
    with open(path, "w") as f:
        if len(v):
            np.savetxt(f, np.concatenate((v, c), axis=1).astype(np.float64), fmt="v %.9g %.9g %.9g %.9g %.9g %.9g")
        if len(t):
            np.savetxt(f, t.astype(np.int64) + 1, fmt="f %d %d %d")


class MeshExtractor:
    """LaRa's ``tools.meshExtractor.MeshExtractor`` (same constructor) with the TSDF fusion and marching cubes on the
    GPU.  ``extract`` takes the camera list (``uni_mesh_path(16, cfg.infer.dataset, sample, fov)`` in LaRa's
    evaluation.py) instead of the arguments LaRa passes on to ``uni_mesh_path``."""

    def __init__(self, gs_params, render, aabb, bg_color=(1.0, 1.0, 1.0)):
        self.background = torch.tensor(bg_color, dtype=torch.float32)
        self.aabb = np.array(aabb).reshape(2, 3) * 1.1 if aabb is not None else None
        self.gs_params = gs_params
        self.render = render

    def _render(self, cams, device):
        """(depth [V,H,W], acc [V,H,W], image [V,3,H,W]) of every camera, planar."""
        _centers, _shs, _opacity, _scaling, _rotation, mask = self.gs_params
        for cam in cams:
            cam.to_device(device)
        rays = [cam.get_rays().squeeze(0).to(device) for cam in cams]
        if hasattr(self.render, "render_views"):     # one forward-only launch set for the whole path
            out = self.render.render_views(cams, torch.stack(rays), _centers, _shs, _opacity[mask], _scaling[mask],
                                           _rotation[mask], device)
            return (out["depth"].permute(0, 3, 1, 2)[:, 0], out["acc_map"], out["image"].permute(0, 3, 1, 2))
        outs = [self.render.render_img(cam, r, _centers, _shs, _opacity[mask], _scaling[mask], _rotation[mask], device)
                for cam, r in zip(cams, rays)]
        return (torch.stack([o["depth"].reshape(o["acc_map"].shape) for o in outs]).contiguous(),
                torch.stack([o["acc_map"] for o in outs]).contiguous(),
                torch.stack([o["image"].permute(2, 0, 1) for o in outs]).contiguous())

    @torch.no_grad()
    def extract(self, save_mesh_path: Optional[str], cams: Sequence, voxel_size: float = 2 / 256,
                sdf_trunc: float = 0.08, alpha_thres: float = 0.08, depth_trunc: float = 10, device="cuda"):
        """Render ``cams``, fuse, extract and filter on the device, and write the mesh to ``save_mesh_path`` (OBJ; None
        writes nothing).  Returns (vertices [Nv,3], triangles [Nt,3] int32, colors [Nv,3]) as CPU tensors."""
        voxel_size, sdf_trunc, center, radius = mesh_settings(self.aabb, voxel_size, sdf_trunc)
        device = torch.device(device)
        depth, acc, image = self._render(cams, device)
        records = camera_records(cams, device, center, radius, depth_trunc)
        vol = tsdf_volume(depth, acc, records, voxel_size, sdf_trunc, alpha_thres, self.aabb)
        integrate(vol, depth, acc, image, records, alpha_thres)
        vertices, triangles, colors = (x.cpu() for x in filter_mesh_device(extract_triangle_mesh(vol), self.aabb))
        if save_mesh_path is not None:
            write_obj(save_mesh_path, vertices, triangles, colors)
        return vertices, triangles, colors
