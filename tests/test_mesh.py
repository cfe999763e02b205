"""Mesh extractor, no GPU: LaRa's extract glue (recorded from tools/meshExtractor.py with stub open3d, renderer and
camera path into tests/golden/reference/test_mesh.npz; run this file as a script to write it), the float64
restatement's grid-bound equivalence and filter, and host-only argument checks of the C entries."""
import ctypes
import importlib.util
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import fingerprint, reference_record

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GLUE_CASES = {"aabb": [-0.5, -0.5, -0.5, 0.5, 0.5, 0.5], "noaabb": None}
GLUE_H, GLUE_W, GLUE_N = 24, 32, 3         # a non-square image, 3 azimuths x 3 elevations


class _Cam:
    """The attributes of LaRa's MiniCam that extract reads."""

    def __init__(self, c2w, H, W, fov):
        from lara_b200 import scene as S
        cam = S.camera_from_c2w(c2w, H, W, fov, fov * H / W)
        self.image_width, self.image_height, self.FoVx, self.FoVy = W, H, fov, fov * H / W
        self.world_view_transform, self.camera_center = cam.viewmatrix, cam.campos

    def to_device(self, device):
        pass

    def get_rays(self):
        return torch.zeros(1, self.image_height, self.image_width, 6)


def glue_cameras():
    from lara_b200 import scene as S
    return [_Cam(S.look_at_c2w(2 * math.pi * a / GLUE_N + 0.1, math.radians(e), 1.905), GLUE_H, GLUE_W, 0.75)
            for e in (0.0, -30.0, 30.0) for a in range(GLUE_N)]


def glue_render(v):
    """Seeded depth [H,W,1], acc [H,W], image [H,W,3] of view v: some acc below 0.08, some depth beyond 3."""
    g = torch.Generator().manual_seed(300 + v)
    return {"depth": torch.rand(GLUE_H, GLUE_W, 1, generator=g) * 3.0 + 0.5,
            "acc_map": torch.rand(GLUE_H, GLUE_W, generator=g) * 0.3,
            "image": torch.rand(GLUE_H, GLUE_W, 3, generator=g)}


def record_reference(lara, dev):
    """LaRa's MeshExtractor.extract on the CPU with a recording open3d stub (tests/golden/make_reference_records.py):
    per integrated view the RGBD images, intrinsic, extrinsic and depth_trunc open3d receives, and the volume's
    voxel_length and sdf_trunc."""
    calls, volume = [], {}

    class Stop(Exception):
        pass

    o3d = types.ModuleType("open3d")

    class Volume:
        def __init__(self, voxel_length, sdf_trunc, color_type):
            volume.update(voxel_length=voxel_length, sdf_trunc=sdf_trunc)

        def integrate(self, rgbd, intrinsic, extrinsic):
            calls.append(dict(rgbd, intrinsic=np.array(intrinsic, np.float64), extrinsic=np.array(extrinsic)))

        def extract_triangle_mesh(self):
            raise Stop()
    o3d.pipelines = types.SimpleNamespace(integration=types.SimpleNamespace(
        ScalableTSDFVolume=Volume, TSDFVolumeColorType=types.SimpleNamespace(RGB8=0)))
    o3d.camera = types.SimpleNamespace(PinholeCameraIntrinsic=lambda width, height, cx, cy, fx, fy: (
        width, height, cx, cy, fx, fy))
    o3d.geometry = types.SimpleNamespace(
        Image=lambda a: np.array(a),
        RGBDImage=types.SimpleNamespace(create_from_color_and_depth=lambda color, depth, depth_trunc, **kw: dict(
            color=color, depth=depth, depth_trunc=np.float64(depth_trunc))))
    cams = glue_cameras()
    path = types.ModuleType("tools.gen_video_path")
    path.uni_mesh_path = lambda N, data, sample, fov=None: cams
    stubs = {"open3d": o3d, "tools": types.ModuleType("tools"), "tools.gen_video_path": path}
    for name in ("matplotlib", "matplotlib.pyplot"):
        if importlib.util.find_spec(name.split(".")[0]) is None:
            stubs[name] = types.ModuleType(name)
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    try:
        return _record_with_stubs(lara, calls, volume, Stop)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _record_with_stubs(lara, calls, volume, Stop):
    spec = importlib.util.spec_from_file_location("ref_mesh_extractor", os.path.join(lara, "tools", "meshExtractor.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)

    class Torch:        # the constructor puts its (unused) background on "cuda"; keep it on the CPU
        def __getattr__(self, k):
            return getattr(torch, k)

        @staticmethod
        def tensor(*a, device=None, **kw):
            return torch.tensor(*a, **kw)
    mod.torch = Torch()

    class Render:
        def __init__(self):
            self.v = 0

        def render_img(self, cam, rays, *args):
            out = glue_render(self.v)
            self.v += 1
            return out
    gs = (torch.zeros(4, 3), torch.zeros(4, 4, 3), torch.zeros(4, 1), torch.zeros(4, 2), torch.zeros(4, 4),
          torch.ones(4, dtype=torch.bool))
    recs = {}
    for case, aabb in GLUE_CASES.items():
        calls.clear()
        volume.clear()
        ex = mod.MeshExtractor(gs, Render(), aabb)
        with pytest.raises(Stop):
            ex.extract("unused.ply", "stub", device="cpu")
        rec = {"voxel_length": np.float64(volume["voxel_length"]), "sdf_trunc": np.float64(volume["sdf_trunc"])}
        for v, c in enumerate(calls):
            rec[f"color_{v}"] = fingerprint(c["color"])
            rec[f"depth_{v}"] = fingerprint(c["depth"])
            rec[f"depth_trunc_{v}"] = c["depth_trunc"]
            rec[f"intrinsic_{v}"] = c["intrinsic"]
            rec[f"extrinsic_{v}"] = c["extrinsic"]
        recs[case] = rec
    return recs


@pytest.mark.parametrize("case", sorted(GLUE_CASES))
def test_glue_restatement_matches_laras_extract(case):
    """What lara_b200.mesh feeds the kernel is what LaRa's extract feeds open3d, bit for bit: the volume's voxel size
    and truncation, per view the intrinsic, the extrinsic, depth_trunc, the alpha-masked depth and the uint8 colour."""
    from lara_b200 import mesh as MS
    ref = reference_record("test_mesh", case)
    cams = glue_cameras()
    aabb = np.array(GLUE_CASES[case]).reshape(2, 3) * 1.1 if GLUE_CASES[case] else None
    vs, st, center, radius = MS.mesh_settings(aabb, 2 / 256, 0.08)
    assert np.float64(vs) == ref["voxel_length"] and np.float64(st) == ref["sdf_trunc"]
    rec = MS.camera_records64(cams, center, radius, 10)
    for v in range(len(cams)):
        fx, fy, cx, cy, dt = (rec[v, k] for k in (MS.CAM_FX, MS.CAM_FY, MS.CAM_CX, MS.CAM_CY, MS.CAM_DEPTH_TRUNC))
        assert np.array_equal(ref[f"intrinsic_{v}"], [GLUE_W, GLUE_H, cx, cy, fx, fy])
        assert np.array_equal(ref[f"extrinsic_{v}"].astype(np.float64), rec[v, :16].reshape(4, 4))
        assert np.float64(dt) == ref[f"depth_trunc_{v}"]
        r = glue_render(v)
        depth = np.where(r["acc_map"].numpy()[..., None] < np.float32(0.08), np.float32(0), r["depth"].numpy())
        assert fingerprint(depth) == ref[f"depth_{v}"]
        rgb = np.trunc(r["image"].numpy() * np.float32(255)).astype(np.uint8)
        assert fingerprint(rgb) == ref[f"color_{v}"]
    assert f"color_{len(cams)}" not in ref


# ---- float64 restatement: grid choice and filter ----

def _sphere_views(V, H, W, r=0.3, seed=0):
    """Analytic renders of a sphere of radius r at the origin on a camera ring: depth = z of the ray's first hit."""
    from lara_b200 import scene as S
    from lara_b200 import mesh as MS
    cams = S.mesh_path(max(V // 3, 1), H, W, 0.75)[:V]
    rec = MS.camera_records64(cams, None, None, 10)
    depth, acc, image = np.zeros((V, H, W), np.float32), np.zeros((V, H, W), np.float32), np.zeros((V, 3, H, W), np.float32)
    g = np.random.default_rng(seed)
    for v, cam in enumerate(cams):
        E = rec[v, :16].reshape(4, 4)
        o = -E[:3, :3].T @ E[:3, 3]
        y, x = np.mgrid[0:H, 0:W] + 0.5
        d = np.stack(((x - W / 2) / rec[v, 16], (y - H / 2) / rec[v, 17], np.ones_like(x)), -1)
        dw = d @ E[:3, :3]
        a, b, c = (dw * dw).sum(-1), 2 * dw @ o, o @ o - r * r
        disc = b * b - 4 * a * c
        hit = disc > 0
        t = np.where(hit, (-b - np.sqrt(np.where(hit, disc, 0))) / (2 * a), 0)
        depth[v] = np.where(hit, t, 0)
        acc[v] = np.where(hit, 1.0, 0.0)
        image[v] = g.random((3, H, W))
    return cams, torch.from_numpy(rec.astype(np.float32)), torch.from_numpy(depth), torch.from_numpy(acc), image


def _restated_mesh(n0, dims, vs, st, depth, acc, image, rec, aabb):
    from oracle import mesh64
    tsdf, w, col, _ = mesh64.integrate(mesh64.grid_voxels(n0, dims), vs, st, depth, acc, image, rec, 0.08)
    nz_, ny_, nx_ = dims[2], dims[1], dims[0]
    v, t, c = mesh64.extract(n0, dims, vs, tsdf.reshape(nz_, ny_, nx_), w.reshape(nz_, ny_, nx_),
                             col.T.reshape(3, nz_, ny_, nx_))
    return mesh64.filter_mesh(v, t, c, aabb)


@pytest.mark.parametrize("with_aabb", [False, True])
def test_grid_bound_gives_the_unbounded_volumes_mesh(with_aabb):
    """The block tsdf_volume chooses and the same block grown by 8 voxels on every side give the same filtered mesh."""
    from lara_b200 import mesh as MS
    cams, rec, depth, acc, image = _sphere_views(6, 40, 48)
    aabb = np.array([[-0.25, -0.5, -0.5], [0.5, 0.5, 0.5]]) if with_aabb else None
    vs, st = 0.02, 0.05
    vol = MS.tsdf_volume(depth, acc, rec, vs, st, 0.08, aabb)
    assert not vol.empty
    a = _restated_mesh(vol.n0, vol.dims, vol.voxel_size, vol.sdf_trunc, depth.numpy(), acc.numpy(), image,
                       rec.numpy(), aabb)
    b = _restated_mesh(tuple(x - 8 for x in vol.n0), tuple(x + 16 for x in vol.dims), vol.voxel_size, vol.sdf_trunc,
                       depth.numpy(), acc.numpy(), image, rec.numpy(), aabb)
    assert len(a[1]) > 200
    # same triangles over the same vertex positions (vertex ids differ with the block's origin)
    ta = {tuple(x) for x in np.round(a[0][a[1]].reshape(-1, 9) / 1e-9).astype(np.int64)}
    tb = {tuple(x) for x in np.round(b[0][b[1]].reshape(-1, 9) / 1e-9).astype(np.int64)}
    assert ta == tb


def test_filter_matches_the_restatement():
    """lara_b200.mesh.filter_mesh and oracle.mesh64.filter_mesh agree on a mesh with many components and ties."""
    from lara_b200 import mesh as MS
    from oracle import mesh64
    rng = np.random.default_rng(5)
    f = np.ones((26, 26, 26))
    f[1:-1, 1:-1, 1:-1] = np.where(rng.random((24, 24, 24)) < 0.12, -1.0, 1.0)
    v, t, c = mesh64.extract((0, 0, 0), (26, 26, 26), 0.05, f, np.ones_like(f), rng.random((3, 26, 26, 26)) * 255)
    for aabb in (None, np.array([[0.2, 0.1, 0.0], [1.0, 1.2, 0.9]])):
        for keep in (1, 10, 40):
            mine = MS.filter_mesh((v, t, c), aabb, keep)
            ref = mesh64.filter_mesh(v, t, c, aabb, keep)
            assert len(mine[1]) > 0
            for x, y in zip(mine, ref):
                assert np.array_equal(np.asarray(x), np.asarray(y))


def test_write_obj_reads_back(tmp_path):
    from lara_b200 import mesh as MS
    rng = np.random.default_rng(1)
    v = rng.random((50, 3)).astype(np.float32) - 0.5
    c = rng.random((50, 3)).astype(np.float32)
    t = rng.integers(0, 50, (70, 3)).astype(np.int32)
    MS.write_obj(str(tmp_path / "m.obj"), v, t, c)
    rv, rc, rt = read_obj(str(tmp_path / "m.obj"))
    assert np.array_equal(rv, v) and np.array_equal(rc, c) and np.array_equal(rt, t)


def read_obj(path):
    vs, fs = [], []
    with open(path) as f:
        for line in f:
            p = line.split()
            if p and p[0] == "v":
                vs.append([float(x) for x in p[1:7]])
            elif p and p[0] == "f":
                fs.append([int(x) - 1 for x in p[1:4]])
    v = np.array(vs, np.float32).reshape(-1, 6)
    return v[:, :3], v[:, 3:], np.array(fs, np.int32).reshape(-1, 3)


# ---- host-only argument checks of the C entries ----

def _i3(*x):
    return (ctypes.c_int * 3)(*x)


def test_mesh_workspace_query(lib):
    from lara_b200 import _lib
    b = _lib.mesh_workspace_bytes(lib, (10, 20, 30))
    N = 6000
    assert b >= 4 * (3 * N + 1) + 4 * (N + 1) + N and b % 256 == 0
    assert _lib.mesh_workspace_bytes(lib, (1, 1, 1)) > 0
    n = ctypes.c_size_t()
    assert lib.srf_mesh_workspace_bytes(_i3(0, 4, 4), ctypes.byref(n)) != 0
    assert lib.srf_mesh_workspace_bytes(None, ctypes.byref(n)) != 0
    assert lib.srf_mesh_workspace_bytes(_i3(4, 4, 4), None) != 0


def test_grids_whose_indices_exceed_int32_are_rejected(lib):
    """Vertex ids (3 per voxel) and triangle offsets (up to 5 per voxel) are int32: a block of more than
    2^31 / 5 voxels is refused before anything is enqueued, by every entry."""
    n = ctypes.c_size_t()
    assert lib.srf_mesh_workspace_bytes(_i3(750, 750, 750), ctypes.byref(n)) == 0      # 421.9 M voxels: accepted
    assert lib.srf_mesh_workspace_bytes(_i3(1024, 1024, 512), ctypes.byref(n)) != 0
    assert b"over the limit" in lib.srf_last_error()
    assert lib.srf_mesh_count(None, _i3(1024, 1024, 512), 8, 8, 256, 8) != 0
    assert lib.srf_tsdf_integrate(None, _i3(0, 0, 0), _i3(1024, 1024, 512), 0.01, 0.02, 8, 8, 8, 1, 4, 4, 8, 8, 8, 8,
                                  0.08) != 0
    assert b"over the limit" in lib.srf_last_error()
    assert lib.srf_tsdf_integrate(None, _i3(1 << 24, 0, 0), _i3(4, 4, 4), 0.01, 0.02, 8, 8, 8, 1, 4, 4, 8, 8, 8, 8,
                                  0.08) != 0
    assert b"2^24" in lib.srf_last_error()


def test_mesh_entries_reject_null_and_bad_arguments(lib):
    d, z = _i3(4, 4, 4), _i3(0, 0, 0)
    integ = [None, z, d, 0.01, 0.02, 8, 8, 8, 1, 4, 4, 8, 8, 8, 8, 0.08]
    for i, bad in ((1, None), (2, None), (2, _i3(4, 0, 4)), (3, 0.0), (4, -1.0), (5, None), (6, None), (7, None),
                   (12, None), (14, None), (8, -1), (9, 0)):
        args = list(integ)
        args[i] = bad
        assert lib.srf_tsdf_integrate(*args) != 0, i
        assert lib.srf_last_error().startswith(b"srf_tsdf_integrate"), i
    cnt = [None, d, 8, 8, 256, 8]
    for i, bad in ((1, None), (2, None), (3, None), (4, None), (4, 264), (5, None)):
        args = list(cnt)
        args[i] = bad
        assert lib.srf_mesh_count(*args) != 0, i
    emit = [None, z, d, 0.01, 8, 8, 256, 1, 1, 8, 8, 8]
    for i, bad in ((1, None), (3, float("nan")), (4, None), (5, None), (6, None), (7, -1), (9, None), (10, None),
                   (11, None)):
        args = list(emit)
        args[i] = bad
        assert lib.srf_mesh_emit(*args) != 0, i
        assert lib.srf_last_error().startswith(b"srf_mesh_emit"), i


if __name__ == "__main__":
    # python tests/test_mesh.py OUT_DIR LARA_CHECKOUT: record LaRa's glue, as tests/golden/make_reference_records.py
    # does for the other modules
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    out_dir, lara = sys.argv[1:3]
    os.makedirs(out_dir, exist_ok=True)
    save(out_dir, "test_mesh", record_reference(lara, "cpu"))
