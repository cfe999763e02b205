"""LaRa's mesh path on the GPU (DESIGN §3.15), stage by stage: the forward-only render of the 48 cameras (16 azimuths x
{0, -30, 30} deg, radius 1.905, fov 0.75, 512 x 512), TSDF integration, marching-cubes count, the host read of the
two totals, emit, the device filter (filter_mesh_device, its one host read of the counts included), the host copy of
the filtered mesh and the OBJ write, for scene(524288) and for an almost empty scene (the fixed costs), with LaRa's
aabb config.  The host filter (filter_mesh, with its copy of the unfiltered mesh) is timed in the same rounds for
comparison, and its output is checked equal to the device filter's.  Device stages are timed with CUDA events, host
stages with a host clock after a synchronise; each stage's median and range over --rounds rounds after one warm-up
round.  Also the peak memory, Nv / Nt before and after the filter and the integrate kernel against its floor computed
from the shapes.  open3d's CPU integration is not measured (it is not installed in any environment of this project).
Prints the card name and power limit, then one JSON line per scene.

    python tools/bench_mesh.py [--rounds 5] [--points 524288,64]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import card, summary  # noqa: E402  (tools/ is on sys.path when run as a script)

HBM_BPS = 3.35e12           # H100 SXM data sheet HBM3 bandwidth
FP32_FLOPS = 67e12          # H100 SXM data sheet dense FP32
FLOPS_PER_PROJECTION = 40   # 12 for the transform, 2 divides + sqrt counted as 1 each, bounds, the update (approx.)


def run_point(P: int, rounds: int) -> dict:
    from lara_b200 import _lib, mesh as MS, scene as S
    from lara_b200.renderer import Renderer
    dev = torch.device("cuda:0")
    sc = S.scene(P, 0)
    cams = S.mesh_path(16, 512, 512, 0.75)
    for c in cams:
        c.to_device(dev)
    rays = torch.cat([c.get_rays() for c in cams]).to(dev)
    r = Renderer(sh_degree=1, fused_activations=False)
    t = {k: sc[k].to(dev) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    opac, scl = torch.logit(t["opacities"]), torch.log(t["scales"])
    aabb = np.array([-0.5, -0.5, -0.5, 0.5, 0.5, 0.5]).reshape(2, 3) * 1.1
    vs, st, center, radius = MS.mesh_settings(aabb, 2 / 256, 0.08)
    rec = MS.camera_records(cams, dev, center, radius)
    ev = lambda: torch.cuda.Event(enable_timing=True)      # noqa: E731
    times = {k: [] for k in ("render", "integrate", "count", "readback", "emit", "filter_device", "filtered_copy",
                             "host_filter", "obj_write")}
    tmp = tempfile.mkdtemp()
    out = {}
    for rnd in range(rounds + 1):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        e = [ev() for _ in range(6)]
        e[0].record()
        with torch.no_grad():
            o = r.render_views(cams, rays, t["means3D"], t["shs"], opac, scl, t["rotations"], dev)
        depth, acc, image = o["depth"].permute(0, 3, 1, 2)[:, 0], o["acc_map"], o["image"].permute(0, 3, 1, 2)
        e[1].record()
        vol = MS.tsdf_volume(depth, acc, rec, vs, st, 0.08, aabb)     # grid choice and allocation: not timed
        e[2].record()
        MS.integrate(vol, depth, acc, image, rec, 0.08)
        e[3].record()
        dims = _lib.int3(vol.dims)
        ws = torch.empty(_lib.mesh_workspace_bytes(_lib.load(), vol.dims), dtype=torch.uint8, device=dev)
        totals = torch.empty(2, dtype=torch.int32, device=dev)
        e[4].record()
        _lib.launch("srf_mesh_count", dev, dims, vol.tsdf.data_ptr(), vol.weight.data_ptr(), ws.data_ptr(),
                    totals.data_ptr())
        e[5].record()
        e[5].synchronize()
        h0 = time.perf_counter()
        Nv, Nt = (int(x) for x in totals.cpu())
        h1 = time.perf_counter()
        verts = torch.empty((Nv, 3), dtype=torch.float32, device=dev)
        cols = torch.empty((Nv, 3), dtype=torch.float32, device=dev)
        tris = torch.empty((Nt, 3), dtype=torch.int32, device=dev)
        f = [ev(), ev()]
        f[0].record()
        _lib.launch("srf_mesh_emit", dev, _lib.int3(vol.n0), dims, vol.voxel_size, vol.tsdf.data_ptr(),
                    vol.color.data_ptr(), ws.data_ptr(), Nv, Nt, verts.data_ptr(), cols.data_ptr(), tris.data_ptr())
        f[1].record()
        g = [ev(), ev()]
        g[0].record()
        dv = MS.filter_mesh_device((verts, tris, cols), aabb)
        g[1].record()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        h2 = time.perf_counter()
        fv, ft, fc = (x.cpu().numpy() for x in dv)
        h3 = time.perf_counter()
        MS.write_obj(os.path.join(tmp, "mesh.obj"), fv, ft, fc)
        h4 = time.perf_counter()
        hv, ht, hc = MS.filter_mesh((verts, tris, cols), aabb)
        h5 = time.perf_counter()
        if not (np.array_equal(fv, hv) and np.array_equal(ft, ht) and np.array_equal(fc, hc)):
            raise SystemExit("bench_mesh: the device filter's output differs from the host filter's")
        if rnd == 0:      # warm-up round
            continue
        times["render"].append(e[0].elapsed_time(e[1]))
        times["integrate"].append(e[2].elapsed_time(e[3]))
        times["count"].append(e[4].elapsed_time(e[5]))
        times["readback"].append(1e3 * (h1 - h0))
        times["emit"].append(f[0].elapsed_time(f[1]))
        times["filter_device"].append(g[0].elapsed_time(g[1]))
        times["filtered_copy"].append(1e3 * (h3 - h2))
        times["host_filter"].append(1e3 * (h5 - h4))
        times["obj_write"].append(1e3 * (h4 - h3))
        out = {"dims": list(vol.dims), "voxels": int(np.prod(vol.dims)), "Nv": Nv, "Nt": Nt,
               "Nv_filtered": len(fv), "Nt_filtered": len(ft), "peak_bytes": int(peak)}
        del o, depth, acc, image, vol, ws, verts, cols, tris, dv
    N = out["voxels"]
    V, HW = len(cams), 512 * 512
    floor_bytes = 40 * N + V * HW * 4 * 5           # state read + written once; depth, acc, image read once
    floor_ops = N * V * FLOPS_PER_PROJECTION
    ms = {k: summary(v) for k, v in times.items()}
    t_int = ms["integrate"]["median"] * 1e-3
    out.update({
        "point": {"P": P, "views": V, "H": 512, "W": 512},
        "ms": ms,
        "integrate_floor": {"bytes": floor_bytes, "hbm_floor_ms": 1e3 * floor_bytes / HBM_BPS,
                            "voxel_view_projections": N * V, "fp32_floor_ms": 1e3 * floor_ops / FP32_FLOPS,
                            "achieved_GBps": floor_bytes / t_int / 1e9,
                            "achieved_G_projections_per_s": N * V / t_int / 1e9},
        "open3d_cpu": "not measured",
    })
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--points", default="524288,64", help="comma-separated Gaussian counts")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh: needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    for p in args.points.split(","):
        print(json.dumps(run_point(int(p), args.rounds)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
