"""Host-side mirror of the reference's Python surface: names, argument checks, error behaviour
(DSR/diff_surfel_rasterization/__init__.py), all without a GPU."""
import inspect
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_drop_in_names_import_without_gpu():
    import diff_surfel_rasterization as d
    assert d.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix",
        "projmatrix", "sh_degree", "campos", "prefiltered", "debug")
    sig = inspect.signature(d.GaussianRasterizer.forward)
    assert list(sig.parameters) == ["self", "means3D", "means2D", "opacities", "shs", "colors_precomp",
                                    "scales", "rotations", "cov3D_precomp"]
    assert callable(d.rasterize_gaussians)
    assert hasattr(d.GaussianRasterizer, "markVisible")


def _settings():
    import diff_surfel_rasterization as d
    z = torch.zeros(4, 4)
    return d.GaussianRasterizationSettings(16, 16, 1.0, 1.0, torch.zeros(3), 1.0, z, z, 0, torch.zeros(3), False, False)


def test_forward_argument_validation_matches_reference():
    import diff_surfel_rasterization as d
    r = d.GaussianRasterizer(_settings())
    m = torch.zeros(4, 3)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), scales=torch.zeros(4, 2), rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), colors_precomp=m,
          scales=torch.zeros(4, 2), rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), shs=torch.zeros(4, 1, 3))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.zeros(4, 2),
          rotations=torch.zeros(4, 4), cov3D_precomp=torch.zeros(4, 9))


def test_cpu_tensors_are_rejected_not_silently_computed():
    """No CPU fallback: CPU tensors raise, like the reference's CHECK_INPUT (rasterize_points.cu:27-29)."""
    import diff_surfel_rasterization as d
    r = d.GaussianRasterizer(_settings())
    m = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.zeros(4, 2),
          rotations=torch.zeros(4, 4))


def test_shape_checks():
    from lara_b200 import rasterizer as R

    class Fake(torch.Tensor):
        pass
    with pytest.raises(RuntimeError, match=r"means3D must have dimensions \(num_points, 3\)"):
        R._normalise_inputs(torch.zeros(4, 2), None, None, torch.zeros(4, 1), None, None, None)
    with pytest.raises(RuntimeError, match=r"scales must have dimensions \(num_points, 2\)"):
        R._normalise_inputs(torch.zeros(4, 3), None, None, torch.zeros(4, 1), torch.zeros(4, 3), torch.zeros(4, 4), None)
    with pytest.raises(RuntimeError, match=r"rotations must have dimensions \(num_points, 4\)"):
        R._normalise_inputs(torch.zeros(4, 3), None, None, torch.zeros(4, 1), torch.zeros(4, 2), torch.zeros(4, 3), None)


def test_empty_tensor_means_not_given():
    from lara_b200 import rasterizer as R
    assert R._opt(torch.empty(0)) is None and R._opt(None) is None
    t = torch.zeros(2, 3)
    assert R._opt(t) is t


def test_optimistic_capacity_policy():
    from lara_b200 import rasterizer as R
    dev = torch.device("cuda", 0)
    R._capacity_hwm.clear()
    assert R.initial_capacity(1000, dev) == 1 << 16
    assert R.initial_capacity(100000, dev) == 800000
    R._note_rendered(2_000_000, dev)
    assert R.initial_capacity(1000, dev) >= 2_500_000
    R._note_rendered(10, dev)           # high-water mark never shrinks
    assert R.initial_capacity(1000, dev) >= 2_500_000
    R._capacity_hwm.clear()


def test_scene_generator_is_deterministic_and_shaped():
    from lara_b200 import scene as S
    a, b = S.scene(257, 3, sh_degree=3), S.scene(257, 3, sh_degree=3)
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        assert torch.equal(a[k], b[k])
    assert a["shs"].shape == (257, 16, 3) and a["opacities"].shape == (257, 1)
    assert torch.allclose(a["rotations"].norm(dim=-1), torch.ones(257), atol=1e-6)
    cams = S.cameras(4, 64, 48, 1)
    for c in cams:
        # MiniCam convention: viewmatrix = w2c^T, campos = -c2w[:3,3]; origin lies in front of the camera
        w2c = c.viewmatrix.t()
        assert torch.allclose(w2c @ c.c2w, torch.eye(4), atol=1e-5)
        assert torch.allclose(c.campos, -c.c2w[:3, 3])
        assert abs(float(w2c[2, 3]) - 1.905) < 1e-4
    gc, ga = S.upstream_grads(8, 8, 0, lara_like=True)
    assert float(ga[5].abs().max()) == 0.0 and float(ga[7].abs().max()) == 0.0 and float(ga[6].abs().max()) > 0


def test_product_never_touches_the_oracle():
    """lara_b200/ and the drop-in shim must not import, load or execute anything under oracle/."""
    pat = re.compile(r"\boracle\b|liboracle|_ref\b")
    for pkg in ("lara_b200", "diff_surfel_rasterization"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, pkg)):
            for fn in files:
                if fn.endswith((".py", ".cu", ".cuh", ".h")):
                    src = open(os.path.join(dirpath, fn)).read()
                    code = "\n".join(l for l in src.splitlines() if "import" in l or "CDLL" in l or "dlopen" in l)
                    assert not pat.search(code), f"{pkg}/{fn} references the oracle"


def test_view_sharding_partition():
    from lara_b200.sharded import shard_views
    for n, w in ((8, 1), (8, 2), (32, 8), (7, 4), (3, 8)):
        seen = sorted(v for r in range(w) for v in shard_views(n, r, w))
        assert seen == list(range(n))
        sizes = [len(shard_views(n, r, w)) for r in range(w)]
        assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        shard_views(8, 2, 2)


def test_grad_buffer_layout():
    from lara_b200.sharded import GradBuffer
    g = GradBuffer(5, 4, "cpu")
    assert g.views["means3D"].shape == (5, 3) and g.views["sh"].shape == (5, 4, 3)
    assert g.views["opacities"].shape == (5, 1) and g.views["rotations"].shape == (5, 4)
    base = g.flat.data_ptr()
    for k, v in g.views.items():
        assert v.is_contiguous() and (v.data_ptr() - base) % 16 == 0
    g.views["scales"].fill_(2.0)
    assert float(g.flat.sum()) == 20.0
    g.zero_()
    assert float(g.flat.abs().sum()) == 0.0


def test_concat_views_matches_the_callers_cat():
    """multiview.concat_views == what lightning/network.py:525 builds from per-view frames
    (`torch.cat([frame[k] for frame in views], dim=1)`)."""
    import torch
    from lara_b200.multiview import concat_views
    V, H, W = 3, 4, 5
    g = torch.Generator().manual_seed(0)
    stacked = {"image": torch.rand((V, H, W, 3), generator=g), "acc_map": torch.rand((V, H, W), generator=g),
               "radii": torch.zeros((V, 7), dtype=torch.int32)}
    out = concat_views(stacked)
    assert sorted(out) == ["acc_map", "image"]              # radii is per Gaussian, not an image
    frames = [{k: stacked[k][v] for k in ("image", "acc_map")} for v in range(V)]
    for k in ("image", "acc_map"):
        assert torch.equal(out[k], torch.cat([f[k] for f in frames], dim=1))


def test_render_scene_views_rejects_empty_view_list():
    import pytest
    import torch
    from lara_b200.multiview import render_scene_views
    z = torch.zeros((0, 3))
    with pytest.raises(ValueError):
        render_scene_views(z, z, z, z, z, [])


def _cpu_settings(H=64, W=48, fov=0.5, deg=1, seed=0, **kw):
    from lara_b200 import rasterizer as R
    g = torch.Generator().manual_seed(seed)
    d = dict(image_height=H, image_width=W, tanfovx=fov, tanfovy=fov, bg=torch.rand(3, generator=g), scale_modifier=1.0,
             viewmatrix=torch.rand(4, 4, generator=g), projmatrix=torch.rand(4, 4, generator=g), sh_degree=deg,
             campos=torch.rand(3, generator=g), prefiltered=False, debug=False)
    d.update(kw)
    return R.GaussianRasterizationSettings(**d)


def test_camera_records_follow_the_header_layout():
    """pack_cameras: [V, SRF_CAM_FLOATS] rows = view matrix (row-major as stored) | campos | bg | zero pad, at the
    offsets include/surfel_rasterizer.h names."""
    import re
    from lara_b200 import _lib, rasterizer as R
    hdr = open(os.path.join(ROOT, "include", "surfel_rasterizer.h")).read()
    consts = {k: int(v) for k, v in re.findall(r"#define (SRF_CAM_[A-Z]+) (\d+)", hdr)}
    assert (consts["SRF_CAM_FLOATS"], consts["SRF_CAM_VIEW"], consts["SRF_CAM_CAMPOS"], consts["SRF_CAM_BG"]) == \
        (_lib.CAM_FLOATS, _lib.CAM_VIEW, _lib.CAM_CAMPOS, _lib.CAM_BG)
    sets = [_cpu_settings(seed=s) for s in range(3)]
    sets[1] = sets[1]._replace(viewmatrix=sets[1].viewmatrix.t())          # LaRa passes a transposed (non-contiguous) view
    cams = R.pack_cameras(sets, torch.device("cpu"))
    assert cams.shape == (3, _lib.CAM_FLOATS) and cams.dtype == torch.float32 and cams.is_contiguous()
    for v, rs in enumerate(sets):
        assert torch.equal(cams[v, _lib.CAM_VIEW:_lib.CAM_VIEW + 16], rs.viewmatrix.reshape(16))
        assert torch.equal(cams[v, _lib.CAM_CAMPOS:_lib.CAM_CAMPOS + 3], rs.campos)
        assert torch.equal(cams[v, _lib.CAM_BG:_lib.CAM_BG + 3], rs.bg)
        assert torch.count_nonzero(cams[v, _lib.CAM_BG + 3:]) == 0


def test_views_of_a_batched_call_must_share_size_fov_and_degree():
    from lara_b200.multiview import shared_view_settings
    a = _cpu_settings()
    assert shared_view_settings([a, _cpu_settings(seed=1)]) == (64, 48, 0.5, 0.5, 1, False, False)
    assert shared_view_settings([a, _cpu_settings(seed=1, debug=True)])[-1] is True       # one debug view makes the call eager
    with pytest.raises(RuntimeError, match="one image size"):
        shared_view_settings([a, _cpu_settings(H=32)])
    with pytest.raises(RuntimeError, match="field of view"):
        shared_view_settings([a, _cpu_settings(fov=0.6)])
    with pytest.raises(RuntimeError, match="SH degree"):
        shared_view_settings([a, _cpu_settings(deg=2)])


def test_view_workspaces_are_the_one_view_ones_back_to_back():
    """srf_views_workspace_bytes (host only): V per-view workspaces at a byte stride of the single-view size."""
    from lara_b200 import _lib
    lib = _lib.load()
    P, H, W, cap = 5000, 200, 136, 123456
    g1, t1, i1, e1, p1, s1 = _lib.views_sizes(lib, 1, P, H, W, cap)
    for V in (1, 3, 8):
        g, t, i, e, pl, s = _lib.views_sizes(lib, V, P, H, W, cap)
        assert (g, t, i, e, pl) == (V * g1, V * t1, V * i1, V * e1, V * p1)
        assert s >= s1 and s % 256 == 0
    assert all(x % 256 == 0 for x in (g1, t1, i1, e1, p1))


def test_next_row_entries_validate_before_touching_the_device():
    """The fused epilogue / loss / decoder-layout entries take raw pointers underneath, so wrong inputs must raise the
    clear errors the reference's torch ops would (checked on the CPU: the checks come before any launch)."""
    from lara_b200.decoder_layout import gaussians_from_decoder
    from lara_b200.epilogue import render_img_epilogue
    from lara_b200.loss import scene_loss
    H, W = 8, 12
    with pytest.raises(RuntimeError, match="rendered_image must be a CUDA tensor"):
        render_img_epilogue(torch.zeros(3, H, W), torch.zeros(8, H, W), torch.zeros(H, W, 6), torch.eye(4), 0.0, "")
    with pytest.raises(RuntimeError, match=r"parameters must be \[B, N, K\*C\]"):
        gaussians_from_decoder(torch.zeros(5, 26), torch.zeros(5, 3), 2, 3, 0.0, 0.0, 0.1)
    with pytest.raises(RuntimeError, match=r"last dim 27 != K\*\(10\+sh_dim\) = 26"):
        gaussians_from_decoder(torch.zeros(1, 5, 27), torch.zeros(5, 3), 2, 3, 0.0, 0.0, 0.1)
    with pytest.raises(RuntimeError, match="group_centers must hold N = 5 voxel centres, got 4"):
        gaussians_from_decoder(torch.zeros(1, 5, 26), torch.zeros(4, 3), 2, 3, 0.0, 0.0, 0.1)
    with pytest.raises(RuntimeError, match="parameters must be a float32 CUDA tensor"):
        gaussians_from_decoder(torch.zeros(1, 5, 26), torch.zeros(5, 3), 2, 3, 0.0, 0.0, 0.1)
    out = {"image": torch.zeros(2, H, W, 3), "rend_normal": torch.zeros(2, H, W, 3), "depth_normal": torch.zeros(2, H, W, 3),
           "rend_dist": torch.zeros(2, H, W), "acc_map": torch.zeros(2, H, W)}
    with pytest.raises(RuntimeError, match="scene_loss: .* must be a contiguous float32 CUDA tensor"):
        scene_loss(out, torch.zeros(2, H, W, 3), 5000)
