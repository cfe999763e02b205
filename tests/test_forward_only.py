"""Forward-only rendering, host side (no GPU needed): the for_backward flag of srf_scenes_forward, its stage-2 re-run
and the workspace query, their argument checks, and the rule by which the public wrappers pick the forward-only path --
taken iff no gradient can flow (grad mode off, or no tensor input requires grad) -- driven with stand-ins for the raw
forward functions."""
import ctypes
import os
import re

import pytest
import torch

from lara_b200 import _lib
from lara_b200 import multiview as MV
from lara_b200 import rasterizer as R

from test_abi import ROOT, declared_symbols

# the forward-only twins of ABI 11, folded into the flag, and the one-scene entries of ABI 12, now S = 1 of the scene
# entries
REMOVED = ("srf_views_forward_inference", "srf_views_forward_inference_render", "srf_views_inference_workspace_bytes",
           "srf_views_forward", "srf_views_subset_forward", "srf_views_backward")


def align256(x):
    return (x + 255) // 256 * 256


def test_forward_only_is_a_flag_of_the_scene_forward_entries(lib):
    syms = declared_symbols()
    for name in REMOVED:
        assert name not in syms and name not in _lib.SIGNATURES and not hasattr(lib, name), name
    assert lib.srf_abi_version() == _lib.ABI_VERSION == 13
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "surfel_rasterizer.h")).read(), flags=re.S)
    header = re.sub(r"\s+", " ", header)
    for name in ("srf_scenes_forward", "srf_views_forward_render"):
        assert re.search(rf"\b{name}\([^;]*, int for_backward\);", header), name
        assert _lib.SIGNATURES[name][1][-1] is ctypes.c_int, name
    assert "srf_views_workspace_bytes(int V, int P, int H, int W, size_t capacity, int for_backward, size_t bytes[6]);" \
        in header


@pytest.mark.parametrize("V,P,H,W,capacity", [(1, 1000, 300, 500, 12345), (8, 131072, 512, 512, 1 << 20),
                                              (48, 524288, 512, 512, 8 * 524288), (3, 0, 16, 16, 0)])
def test_forward_only_workspace_sizes(lib, V, P, H, W, capacity):
    geom, tile, image, entries, plist, scratch = _lib.views_sizes(lib, V, P, H, W, capacity, for_backward=False)
    tg, tt, ti, te, tp, _ = _lib.views_sizes(lib, V, P, H, W, capacity, for_backward=True)
    assert plist == align256(4 * capacity) * V
    assert 8 * plist <= tp
    assert tp - plist >= 32 * capacity * V              # the contribution record is what goes
    assert image == 0 and ti > 0
    assert scratch == 0
    assert (geom, tile, entries) == (tg, tt, te)


def test_workspace_query_rejects_bad_arguments_with_either_flag(lib):
    n = (ctypes.c_size_t * 6)()
    for for_backward in (0, 1):
        for args in [(0, 1, 16, 16, 0), (1, -1, 16, 16, 0), (1, 0, 0, 16, 0), (1, 0, 16, -2, 0)]:
            assert lib.srf_views_workspace_bytes(*args, for_backward, n) != 0
            assert b"srf_views_workspace_bytes: bad arguments" == lib.srf_last_error()
        assert lib.srf_views_workspace_bytes(1, 0, 16, 16, 0, for_backward, None) != 0


def _forward_args(V=1, P=4, D=0, H=16, W=16, capacity=0, geom=None, tile=None, entries=None, plist=None, image=None,
                  out=None, for_backward=0):
    """srf_scenes_forward's arguments for one scene (S = 1) of V views."""
    cams = (ctypes.c_float * 24)()
    args = [None, 1, V, P, D, 1, None, None, None, None, None, None, None, ctypes.addressof(cams),
            _lib.tan_fov_array([(1.0, 1.0)]), H, W, 0, capacity, None, geom, tile, entries, plist, image, out, out,
            None, None, 0, for_backward]
    return args, cams


@pytest.mark.parametrize("case", [dict(V=0), dict(H=16 * 65535 + 1), dict(), dict(tile=0x1010),
                                  dict(tile=0x1000, D=4)])
def test_scenes_forward_only_rejects_what_the_training_forward_rejects(lib, case):
    """Same arguments, the same message byte for byte with either flag; every case fails before anything is
    enqueued."""
    msgs = []
    for for_backward in (0, 1):
        args, _cams = _forward_args(**case, for_backward=for_backward)
        assert lib.srf_scenes_forward(*args) != 0
        msgs.append(lib.srf_last_error())
    assert msgs[0].startswith(b"srf_scenes_forward: ") and msgs[0] == msgs[1]


def test_scenes_forward_rejects_null_or_misaligned_workspaces_before_any_cuda_call(lib):
    """Without a device any CUDA call would fail with a CUDA error; these fail with the argument check's message, with
    either flag: the checks of both stages come before stage 1 enqueues anything."""
    x = 0x10000          # a 256-byte aligned address that is never dereferenced: every call below fails its checks
    cases = [
        (dict(P=0, tile=x, capacity=64, entries=x, plist=None, out=x), "null binning buffers"),
        (dict(P=0, tile=x, capacity=64, entries=x, plist=x + 4, out=x), "entries and point_list must be 256-byte aligned"),
        (dict(P=0, tile=x, capacity=64, entries=x + 8, plist=x, out=x), "entries and point_list must be 256-byte aligned"),
        (dict(P=0, tile=x, capacity=64, entries=x, plist=x, out=None), "null required pointer"),
    ]
    for for_backward in (0, 1):
        # the training forward needs an image_state; the forward-only one does not use it
        image = x if for_backward else None
        for kw, msg in cases:
            args, _cams = _forward_args(**kw, image=image, for_backward=for_backward)
            assert lib.srf_scenes_forward(*args) != 0
            assert lib.srf_last_error().decode() == f"srf_scenes_forward: {msg}", (kw, for_backward)
    args, _cams = _forward_args(P=0, tile=x, capacity=64, entries=x, plist=x, out=x, image=None, for_backward=1)
    assert lib.srf_scenes_forward(*args) != 0
    assert lib.srf_last_error() == b"srf_scenes_forward: null required pointer"

    # stage 2 alone: a misaligned geom_state or point_list is rejected; image_state may be NULL when forward-only
    cams = (ctypes.c_float * 24)()
    for for_backward in (0, 1):
        image = x if for_backward else None
        render = [None, 1, 4, 16, 16, 64, x + 16, x, x, x, image, ctypes.addressof(cams), x, x, for_backward]
        assert lib.srf_views_forward_render(*render) != 0
        assert lib.srf_last_error() == b"srf_views_forward_render: geom_state must be 256-byte aligned"
        render[6], render[9] = x, x + 4
        assert lib.srf_views_forward_render(*render) != 0
        assert lib.srf_last_error() == b"srf_views_forward_render: entries and point_list must be 256-byte aligned"
        render[1] = 0
        assert lib.srf_views_forward_render(*render) != 0
        assert lib.srf_last_error() == b"srf_views_forward_render: bad sizes"
        render[1], render[2], render[10], render[11] = 1, 0, None, None
        assert lib.srf_views_forward_render(*render) != 0
        assert lib.srf_last_error() == b"srf_views_forward_render: null required pointer"


# ---------------------------------------------------------------------------------------------- selection rule

P, H, W = 5, 4, 6


def _settings():
    return R.GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=0.5, tanfovy=0.5, bg=torch.zeros(3), scale_modifier=1.0,
        viewmatrix=torch.eye(4), projmatrix=torch.eye(4), sh_degree=0, campos=torch.zeros(3), prefiltered=False,
        debug=False)


def _fake_outputs(V, for_backward, single):
    lead = () if single else (V,)
    color = torch.arange(V * 3 * H * W, dtype=torch.float32).reshape(lead + (3, H, W)) / 100.0
    allmap = torch.full(lead + (8, H, W), 0.25)
    radii = torch.arange(V * P, dtype=torch.int32).reshape(lead + (P,))
    blob = torch.zeros(16, dtype=torch.uint8)
    state = R.ForwardState(blob, blob, blob if for_backward else None, blob if for_backward else None, 0, 0,
                           nviews=V, for_backward=for_backward)
    return color, allmap, radii, state


@pytest.fixture
def stand_ins(monkeypatch):
    """forward_raw / forward_batch_raw record which path was asked for; the CUDA-only input checks pass CPU tensors."""
    calls = []

    def forward_raw(*a, raw_activations=False, for_backward=True):
        calls.append(("forward_raw", for_backward, raw_activations))
        return _fake_outputs(1, for_backward, True)

    def forward_batch_raw(*a, raw_activations=False, for_backward=True, **kw):
        V = int(a[7].shape[0])
        calls.append(("forward_batch_raw", for_backward, raw_activations))
        return _fake_outputs(V, for_backward, False)

    monkeypatch.setattr(R, "forward_raw", forward_raw)
    monkeypatch.setattr(R, "forward_batch_raw", forward_batch_raw)
    monkeypatch.setattr(R, "_f32c", lambda t, name: t.contiguous())
    monkeypatch.setattr(R, "_check_settings", lambda rs, device: rs)
    return calls


def _inputs(requires=()):
    g = torch.Generator().manual_seed(0)
    t = {"means3D": torch.randn((P, 3), generator=g), "means2D": torch.zeros((P, 3)),
         "shs": torch.randn((P, 1, 3), generator=g), "opacities": torch.rand((P, 1), generator=g),
         "scales": torch.rand((P, 2), generator=g), "rotations": torch.randn((P, 4), generator=g)}
    for k in requires:
        t[k].requires_grad_(True)
    return t


ALL = ("means3D", "means2D", "shs", "opacities", "scales", "rotations")
MATRIX = [  # (grad mode, inputs requiring grad, training path expected)
    ("grad", ALL, True),
    ("grad", ("means2D",), True),
    ("grad", ("opacities",), True),
    ("grad", (), False),
    ("no_grad", ALL, False),
    ("no_grad", (), False),
    ("inference_mode", ALL, False),
]


def _mode(name):
    return {"grad": torch.enable_grad, "no_grad": torch.no_grad, "inference_mode": torch.inference_mode}[name]()


@pytest.mark.parametrize("mode,requires,training", MATRIX)
@pytest.mark.parametrize("entry", ["rasterize_gaussians", "rasterize_gaussians_raw", "module", "module_raw"])
def test_dropin_selection_rule(stand_ins, entry, mode, requires, training):
    t = _inputs(requires)
    rs = _settings()
    with _mode(mode):
        if entry == "rasterize_gaussians":
            out = R.rasterize_gaussians(t["means3D"], t["means2D"], t["shs"], None, t["opacities"], t["scales"],
                                        t["rotations"], None, rs)
        elif entry == "rasterize_gaussians_raw":
            out = R.rasterize_gaussians_raw(t["means3D"], t["means2D"], t["shs"], None, t["opacities"], t["scales"],
                                            t["rotations"], None, rs)
        elif entry == "module":
            out = R.GaussianRasterizer(rs)(means3D=t["means3D"], means2D=t["means2D"], shs=t["shs"],
                                           opacities=t["opacities"], scales=t["scales"], rotations=t["rotations"])
        else:
            out = R.GaussianRasterizer(rs).forward_raw_activations(t["means3D"], t["means2D"], t["opacities"],
                                                                   t["scales"], t["rotations"], shs=t["shs"])
    assert stand_ins == [("forward_raw", training, entry.endswith("raw"))]
    color, radii, allmap = out
    ref_c, ref_a, ref_r, _ = _fake_outputs(1, True, True)
    assert torch.equal(color.detach(), ref_c) and torch.equal(allmap.detach(), ref_a) and torch.equal(radii, ref_r)
    assert radii.dtype == torch.int32 and not radii.requires_grad
    assert color.requires_grad == training and (color.grad_fn is not None) == training


@pytest.mark.parametrize("mode,requires,training", [m for m in MATRIX if "means2D" not in m[1] or len(m[1]) > 1])
def test_scene_views_selection_rule_on_the_scene_body(stand_ins, mode, requires, training):
    t = _inputs(requires)
    V = 3
    sets = [_settings() for _ in range(V)]
    with _mode(mode):
        out = MV.render_scene_views(t["means3D"], t["shs"], t["opacities"], t["scales"], t["rotations"], sets,
                                    raw_activations=True)
    assert stand_ins == [("forward_batch_raw", training, True)]
    ref_c, _, ref_r, _ = _fake_outputs(V, True, False)
    assert torch.equal(out["image"].detach(), ref_c.clamp(0, 1)) and torch.equal(out["radii"], ref_r)
    assert out["image"].requires_grad == training


def test_scene_views_rays_requiring_grad_keep_the_training_path_on_the_scene_body(stand_ins, monkeypatch):
    """rays get no gradient, but a call whose only grad-requiring input is rays built an autograd node before; it
    still does."""
    monkeypatch.setattr(MV, "epilogue_views_forward_raw", lambda *a: None)
    t = _inputs()
    rays = torch.zeros((1, H, W, 6), requires_grad=True)
    out = MV.render_scene_views(t["means3D"], t["shs"], t["opacities"], t["scales"], t["rotations"], [_settings()],
                                rays=rays)
    assert stand_ins == [("forward_batch_raw", True, False)]
    assert out["image"].requires_grad


def test_backward_of_a_forward_only_state_raises():
    t = _inputs()
    st = R.ForwardState(None, None, None, None, 0, 0, nviews=1, for_backward=False)
    grad = torch.zeros((3, H, W)), torch.zeros((8, H, W))
    with pytest.raises(RuntimeError, match="forward-only"):
        R.backward_raw(st, torch.zeros(P, dtype=torch.int32), t["means3D"], t["shs"], None, t["scales"], t["rotations"],
                       None, _settings(), *grad)
    with pytest.raises(RuntimeError, match="for_backward=True"):
        R.backward_views_raw(st, torch.zeros((1, P), dtype=torch.int32), t["means3D"], t["shs"], None, t["scales"],
                             t["rotations"], None, torch.zeros((1, 24)), 0.5, 0.5, H, W, 0, *grad)


def test_empty_forward_only_keeps_no_backward_state(monkeypatch):
    """P = 0 returns before any CUDA call: zero outputs, and a state without image state or point list."""
    monkeypatch.setattr(R, "_dev_index", lambda device: 0)
    monkeypatch.setattr(R, "_capacity_hwm", {})
    e = torch.empty((0, 3))
    color, allmap, radii, st = R.forward_raw(e, torch.empty((0, 1, 3)), None, torch.empty((0, 1)), torch.empty((0, 2)),
                                             torch.empty((0, 4)), None, _settings(), for_backward=False)
    assert color.shape == (3, H, W) and allmap.shape == (8, H, W) and radii.shape == (0,)
    assert not color.any() and not allmap.any()
    assert st.image is None and st.point_list is None and not st.for_backward and st.num_rendered == 0
    _, _, _, st_train = R.forward_raw(e, torch.empty((0, 1, 3)), None, torch.empty((0, 1)), torch.empty((0, 2)),
                                      torch.empty((0, 4)), None, _settings())
    assert st_train.for_backward and st_train.image is not None and st_train.geom.numel() == st.geom.numel()
