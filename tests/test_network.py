"""LaRa's ``Network`` on the fused path (lara_b200.network, DESIGN §3.28), the parts that run without a GPU:

* the state dict (keys in order, shapes, dtypes) equals LaRa's for the base config and a small one, the four buffers
  hold LaRa's values, and LaRa's optimizer partition (``system.configure_optimizers``: LayerNorm parameters and
  biases without weight decay) gives the same names in each group.  LaRa's side is recorded in
  tests/golden/reference/test_network.npz by ``record_reference`` (LaRa's ``Network`` imported with
  ``_import_reference_network``'s stubs, ``timm.create_model`` returning this package's ``VisionTransformer``):

      python tests/test_network.py OUT_DIR LARA_CHECKOUT && cp OUT_DIR/test_network.npz tests/golden/reference/

* a synthetic ``net.*`` checkpoint loads strictly through ``from_lara_state_dict``, each LaRa tensor one parameter;
* ``n_views_sel`` takes LaRa's ``random.randint(2, 4)`` draw under the same conditions;
* a float64 restatement of ``srf_batch_cameras``' record equals LaRa's ``MiniCam`` on the CPU within fp32 rounding;
* the argument checks of ``batch_cameras``, ``srf_batch_cameras`` (before any launch) and ``Network.forward``.

The GPU side is tests/test_gpu_network.py.
"""
import ctypes
import os
import random
import sys
import types

import numpy as np
import pytest
import torch
from torch import nn

from helpers import fingerprint, reference_record

MODULE = "test_network"
BUFFERS = ("dense_grid", "centers", "volume_grid", "group_centers")


def lara_cfg(small: bool = False, use_rand_views: bool = False, n_views: int = 4):
    """LaRa's configs/base.yaml model section, or a small one (ViT-S, no view embedding, sh_degree 0, K = 1)."""
    model = dict(encoder_backbone="vit_base_patch16_224.dino", n_groups=[16], n_offset_groups=32, K=2, sh_degree=1,
                 num_layers=12, num_heads=16, view_embed_dim=32, embedding_dim=256, vol_feat_reso=16,
                 vol_embedding_reso=32, vol_embedding_out_dim=80)
    if small:
        model.update(encoder_backbone="vit_small_patch16_224.dino", n_groups=[2, 4], n_offset_groups=8, K=1,
                     sh_degree=0, num_layers=2, num_heads=2, view_embed_dim=0, embedding_dim=32, vol_feat_reso=8,
                     vol_embedding_reso=8, vol_embedding_out_dim=32)
    return types.SimpleNamespace(model=types.SimpleNamespace(**model), n_views=n_views,
                                 train=types.SimpleNamespace(use_rand_views=use_rand_views))


CONFIGS = {"base": dict(), "small": dict(small=True)}


def partition(module: nn.Module):
    """LaRa's ``configure_optimizers`` grouping (lightning/system.py): every parameter of a LayerNorm and every
    module's non-None ``bias`` go without weight decay, the rest with it; the names of each group, sorted."""
    no_decay = []
    for _, m in module.named_modules():
        if isinstance(m, nn.LayerNorm):
            no_decay.extend(m.parameters())
        elif getattr(m, "bias", None) is not None:
            no_decay.append(m.bias)
    ids = set(map(id, no_decay))
    names = {id(p): n for n, p in module.named_parameters()}
    decay = sorted(n for n, p in module.named_parameters() if id(p) not in ids and p.requires_grad)
    return decay, sorted(names[id(p)] for p in no_decay if p.requires_grad)


def _describe(sd):
    return "\n".join(f"{k} {tuple(v.shape)} {v.dtype}" for k, v in sd.items())


def _record(net):
    sd = net.state_dict()
    decay, no_decay = partition(net)
    rec = {"state_dict": _describe(sd), "decay": "\n".join(decay), "no_decay": "\n".join(no_decay)}
    rec.update({b: fingerprint(sd[b].numpy()) for b in BUFFERS})
    return rec


def record_reference(lara, dev="cpu"):
    """LaRa's Network built for each config, with timm's ViT replaced by this package's (the same parameter names);
    the grouping is also taken from LaRa's own configure_optimizers and must equal ``partition``'s."""
    from test_decoder_layout import _import_reference_network
    from lara_b200.image_encoder import MODELS, VisionTransformer
    net = _import_reference_network(lara)
    net.timm.create_model = lambda name, **kw: VisionTransformer(*MODELS[name])
    net.timm.data = types.SimpleNamespace(resolve_model_data_config=lambda m: {"mean": (0.485, 0.456, 0.406),
                                                                              "std": (0.229, 0.224, 0.225)})
    net.transforms.Normalize = lambda mean, std: nn.Identity()
    net.Network.device = property(lambda self: torch.device("cpu"))
    out = {}
    for name, kw in CONFIGS.items():
        torch.manual_seed(0)
        lara_net = net.Network(lara_cfg(**kw))
        out[name] = _record(lara_net)
        assert (out[name]["decay"], out[name]["no_decay"]) == _lara_groups(lara, lara_net), name
    return out


def _lara_groups(lara, lara_net):
    """The two groups LaRa's ``system.configure_optimizers`` hands to AdamW, by name (without the ``net.`` prefix)."""
    stubs = {"pytorch_msssim": dict(MS_SSIM=lambda **kw: nn.Identity()),
             "pytorch_lightning": dict(LightningModule=nn.Module),
             "pytorch_lightning.loggers": dict(TensorBoardLogger=object), "timm": {}, "torchvision": {},
             "torchvision.transforms": {}, "lightning.vis": dict(vis_images=None)}
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.path.insert(0, lara)
    try:
        import importlib
        for k in [k for k in sys.modules if k == "lightning" or k.startswith("lightning.")]:
            del sys.modules[k]
        for k, attrs in stubs.items():
            sys.modules[k] = types.ModuleType(k)
            sys.modules[k].__dict__.update(attrs)
        system = importlib.import_module("lightning.system")
    finally:
        sys.path.remove(lara)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    captured = {}

    def adamw(groups, **kw):
        captured["groups"] = groups
    system.torch = types.SimpleNamespace(optim=types.SimpleNamespace(AdamW=adamw))
    system.CosineWarmupScheduler = lambda **kw: None
    holder = nn.Module()
    holder.net = lara_net
    holder.cfg = types.SimpleNamespace(train=types.SimpleNamespace(weight_decay=0.05, lr=4e-4, beta1=0.9, beta2=0.95,
                                                                    warmup_iters=1000))
    holder.num_steps = lambda: 1
    system.system.configure_optimizers(holder)
    names = {id(p): n[len("net."):] for n, p in holder.named_parameters()}
    decay, no_decay = captured["groups"]
    return ("\n".join(sorted(names[id(p)] for p in decay["params"])),
            "\n".join(sorted(names[id(p)] for p in no_decay["params"])))


@pytest.fixture(scope="module", params=list(CONFIGS))
def built(request):
    from lara_b200.network import Network
    torch.manual_seed(0)
    return request.param, Network(lara_cfg(**CONFIGS[request.param]))


def test_state_dict_is_laras(built):
    name, net = built
    ref = reference_record(MODULE, name)
    assert _describe(net.state_dict()).splitlines() == ref["state_dict"].splitlines()
    for b in BUFFERS:
        assert fingerprint(getattr(net, b).numpy()) == ref[b], b


def test_optimizer_groups_are_laras(built):
    name, net = built
    ref = reference_record(MODULE, name)
    decay, no_decay = partition(net)
    assert decay == ref["decay"].splitlines()
    assert no_decay == ref["no_decay"].splitlines()


def test_each_lara_tensor_is_one_parameter(built):
    """The stage ops run on the network's own modules: no duplicate and no hidden parameter."""
    _, net = built
    stages = net._stages
    own = {id(p) for p in net.parameters()}
    assert len(own) == len(list(net.parameters())) == len(dict(net.named_parameters()))
    for st in stages.values():
        assert {id(p) for p in st.parameters()} <= own
    fv = net._feat_volume()
    assert fv.dir_norm is net.dir_norm and fv.volume_grid is net.volume_grid
    assert stages["coarse"].mlp_coarse is net.decoder.mlp_coarse
    assert stages["fine"].cross_att is net.decoder.cross_att and stages["fine"].norm is net.decoder.norm


def test_from_lara_state_dict_is_strict(built):
    from lara_b200.network import Network
    name, net = built
    g = torch.Generator().manual_seed(5)
    sd = {"net." + k: torch.rand(v.shape, generator=g).to(v.dtype) for k, v in net.state_dict().items()}
    sd["loss.some_buffer"] = torch.zeros(1)          # other entries of LaRa's system are not the network's
    cfg = lara_cfg(**CONFIGS[name])
    loaded = Network.from_lara_state_dict(sd, cfg)
    for k, v in loaded.state_dict().items():
        assert torch.equal(v, sd["net." + k]), k
    fv = loaded._feat_volume()
    assert torch.equal(fv.dir_norm.norm.weight, sd["net.dir_norm.norm.weight"])
    assert torch.equal(loaded._stages["coarse"].mlp_coarse[0].weight, sd["net.decoder.mlp_coarse.0.weight"])
    assert torch.equal(loaded._stages["fine"].mlp_fine[2].bias, sd["net.decoder.mlp_fine.2.bias"])
    missing = dict(sd)
    missing.pop("net.decoder.mlp_fine.2.bias")
    with pytest.raises(RuntimeError, match="Missing key"):
        Network.from_lara_state_dict(missing, cfg)
    extra = dict(sd, **{"net.decoder.extra": torch.zeros(1)})
    with pytest.raises(RuntimeError, match="Unexpected key"):
        Network.from_lara_state_dict(extra, cfg)


def _lara_n_views_sel(training, cfg):
    """network.py:434-437."""
    if training:
        return random.randint(2, 4) if cfg.train.use_rand_views else cfg.n_views
    return cfg.n_views


@pytest.mark.parametrize("training,rand_views", [(True, True), (True, False), (False, True)])
def test_n_views_sel_draws_as_lara(training, rand_views):
    from lara_b200.network import Network
    cfg = lara_cfg(small=True, use_rand_views=rand_views, n_views=3)
    net = Network(cfg).train(training)
    random.seed(17)
    mine = [net.n_views_sel() for _ in range(32)]
    after = random.random()
    random.seed(17)
    lara = [_lara_n_views_sel(training, cfg) for _ in range(32)]
    assert mine == lara and after == random.random()
    if training and rand_views:
        assert set(mine) == {2, 3, 4}


# ---- camera records -------------------------------------------------------------------------------------------------
def camera_record64(c2w: np.ndarray, bg: np.ndarray) -> np.ndarray:
    """srf_batch_cameras' record restated in float64: inverse(c2w)^T rounded once to fp32, -c2w[:3,3], bg, zeros."""
    c2w = np.asarray(c2w, dtype=np.float32).reshape(-1, 4, 4)
    n = c2w.shape[0]
    rec = np.zeros((n, 24), dtype=np.float32)
    inv = np.linalg.inv(c2w.astype(np.float64))
    rec[:, :16] = inv.transpose(0, 2, 1).reshape(n, 16).astype(np.float32)
    rec[:, 16:19] = -c2w[:, :3, 3]
    rec[:, 19:22] = np.asarray(bg, dtype=np.float32).reshape(n, 3)
    return rec


def exact_view_f32(c2w: np.ndarray) -> np.ndarray:
    """inverse(c2w)^T [n,16] computed exactly (rationals) from the fp32 poses and rounded once to fp32."""
    from fractions import Fraction
    out = []
    for m in np.asarray(c2w, dtype=np.float32).reshape(-1, 4, 4):
        a = [[Fraction(float(x)) for x in row] + [Fraction(int(i == j)) for j in range(4)] for i, row in enumerate(m)]
        for c in range(4):
            p = next(r for r in range(c, 4) if a[r][c] != 0)
            a[c], a[p] = a[p], a[c]
            a[c] = [x / a[c][c] for x in a[c]]
            for r in range(4):
                if r != c and a[r][c] != 0:
                    a[r] = [x - a[r][c] * y for x, y in zip(a[r], a[c])]
        inv = np.array([[float(a[i][4 + j]) for j in range(4)] for i in range(4)])    # nearest double of each
        out.append(inv.T.reshape(16))
    # nearest double, then fp32: a double rounding, which can differ from the direct one only at an exact fp32 tie
    return np.stack(out).astype(np.float32)


def poses(n, seed, rigid=True):
    """c2w poses looking at the origin from radius ~2, or with a scaled, sheared (non-rigid) rotation part."""
    from lara_b200.scene import look_at_c2w
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        c2w = look_at_c2w(float(rng.uniform(0, 2 * np.pi)), float(rng.uniform(-0.5, 0.5)),
                          float(rng.uniform(1.5, 2.5))).numpy()
        if not rigid:
            c2w[:3, :3] = c2w[:3, :3] @ (np.diag(rng.uniform(0.5, 2.0, 3)) + rng.uniform(-0.2, 0.2, (3, 3)))
        out.append(c2w)
    return np.stack(out).astype(np.float32)


def _minicam(c2w, bg):
    """The record pack_cameras builds from LaRa's MiniCam (lightning/utils.py:33-48) on the CPU."""
    c = torch.from_numpy(c2w)
    view = torch.inverse(c).transpose(0, 1)
    return torch.cat([view.reshape(16), -c[:3, 3], torch.from_numpy(bg), torch.zeros(2)]).numpy()


@pytest.mark.parametrize("rigid", [True, False])
def test_camera_record_restatement_equals_minicam(rigid):
    c2w = poses(64, 3 if rigid else 4, rigid)
    bg = np.random.default_rng(1).choice([0.0, 0.5, 1.0], (64, 3)).astype(np.float32)
    mine = camera_record64(c2w, bg)
    lara = np.stack([_minicam(c, b) for c, b in zip(c2w, bg)])
    assert np.array_equal(mine[:, 16:], lara[:, 16:])            # campos, bg and the padding: bit for bit
    view, lv = mine[:, :16].astype(np.float64), lara[:, :16].astype(np.float64)
    scale = np.abs(view).reshape(-1, 4, 4).max(axis=(1, 2), keepdims=True).repeat(16, axis=1).reshape(-1, 16)
    # torch's fp32 inverse (LU) differs from the correctly rounded one by a few ulps of the matrix's largest entry
    assert (np.abs(view - lv) <= 2.0 ** -20 * scale).all(), np.abs(view - lv).max()


def test_batch_cameras_rejects_bad_arguments():
    from lara_b200.batch import batch_cameras
    c2w, bg = torch.eye(4).expand(2, 3, 4, 4).contiguous(), torch.ones(2, 3, 3)
    with pytest.raises(TypeError, match="float32"):
        batch_cameras(c2w.double(), bg)
    with pytest.raises(TypeError, match="float32"):
        batch_cameras(c2w, bg.half())
    with pytest.raises(TypeError, match="tensor"):
        batch_cameras(c2w, [1.0, 1.0, 1.0])
    with pytest.raises(ValueError, match="tar_c2w"):
        batch_cameras(c2w[..., :3], bg)
    with pytest.raises(ValueError, match="bg_color"):
        batch_cameras(c2w, bg[:, :2])
    with pytest.raises(ValueError, match="bg_color"):
        batch_cameras(c2w, bg[..., :2])
    with pytest.raises(ValueError, match="65535"):
        batch_cameras(torch.zeros(0, 4, 4), torch.zeros(0, 3))
    with pytest.raises(ValueError, match="65535"):
        batch_cameras(torch.zeros(65536, 4, 4), torch.zeros(65536, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        batch_cameras(c2w, bg)


def test_srf_batch_cameras_rejects_bad_arguments_before_any_launch(lib):
    P = ctypes.c_void_p(256)            # never dereferenced: the checks come before any CUDA call
    for n in (0, -1, 65536):
        assert lib.srf_batch_cameras(None, n, P, P, P) != 0
        assert b"srf_batch_cameras" in lib.srf_last_error() and b"65535" in lib.srf_last_error()
    for k, what in enumerate((b"c2w", b"bg", b"cams")):
        args = [P, P, P]
        args[k] = None
        assert lib.srf_batch_cameras(None, 4, *args) != 0
        assert b"null " + what in lib.srf_last_error()
        args[k] = ctypes.c_void_p(258)
        assert lib.srf_batch_cameras(None, 4, *args) != 0
        assert b"aligned" in lib.srf_last_error()


def _small_batch(B=2, V=4, H=32, W=32):
    g = torch.Generator().manual_seed(0)
    c2w = torch.from_numpy(poses(B * V, 9)).view(B, V, 4, 4)
    return {"tar_rgb": torch.rand(B, V, H, W, 3, generator=g), "tar_c2w": c2w, "tar_w2c": torch.inverse(c2w),
            "tar_ixt": torch.eye(3).expand(B, V, 3, 3), "bg_color": torch.ones(B, V, 3),
            "tar_rays": torch.rand(B, V, H, W, 6, generator=g), "tar_rays_down": torch.rand(B, V, 2, 2, 6, generator=g),
            "fovx": torch.full((B,), 0.8), "fovy": torch.full((B,), 0.8),
            "meta": {"tar_h": torch.full((B,), H), "tar_w": torch.full((B,), W)}}


def test_forward_rejects_mismatched_render_sizes_and_too_few_views():
    from lara_b200.network import Network
    net = Network(lara_cfg(small=True, n_views=3)).eval()
    batch = _small_batch()
    batch["meta"] = {"tar_h": torch.tensor([32, 64]), "tar_w": torch.tensor([32, 32])}
    with pytest.raises(ValueError, match="share the render size"):
        net(batch)
    batch = _small_batch(V=2)
    with pytest.raises(ValueError, match="fewer than the 3 source views"):
        net(batch)
    assert net.render_geometry(_small_batch(), 2)[:2] == (32, 32)
    H, W, tan_fov = net.render_geometry(dict(_small_batch(), render_img_scale=0.5), 2)
    assert (H, W) == (16, 16) and tan_fov == [(np.tan(np.float32(0.8) * 0.5),) * 2] * 2


def test_concat_batch_views_is_laras_cat():
    from lara_b200.network import concat_batch_views
    g = torch.Generator().manual_seed(2)
    out = {"image": torch.rand(2, 3, 4, 5, 3, generator=g), "acc_map": torch.rand(2, 3, 4, 5, generator=g),
           "render_pkg": [], "radii": torch.zeros(2, 3, 7)}
    res = concat_batch_views(out)
    assert set(res) == {"image", "acc_map"}
    for k in res:      # network.py:527-529: per scene, torch.cat of the views along dim 1 (the width)
        lara = torch.stack([torch.cat(list(out[k][b]), dim=1) for b in range(2)])
        assert torch.equal(res[k], lara)


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_reference_records import save
    os.makedirs(sys.argv[1], exist_ok=True)
    save(sys.argv[1], MODULE, record_reference(sys.argv[2], "cpu"))
