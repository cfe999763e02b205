"""Per-scene refinement on an H100: the Adam kernel against torch.optim.Adam(foreach=False) bit for bit, the refinement
loop against the same loop on torch.optim.Adam, determinism, isolation from the novel views, its effect on a perturbed
scene, the refined tuple's structure and the caller's grad modes."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from lara_b200 import finetune as F
from lara_b200.evaluate import novel_view_metrics, render_video_frames
from lara_b200.loss import scene_loss
from lara_b200.mesh import MeshExtractor
from lara_b200.renderer import Renderer
from lara_b200.scene import PathCamera, cameras, mesh_path

pytestmark = pytest.mark.gpu

LRS = dict(position_lr=0.000016, feature_lr=0.0025, opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001)


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _mismatch(a, b):
    """(elements whose bits differ, max |a - b| / max |b|)."""
    n = int((_bits(a) != _bits(b)).sum())
    m = float(b.detach().abs().max()) if b.numel() else 0.0
    return n, (float((a.detach() - b.detach()).abs().max()) / (m or 1.0)) if b.numel() else 0.0


def _torch_adam(leaves6, lrs):
    return torch.optim.Adam([{"params": [t], "lr": lr, "name": k} for t, lr, k in zip(leaves6, lrs, F.GROUPS)],
                            betas=(0.9, 0.999), eps=1e-15, foreach=False, fused=False)


def _adam_pair(n, M, dev, seed, lrs):
    g = torch.Generator().manual_seed(seed)
    shapes = [(n, 3), (n, M, 3), (n, 1), (n, 2), (n, 4)]
    init = [torch.randn(s, generator=g).to(dev) for s in shapes]
    mine = [t.clone().requires_grad_(True) for t in init]
    ref = [init[0].clone(), init[1][:, :1].clone(), init[1][:, 1:].clone()] + [t.clone() for t in init[2:]]
    for t in ref:
        t.requires_grad_(True)
    opt = F.GaussianAdam(*mine, *lrs)
    topt = _torch_adam(ref, F.group_lrs(*lrs))
    return g, shapes, mine, ref, opt, topt


def _run_adam(n, M, dev, seed, lrs, steps=20):
    g, shapes, mine, ref, opt, topt = _adam_pair(n, M, dev, seed, lrs)
    for step in range(steps):
        # magnitudes from 1e-8 to 1e2 so that the moments' and the denominator's roundings all matter
        grads = [(torch.randn(s, generator=g) * torch.exp(torch.randn(s, generator=g) * 4)).to(dev) for s in shapes]
        for t, gt in zip(mine, grads):
            t.grad = gt.clone()
        for t, gt in zip(ref, (grads[0], grads[1][:, :1], grads[1][:, 1:], *grads[2:])):
            t.grad = gt.clone()
        opt.step()
        topt.step()
        for t in mine:
            assert int(torch.count_nonzero(t.grad)) == 0          # zero_grads
    return mine, ref, opt, topt


def _cat_ref(ref, key=None, topt=None):
    ts = ref if key is None else [topt.state[t][key] for t in ref]
    return [ts[0], torch.cat(ts[1:3], 1), *ts[3:]]


@pytest.mark.parametrize("M", [1, 4, 9, 16])
@pytest.mark.parametrize("n", [0, 1, 1000, 131073])
def test_adam_kernel_matches_torch_adam_bit_for_bit(cuda_device, n, M):
    lrs = tuple(LRS.values())
    mine, ref, opt, topt = _run_adam(n, M, cuda_device, 10 * n + M, lrs)
    report = {}
    for what, a_list, b_list in (("param", mine, _cat_ref(ref)),
                                 ("exp_avg", opt.exp_avg(), _cat_ref(ref, "exp_avg", topt) if n else None),
                                 ("exp_avg_sq", opt.exp_avg_sq(), _cat_ref(ref, "exp_avg_sq", topt) if n else None)):
        if b_list is None:
            continue
        for name, a, b in zip(("centers", "shs", "opacity", "scaling", "rotation"), a_list, b_list):
            report[f"{what}.{name}"] = _mismatch(a, b)
    bad = {k: v for k, v in report.items() if v[0]}
    print(f"\nn={n} M={M}: mismatching elements (count, rel) {bad or 'none'}")
    assert not bad
    if n == 0:
        assert opt.moments.numel() == 0 and opt.step_count == 20


def test_adam_kernel_is_repeatable_and_a_zero_lr_group_stays(cuda_device):
    lrs = (0.0, 0.0025, 0.0, 0.005, 0.001)                     # position_lr = opacity_lr = 0
    runs = [_run_adam(4097, 16, cuda_device, 5, lrs) for _ in range(2)]
    for a, b in zip(runs[0][0], runs[1][0]):
        assert torch.equal(_bits(a), _bits(b))
    assert torch.equal(_bits(runs[0][2].moments), _bits(runs[1][2].moments))
    g = torch.Generator().manual_seed(5)
    init = [torch.randn(s, generator=g) for s in [(4097, 3), (4097, 16, 3), (4097, 1)]]
    assert torch.equal(_bits(runs[0][0][0]), _bits(init[0]))
    assert torch.equal(_bits(runs[0][0][2]), _bits(init[2]))
    assert not torch.equal(_bits(runs[0][0][1]), _bits(init[1]))


# ---- the refinement loop ------------------------------------------------------------------------------------------

def _surface_scene(P, seed, M=4):
    """P surfels tangent to a sphere of radius 0.3: raw (pre-activation) parameters, as LaRa's fine tuple holds them."""
    g = torch.Generator().manual_seed(seed)
    nrm = torch.nn.functional.normalize(torch.randn((P, 3), generator=g), dim=-1)
    centers = 0.3 * nrm
    q = torch.stack((1 + nrm[:, 2], -nrm[:, 1], nrm[:, 0], torch.zeros(P)), -1)     # rotates +z onto the normal
    rotation = torch.nn.functional.normalize(q, dim=-1)
    scaling = torch.full((P, 2), math.log(0.008)) + 0.2 * torch.randn((P, 2), generator=g)
    opacity = torch.full((P, 1), 2.0) + 0.3 * torch.randn((P, 1), generator=g)
    shs = 0.5 * torch.randn((P, M, 3), generator=g)
    shs[:, 1:] *= 0.2
    return centers, shs, opacity, scaling, rotation


def _sample(views, H, W, dev, seed=0, fov=0.75):
    """A LaRa-style sample of one scene with views[0] .. as its target views (tar_rgb filled in by _case)."""
    cams = cameras(max(views) + 1, H, W, seed, fov=fov)
    c2w = torch.stack([cams[v].c2w for v in views])
    V = len(views)
    s = {"tar_c2w": c2w[None].to(dev), "fovx": torch.tensor([fov]).to(dev), "fovy": torch.tensor([fov]).to(dev),
         "near_far": torch.tensor([[0.5, 2.5]]).to(dev), "bg_color": torch.ones((1, V, 3)).to(dev),
         "tar_rgb": torch.zeros((1, V, H, W, 3)).to(dev)}
    pcs = [PathCamera(c2w[j], H, W, fov) for j in range(V)]
    s["tar_rays"] = torch.stack([c.get_rays()[0] for c in pcs])[None].to(dev)
    return s


def _render_all(renderer, gs, sample):
    c, s, o, sc, r, mask = gs
    V = sample["tar_rgb"].shape[1]
    with torch.no_grad():
        return renderer.render_views(F.sample_cameras(sample, range(V)), sample["tar_rays"][0], c, s, o[mask],
                                     sc[mask], r[mask], c.device, bg_colors=sample["bg_color"][0])


def _case(dev, P=32768, H=256, perturb=1.0, seed=0, extra=512):
    """Ground truth rendered at 4 source and 4 novel views, and LaRa's fine tuple of a perturbed copy with
    ``extra`` masked-out rows."""
    renderer = Renderer(sh_degree=1)
    views = [0, 2, 4, 6, 1, 3, 5, 7]                                # sources spread around the object, then the novel
    sample = _sample(views, H, H, dev, seed)
    gt = [t.to(dev) for t in _surface_scene(P, seed)]
    mask_all = torch.ones(P, dtype=torch.bool, device=dev)
    out = _render_all(renderer, (*gt, mask_all), sample)
    sample["tar_rgb"] = out["image"].contiguous()[None]
    g = torch.Generator().manual_seed(100 + seed)
    noise = [0.001, 0.3, 1.0, 0.3, 0.05]
    pert = [t.cpu() + perturb * k * torch.randn(t.shape, generator=g) for t, k in zip(gt, noise)]
    pert[1][:, 1:] = gt[1][:, 1:].cpu()                           # f_rest moves at feature_lr / 20: perturb f_dc only
    # full-size opacity / scaling / rotation with `extra` rows the mask leaves out, spread through the tensors
    Pf = P + extra
    mask = torch.ones(Pf, dtype=torch.bool)
    mask[torch.randperm(Pf, generator=g)[:extra]] = False
    full = []
    for t in pert[2:]:
        f = torch.randn((Pf, t.shape[1]), generator=g)
        f[mask] = t
        full.append(f.to(dev))
    gs = (pert[0].to(dev), pert[1].to(dev).contiguous(), *full, mask.to(dev))
    return renderer, sample, gs


def _torch_finetune(renderer, gs, sample, n_views, steps, lrs):
    """The same loop on torch.optim.Adam over get_params' six leaves, f_dc and f_rest concatenated each step."""
    c, s, o, sc, r, mask = gs
    leaves = [c.clone(), s[:, :1].clone(), s[:, 1:].clone(), o[mask].clone(), sc[mask].clone(), r[mask].clone()]
    for t in leaves:
        t.requires_grad_(True)
    opt = _torch_adam(leaves, F.group_lrs(*lrs))
    cams = F.sample_cameras(sample, range(n_views))
    rays, tar, bg = (sample[k][0, :n_views] for k in ("tar_rays", "tar_rgb", "bg_color"))
    losses = []
    for _ in range(steps):
        out = renderer.render_views(cams, rays, leaves[0], torch.cat(leaves[1:3], 1), *leaves[3:], c.device,
                                    bg_colors=bg)
        loss, _ = scene_loss(out, tar, 1001, batch_scenes=1, ms_ssim=True)
        loss.backward()
        losses.append(loss.detach())
        opt.step()
        opt.zero_grad()
    return [leaves[0], torch.cat(leaves[1:3], 1), *leaves[3:]], torch.stack(losses)


@pytest.fixture
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def _refined_tensors(gs):
    c, s, o, sc, r, mask = gs
    return [c, s, o[mask], sc[mask], r[mask]]


def test_loop_matches_torch_adam_loop(cuda_device, deterministic):
    renderer, sample, gs = _case(cuda_device, P=16384, H=192)
    lrs = tuple(LRS.values())
    ref, ref_losses = _torch_finetune(renderer, gs, sample, 4, 20, lrs)
    out, losses = F.finetune_scene(renderer, gs, sample, 4, 20, **LRS)
    worst = {}
    for name, a, b in zip(("centers", "shs", "opacity", "scaling", "rotation"), _refined_tensors(out), ref):
        worst[name] = _mismatch(a, b)
    worst["losses"] = _mismatch(losses, ref_losses)
    print(f"\nloop vs torch.optim.Adam loop, 20 steps: (differing elements, max |diff| / max |ref|) {worst}")
    assert all(v[0] == 0 for v in worst.values())


def test_loop_is_deterministic_and_ignores_the_novel_views(cuda_device, deterministic):
    renderer, sample, gs = _case(cuda_device, P=16384, H=192)
    a, la = F.finetune_scene(renderer, gs, sample, 4, 10, **LRS)
    b, lb = F.finetune_scene(renderer, gs, sample, 4, 10, **LRS)
    poisoned = dict(sample)
    for k in ("tar_rgb", "tar_rays"):
        t = sample[k].clone()
        t[0, 4:] = float("nan")
        poisoned[k] = t
    c, lc = F.finetune_scene(renderer, gs, poisoned, 4, 10, **LRS)
    for x, y, z in zip(a[:5] + (la,), b[:5] + (lb,), c[:5] + (lc,)):
        assert torch.equal(_bits(x), _bits(y)) and torch.equal(_bits(x), _bits(z))
    assert torch.equal(a[5], gs[5])


def test_refinement_recovers_a_perturbed_scene(cuda_device):
    renderer, sample, gs = _case(cuda_device)
    before = novel_view_metrics(_render_all(renderer, gs, sample), sample, 4, image_key="image")
    out, losses = F.finetune_scene(renderer, gs, sample, 4, 200, **LRS)
    after = novel_view_metrics(_render_all(renderer, out, sample), sample, 4, image_key="image")
    l = losses.cpu().numpy()
    print(f"\nsource-view loss {l[0]:.5f} -> {l[-1]:.5f}; novel-view PSNR {before['psnr']:.2f} -> {after['psnr']:.2f} dB, "
          f"SSIM {before['ssim']:.4f} -> {after['ssim']:.4f}")
    assert np.isfinite(l).all() and l[-1] < 0.5 * l[0]
    assert after["psnr"] > before["psnr"]


def test_refined_tuple_keeps_structure_and_feeds_video_and_mesh(cuda_device):
    renderer, sample, gs = _case(cuda_device, P=8192, H=192)
    out, losses = F.finetune_scene(renderer, gs, sample, 4, 5, **LRS)
    assert len(out) == 6 and losses.shape == (5,) and losses.device == gs[0].device
    mask = gs[5]
    for a, b in zip(out[:5], gs[:5]):
        assert a.shape == b.shape and a.dtype == b.dtype and not a.requires_grad
    for k in (2, 3, 4):
        assert torch.equal(_bits(out[k][~mask]), _bits(gs[k][~mask]))
        assert not torch.equal(_bits(out[k][mask]), _bits(gs[k][mask]))
    cams = mesh_path(n=4, H=64, W=64)
    rgb, nrm = render_video_frames(renderer, out, cams[:4], device=cuda_device)
    assert rgb.shape == (4, 64, 64, 3) and nrm.shape == (4, 64, 64, 3)
    v, t, c = MeshExtractor(out, renderer, aabb=[-0.5, -0.5, -0.5, 0.5, 0.5, 0.5]).extract(None, cams,
                                                                                           device=cuda_device)
    assert v.shape[0] > 0 and t.shape[0] > 0


def test_runs_under_no_grad_and_inference_mode(cuda_device, deterministic):
    renderer, sample, gs = _case(cuda_device, P=8192, H=192)
    bg = renderer.bg_color
    ref, lref = F.finetune_scene(renderer, gs, sample, 4, 5, **LRS)
    assert renderer.bg_color is bg
    with torch.no_grad():
        a, la = F.finetune_scene(renderer, gs, sample, 4, 5, **LRS)
    with torch.inference_mode():
        inf_gs = tuple(t.clone() for t in gs)
        inf_sample = {k: v.clone() for k, v in sample.items()}
        b, lb = F.finetune_scene(renderer, inf_gs, inf_sample, 4, 5, **LRS)
    for x, y, z in zip(ref[:5] + (lref,), a[:5] + (la,), b[:5] + (lb,)):
        assert torch.equal(_bits(x), _bits(y)) and torch.equal(_bits(x), _bits(z))
