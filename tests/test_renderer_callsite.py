"""The consumer: LaRa's lightning/renderer_2dgs.py must run unchanged on top of this package.

* GPU: the call pattern of Renderer.render_img (renderer_2dgs.py:167-268) -- activations,
  zeros+0 screenspace tensor with retain_grad, keyword call, the torch post-processing of the aux
  maps and a loss -- is replayed with this package and compared with the same replay on the reference
  build (recorded in tests/golden/reference/, see record_reference); images and the gradients wrt the
  *raw* network outputs must agree.
"""
import numpy as np
import pytest
import torch

from helpers import allmap_records, compare_records, fingerprint, reference_record, sampled_rel_err, tolerance_record


def _render_img_like(mod, cam, raw, bg, dev):
    """Replays renderer_2dgs.Renderer.render_img with module `mod` as the rasterizer package."""
    from lara_b200 import scene as S
    rs = S.settings_for(cam, bg, 1, dev, mod.GaussianRasterizationSettings)
    # MiniCam hands over w2c.transpose(0, 1): a NON-contiguous view matrix (lightning/utils.py:40)
    w2c = rs.viewmatrix.t().contiguous()
    rs = rs._replace(viewmatrix=w2c.transpose(0, 1))
    assert not rs.viewmatrix.is_contiguous()
    rast = mod.GaussianRasterizer(raster_settings=rs)
    opacity = torch.sigmoid(raw["opacity"])
    scales = torch.exp(raw["scales"])
    rotations = torch.nn.functional.normalize(raw["rotations"])
    centers = raw["centers"]
    screenspace = torch.zeros_like(centers, dtype=centers.dtype, requires_grad=True, device=dev) + 0
    screenspace.retain_grad()
    img, radii, allmap = rast(means3D=centers, means2D=screenspace, shs=raw["shs"], opacities=opacity,
                              scales=scales, rotations=rotations, cov3D_precomp=None)
    img = img.clamp(0, 1)
    alpha = allmap[1:2]
    normal = (allmap[2:5].permute(1, 2, 0) @ (rs.viewmatrix[:3, :3].T)).permute(2, 0, 1)
    # (LaRa divides by alpha and nan_to_num()s the result; with anomaly mode on, 0/0 at empty pixels
    #  would trip DivBackward itself, so the replay guards the denominator)
    depth = torch.nan_to_num(allmap[0:1] / alpha.clamp_min(1e-6), 0, 0)
    dist = allmap[6:7]
    loss = ((img - 0.3) ** 2).mean() + 0.2 * (normal ** 2).mean() + 1000.0 * dist.mean() + 0.1 * depth.mean() + alpha.mean()
    return img, allmap, radii, loss, screenspace


def _replay(mod, dev):
    from lara_b200 import scene as S
    sc = S.scene(20000, 11)
    cam = S.cameras(2, 160, 160, 3)[1]
    base = {"centers": sc["means3D"], "shs": sc["shs"], "opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)),
            "scales": torch.log(sc["scales"]), "rotations": sc["rotations"] * 1.7}
    raw = {k: v.to(dev).clone().requires_grad_(True) for k, v in base.items()}
    with torch.autograd.set_detect_anomaly(True):
        img, allmap, radii, loss, ss = _render_img_like(mod, cam, raw, torch.ones(3), dev)
        loss.backward()
    return (img.detach().cpu().numpy(), allmap.detach().cpu().numpy(), radii.cpu().numpy(),
            {k: v.grad.cpu().numpy() for k, v in raw.items()}, ss.grad.cpu().numpy(), float(loss))


def record_reference(ref, dev):
    """The reference's side of the replay (tests/golden/make_reference_records.py)."""
    img, allmap, radii, grads, ss, loss = _replay(ref, dev)
    rec = {"img": tolerance_record(img), **allmap_records(allmap), "radii": fingerprint(radii),
           "loss": tolerance_record(loss), "screenspace": tolerance_record(ss)}
    rec.update({"g_" + k: tolerance_record(v) for k, v in grads.items()})
    return {"render_img": rec}


@pytest.mark.gpu
def test_render_img_call_pattern_matches_reference(cuda_device):
    import diff_surfel_rasterization as DSR
    img, allmap, radii, grads, ss, loss = _replay(DSR, cuda_device)
    rec = reference_record("test_renderer_callsite", "render_img")
    assert not compare_records({"img": tolerance_record(img), **allmap_records(allmap), "radii": fingerprint(radii),
                                "loss": tolerance_record(loss)}, rec)
    for k in grads:
        assert np.isfinite(grads[k]).all()
        assert sampled_rel_err(grads[k], rec, "g_" + k) < 1e-4, k
    assert sampled_rel_err(ss, rec, "screenspace") < 1e-4        # viewspace (means2D) gradient used for densification statistics
