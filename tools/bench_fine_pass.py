"""LaRa's fine pass over the B scenes of a batch (DESIGN §3.26): the per-scene loop against the three batched calls.

One step renders the coarse pass of B = 3 scenes (8 target views of 512^2, P = 524288 Gaussians, SH degree 1) with
``render_batch_views(keep_binning=True)``.  Two arms then run the fine pass, forward and backward to the leaves:

* ``loop``: LaRa's per-scene loop on the fused ops, ``sample_point_feats(centers[b][mask_b], ...)`` and
  ``FineHead.fine_shs`` per scene, then ``render_batch_subset_views(binning, masks, torch.cat(shs))``;
* ``batched``: ``FineSubset(masks)``, ``sample_batch_point_feats``, the batch form of ``fine_shs`` and
  ``render_batch_subset_views(binning, subset, shs)``.

The masks are LaRa's opacity cut (scene 0), an empty scene and a full scene.  The first step checks that the arms agree
bit for bit (forward, and the gradients under ``torch.use_deterministic_algorithms(True)``).  The arms then alternate
over --repeats; each repeat times one step (coarse render + fine pass + backward) on the host clock around a device
synchronise, and the coarse render alone is timed the same way.  ``--profile`` instead records device time per arm
with ``torch.profiler`` in a run of its own, and ``--memory`` the peak-allocation increase of one step.  Prints the
card's name and power limit, then one JSON line.

    python tools/bench_fine_pass.py [--repeats 9] [--profile] [--memory]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from timing import alternate, card, host_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)

B, V, VS, H, W = 3, 8, 4, 512, 512
N, K, D, SH_DIM = 64 ** 3, 2, 80, 12
P = N * K
KEYS = tuple(k + "_fine" for k in ("image", "depth", "acc_map", "rend_normal", "depth_normal", "rend_dist"))


def setup(dev):
    from lara_b200 import rasterizer as R
    from lara_b200 import scene as S
    from lara_b200.fine_head import FineHead
    from test_chain_per_element import lara_rays
    params, settings, rays = [], [], []
    for b in range(B):
        sc = S.scene(P, 41 + 17 * b, 1)
        params.append((sc["means3D"], sc["shs"], torch.logit(sc["opacities"]), torch.log(sc["scales"]),
                       sc["rotations"] * 1.7))
        cams = S.cameras(V, H, W, 41 + b, fov=0.65 + 0.1 * b)
        bg = torch.tensor([0.2 * b, 0.5, 1.0 - 0.3 * b])
        settings.append([S.settings_for(c, bg, 1, dev, R.GaussianRasterizationSettings) for c in cams])
        rays.append(torch.stack([lara_rays(c) for c in cams]))
    params = [torch.stack([p[k] for p in params]).to(dev).contiguous() for k in range(5)]
    w2c = torch.stack([torch.stack([s.viewmatrix.T for s in sc[:VS]]) for sc in settings]).contiguous().to(dev)
    ixt = torch.zeros(B, VS, 3, 3)
    for b, sc in enumerate(settings):
        fx, fy = W / (2 * float(sc[0].tanfovx)), H / (2 * float(sc[0].tanfovy))
        ixt[b, :, 0, 0], ixt[b, :, 1, 1], ixt[b, :, 0, 2], ixt[b, :, 1, 2], ixt[b, :, 2, 2] = fx, fy, W / 2, H / 2, 1
    g = torch.Generator(device=dev).manual_seed(5)
    masks = (torch.sigmoid(params[2]) > 0.005).view(B, P)
    masks[1] = False
    masks[2] = True
    return dict(params=params, settings=settings, rays=torch.stack(rays).to(dev).contiguous(),
                tar_rgb=torch.rand(B, V, H, W, 3, generator=g, device=dev), vf=torch.randn(B, N, D, generator=g, device=dev),
                masks=masks, head=FineHead(D, SH_DIM).to(dev), w2c=w2c, ixt=ixt.to(dev),
                up={k: None for k in KEYS})


def step(d, batched, coarse_only=False):
    """Coarse render, fine pass and backward to the leaves; returns (fine outputs, leaf gradients)."""
    from lara_b200.multiview import FineSubset, render_batch_subset_views, render_batch_views
    from lara_b200.point_feats import sample_batch_point_feats, sample_point_feats
    leaves = [p.detach().requires_grad_(True) for p in d["params"]]
    vf = d["vf"].detach().requires_grad_(True)
    head = d["head"]
    head.zero_grad(set_to_none=True)
    out = render_batch_views(*leaves, d["settings"], rays=d["rays"], raw_activations=True, keep_binning=True)
    if coarse_only:
        return out, None
    img_ref = d["tar_rgb"][:, :VS].permute(0, 1, 4, 2, 3)
    if batched:
        sub = FineSubset(d["masks"])
        pf = sample_batch_point_feats(sub, leaves[0], img_ref, out, d["w2c"], d["ixt"])
        shs = head.fine_shs(vf, K, sub, pf, leaves[1])
        fine = render_batch_subset_views(out["binning"], sub, shs)
    else:
        shs_l = []
        for b in range(B):
            m = d["masks"][b]
            rend = {k: out[k][b][:VS] for k in ("image", "acc_map", "depth")}
            pf = sample_point_feats(leaves[0][b][m], img_ref[b], rend, d["w2c"][b], d["ixt"][b])
            # the one-scene head takes no empty mask (LaRa's _check_mask never leaves one)
            shs_l.append(head.fine_shs(vf[b], K, m, pf, leaves[1][b]) if m.any() else leaves[1][b][:0])
        fine = render_batch_subset_views(out["binning"], d["masks"], torch.cat(shs_l))
    ups = d["up"]
    for k in KEYS:
        if ups[k] is None:
            ups[k] = torch.randn(fine[k].shape, generator=torch.Generator(device="cuda").manual_seed(len(k)),
                                 device=fine[k].device)
    torch.autograd.backward([fine[k] for k in KEYS], [ups[k] for k in KEYS])
    grads = [t.grad for t in leaves] + [vf.grad] + [p.grad for p in head.parameters()]
    return fine, grads


def check_agree(d):
    """Forward bits and, under torch.use_deterministic_algorithms(True), the leaf gradients (the fine head's parameter
    gradients within 1e-5 of each tensor's maximum: they are summed in another grouping)."""
    torch.use_deterministic_algorithms(True)
    try:
        fa, ga = step(d, False)
        fb, gb = step(d, True)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    same_fwd = all(torch.equal(fa[k], fb[k]) for k in KEYS)
    same_leaf = all(torch.equal(x, y) for x, y in zip(ga[:6], gb[:6]))
    head_err = max(float((x.double() - y.double()).abs().max() / max(float(x.double().abs().max()), 1e-30))
                   for x, y in zip(ga[6:], gb[6:]))
    return {"forward_bitwise": same_fwd, "leaf_grads_bitwise": same_leaf, "head_param_grad_rel_err": head_err}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=9)
    ap.add_argument("--profile", action="store_true", help="device time per arm from torch.profiler (a run of its own)")
    ap.add_argument("--memory", action="store_true", help="peak-allocation increase of one step per arm")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    d = setup(dev)
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}", flush=True)
    res = {"card": info, "B": B, "V": V, "Vs": VS, "H": H, "W": W, "P": P, "counts": d["masks"].sum(1).tolist()}
    arms = {"loop": lambda: step(d, False), "batched": lambda: step(d, True), "coarse_only": lambda: step(d, False, True)}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for name in ("loop", "batched"):
            for _ in range(2):
                arms[name]()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    arms[name]()
                torch.cuda.synchronize()
            dev_us = sum(e.self_device_time_total for e in prof.key_averages()) / 3
            res.setdefault("device_ms_per_step", {})[name] = dev_us / 1e3
    elif args.memory:
        for name in ("loop", "batched"):
            arms[name]()
            res.setdefault("peak_mib", {})[name] = peak_mib(arms[name])
    else:
        res["agree"] = check_agree(d)
        for fn in arms.values():           # warm-up of every shape the timed window uses
            fn()
        samples = alternate(arms, args.repeats, host_ms)
        res["step_ms"] = {k: summary(v) for k, v in samples.items()}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
