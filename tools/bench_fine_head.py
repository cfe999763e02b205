"""The fine-pass decoder head per scene (DESIGN §3.16): forward + backward of network.py:508-512 at LaRa's size (V = 4
source views, N = 262144 voxels, K = 2, a mask keeping half the Gaussians, so n ~ 262144 points, D = 80, sh_dim 12).

Three arms, alternating in one process after a warm-up: the fused head (``FineHead.fine_shs``), and LaRa's torch head
(the same ``norm`` / ``cross_att`` / ``mlp_fine`` modules called as ``Decoder.forward_fine`` calls them, with the gathers,
einsum and residual around it) in fp32 and under bf16 autocast.  Each is timed with CUDA events; the median and range
over --repeats are printed, with the peak-memory increase (the peak allocation over the allocation before the call)
of one forward + backward.  Prints the card's name and power limit, then one JSON line.

    python tools/bench_fine_head.py [--repeats 7] [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from timing import alternate, card, cuda_ms, peak_mib, summary  # noqa: E402  (tools/ is on sys.path as a script)

V, N, K, D, SH = 4, 262144, 2, 80, 12


def torch_head(head, vf_up, mask, pf, shs):
    """network.py:508-512 with LaRa's modules (Decoder.forward_fine, :280-284)."""
    point_feats = torch.einsum("lcb->blc", pf)
    vpf = vf_up.unsqueeze(1).expand(-1, K, -1)[mask.view(-1, K)]
    x = head.norm(vpf.unsqueeze(1))
    x = head.cross_att(x, point_feats, point_feats, need_weights=False)[0]
    return head.mlp_fine(x).float().view(-1, *shs.shape[-2:]) + shs[mask]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10, help="forward + backward calls per timed repeat")
    args = ap.parse_args()
    from lara_b200.fine_head import FineHead
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    head = FineHead(D, SH).to(dev)
    vf = torch.randn((N, D), device=dev, generator=g).requires_grad_(True)
    mask = torch.rand(N * K, device=dev, generator=g) < 0.5
    n = int(mask.sum())
    pf = torch.rand((V, 8, n), device=dev, generator=g).requires_grad_(True)
    shs = torch.randn((N * K, SH // 3, 3), device=dev, generator=g).requires_grad_(True)
    up = torch.randn((n, SH // 3, 3), device=dev, generator=g)

    def fused():
        head.fine_shs(vf, K, mask, pf, shs).backward(up)

    def fp32():
        torch_head(head, vf, mask, pf, shs).backward(up)

    def bf16():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = torch_head(head, vf, mask, pf, shs)
        out.backward(up)

    arms = {"fused": fused, "torch_fp32": fp32, "torch_bf16_autocast": bf16}

    def clear():
        for t in [vf, pf, shs, *head.parameters()]:
            t.grad = None

    peak, failed = {}, {}
    for name, fn in list(arms.items()):
        try:
            fn()                                   # one call first: an arm that cannot run at this size is reported
        except RuntimeError as ex:
            failed[name] = str(ex).strip().splitlines()[0]
            del arms[name]
            clear()
            continue
        clear()
        for _ in range(2):                         # warm-up (and the first-call allocations)
            fn()
            clear()
        peak[name] = peak_mib(fn)
        clear()
    times = alternate(arms, args.repeats, lambda fn: 1e3 * cuda_ms(lambda: (fn(), clear()), args.iters))
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}; V={V} n={n} D={D} sh_dim={SH}")
    res = {"card": c, "V": V, "n": n, "D": D, "sh_dim": SH}
    for name, ts in times.items():
        t = summary(ts)
        print(f"  {name:22s} fwd+bwd {t['median']:9.1f} us (range {t['min']:.1f} - {t['max']:.1f})  "
              f"peak +{peak[name]:8.1f} MB")
        res[name] = {"fwd_bwd_us": t, "peak_increase_mb": round(peak[name], 1)}
    for name, msg in failed.items():
        print(f"  {name:22s} fails at this size: {msg}")
        res[name] = {"error": msg}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
