"""Per-scene refinement, host side (no GPU needed): a float64 restatement of the Adam step over the flat Gaussian record
against torch.optim.Adam on get_params' six groups, the groups' learning rates, the C entry's argument checks and the
mapping of LaRa's ``finetuning`` config."""
import ctypes

import numpy as np
import pytest
import torch

from lara_b200 import finetune as F

LRS = dict(position_lr=0.000016, feature_lr=0.0025, opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001)


def group_of_record(n: int, M: int) -> np.ndarray:
    """The group (index into F.GROUPS) of every element of the record centers | shs | opacity | scaling | rotation."""
    shs = np.full((n, M, 3), 2)
    shs[:, 0, :] = 1
    return np.concatenate([np.zeros(3 * n), shs.reshape(-1), np.full(n, 3), np.full(2 * n, 4), np.full(4 * n, 5)]).astype(int)


def adam64(x, grads, lrs, group, betas=(0.9, 0.999), eps=1e-15):
    """Adam (Kingma & Ba, with torch's placement of eps) in float64 over a flat record: x [E], grads [T, E], the learning
    rate of element e lrs[group[e]].  Returns (x, exp_avg, exp_avg_sq) after the T steps."""
    x = np.array(x, dtype=np.float64)
    m, v = np.zeros_like(x), np.zeros_like(x)
    lr = np.asarray(lrs, dtype=np.float64)[group]
    b1, b2 = betas
    for t, g in enumerate(grads, start=1):
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        x = x - lr / (1 - b1 ** t) * m / (np.sqrt(v) / np.sqrt(1 - b2 ** t) + eps)
    return x, m, v


def record(tensors):
    return np.concatenate([t.detach().reshape(-1).numpy() for t in tensors])


@pytest.mark.parametrize("M", [1, 4, 9, 16])
def test_float64_restatement_agrees_with_torch_adam_on_get_params_groups(M):
    n, steps = 37, 50
    g = torch.Generator().manual_seed(M)
    shapes = [(n, 3), (n, M, 3), (n, 1), (n, 2), (n, 4)]
    init = [torch.randn(s, generator=g, dtype=torch.float64) for s in shapes]
    grads = [[torch.randn(s, generator=g, dtype=torch.float64) * 10 ** float(torch.randint(-6, 1, (1,), generator=g))
              for s in shapes] for _ in range(steps)]
    # torch: get_params' six leaves, f_dc = shs[:, :1] and f_rest = shs[:, 1:]
    xyz, shs, opa, sca, rot = (t.clone() for t in init)
    leaves = [xyz, shs[:, :1].clone(), shs[:, 1:].clone(), opa, sca, rot]
    for t in leaves:
        t.requires_grad_(True)
    lrs = F.group_lrs(**LRS)
    opt = torch.optim.Adam([{"params": [t], "lr": lr, "name": name} for t, lr, name in zip(leaves, lrs, F.GROUPS)],
                           betas=(0.9, 0.999), eps=1e-15, foreach=False)
    for gs in grads:
        gx, gsh, go, gsc, gr = gs
        for t, gt in zip(leaves, (gx, gsh[:, :1], gsh[:, 1:], go, gsc, gr)):
            t.grad = gt.clone()
        opt.step()
    got = record([leaves[0], torch.cat(leaves[1:3], 1)] + leaves[3:])
    st = [opt.state[t] for t in leaves]
    got_m = record([st[0]["exp_avg"], torch.cat([st[1]["exp_avg"], st[2]["exp_avg"]], 1)] + [s["exp_avg"] for s in st[3:]])
    got_v = record([st[0]["exp_avg_sq"], torch.cat([st[1]["exp_avg_sq"], st[2]["exp_avg_sq"]], 1)] +
                   [s["exp_avg_sq"] for s in st[3:]])
    want, want_m, want_v = adam64(record(init), np.stack([record(gs) for gs in grads]), lrs, group_of_record(n, M))
    for a, b in ((got, want), (got_m, want_m), (got_v, want_v)):
        assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(b).max())


@pytest.mark.parametrize("M", [1, 4, 9, 16])
def test_groups_and_learning_rates_follow_get_params(M):
    n = 5
    lrs = F.group_lrs(**LRS)
    assert lrs == (0.000016, 0.0025, 0.0025 / 20.0, 0.05, 0.005, 0.001)
    grp = group_of_record(n, M)
    assert grp.size == n * (10 + 3 * M)
    counts = np.bincount(grp, minlength=6)
    assert counts.tolist() == [3 * n, 3 * n, 3 * (M - 1) * n, n, 2 * n, 4 * n]
    # only the group differs between the restatement's runs: each group moves at its own rate, f_rest at feature_lr/20
    x0 = np.zeros(grp.size)
    x1, _, _ = adam64(x0, np.ones((1, grp.size)), lrs, grp)
    for k in range(6):
        if counts[k]:
            np.testing.assert_allclose(-x1[grp == k], lrs[k], rtol=1e-12)


def test_finetune_settings_read_laras_config():
    # configs/infer.yaml's finetuning block
    cfg = {"with_ft": False, "steps": 500, "position_lr": 0.000016, "feature_lr": 0.0025, "opacity_lr": 0.05,
           "scaling_lr": 0.005, "rotation_lr": 0.001}
    kw = F.finetune_settings(cfg)
    assert kw == {"steps": 500, **LRS}
    import inspect
    params = inspect.signature(F.finetune_scene).parameters
    assert set(kw) <= set(params)


def _ptrs(vals):
    return (ctypes.c_void_p * 5)(*vals)


def test_adam_entry_rejects_bad_arguments_without_a_device(lib):
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    ok = dict(n=1, M=4, params=_ptrs([p] * 5), grads=_ptrs([p] * 5), moments=p,
              lr=(ctypes.c_double * 6)(*F.group_lrs(**LRS)), beta1=0.9, beta2=0.999, eps=1e-15, bc1=0.1, bc2=0.0316)

    def call(**kw):
        a = {**ok, **kw}
        return lib.srf_gaussian_adam_step(None, a["n"], a["M"], a["params"], a["grads"], a["moments"], a["lr"],
                                          a["beta1"], a["beta2"], a["eps"], a["bc1"], a["bc2"], 1)

    cases = [dict(n=-1), dict(n=-1, params=None), dict(M=0), dict(M=2), dict(M=25), dict(params=None), dict(grads=None), dict(lr=None),
             dict(moments=None), dict(params=_ptrs([p, p, None, p, p])), dict(grads=_ptrs([p, p, p, p, None])),
             dict(beta1=1.0), dict(beta2=-0.1), dict(beta1=float("nan")), dict(eps=-1.0), dict(bc1=0.0),
             dict(bc2=float("nan"))]
    for kw in cases:
        assert call(**kw) != 0, kw
        assert lib.srf_last_error().startswith(b"srf_gaussian_adam_step"), kw
    # n = 0 is a no-op: accepted without any CUDA call, whatever the (empty tensors') pointers
    assert call(n=0) == 0
    assert call(n=0, M=16, params=_ptrs([None] * 5), grads=_ptrs([None] * 5), moments=None) == 0
    assert call(n=0, M=3) != 0 and call(n=-1, M=4) != 0


def test_gaussian_adam_checks_its_tensors():
    t = torch.zeros(4, 3)
    with pytest.raises(ValueError):
        F.GaussianAdam(t, torch.zeros(4, 4, 3), torch.zeros(4, 1), torch.zeros(4, 2), torch.zeros(4, 4), **LRS)
