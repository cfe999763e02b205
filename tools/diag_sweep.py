"""Gradient errors of one configuration of the fixed-seed parity sweep slice (tests/test_gpu_headline.py) vs the
reference, plus the reference's own run-to-run noise.   python tools/diag_sweep.py INDEX"""
import os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_gpu_headline as T
from lara_b200 import scene as S
from oracle import ref as REF
from helpers import run_candidate, rel_err

idx = int(sys.argv[1])
rng = np.random.default_rng(20260924)
for it in range(idx + 1):
    tag, sc, cam = T._sweep_config(rng)
dev = torch.device("cuda:0")
ref = REF.load()
bg = torch.full((3,), tag["bg"])
gc, ga = S.upstream_grads(tag["H"], tag["W"], tag["seed"])
mine = run_candidate(sc, cam, bg, dev, grads=(gc, ga))
r, g1, g2 = T._reference_state_and_grads(ref, sc, cam, bg, tag["deg"], dev, gc, ga, twice=True)
errs, worst = T._compare(mine, r, g1, g2, tag["H"], tag["W"])
print(tag, "R", mine["num_rendered"], "errs", errs)
for a_, b_ in T.GRAD_KEYS:
    d = np.abs(mine[a_].astype(np.float64) - g1[b_])
    i = np.unravel_index(np.argmax(d), d.shape)
    print(f"   {b_:10s} rel {rel_err(mine[a_], g1[b_]):.2e} noise {rel_err(g2[b_], g1[b_]):.2e} max|ref| {np.abs(g1[b_]).max():.3e} worst idx {i} mine {mine[a_][i]:.5e} ref {g1[b_][i]:.5e}")
