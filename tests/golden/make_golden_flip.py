"""Generates tests/golden/flip_test.npz by running the UNMODIFIED reference (imported read-only
through oracle/refshim.py) on the seeded inputs of tests/flip_cases.py.  Build container only:
    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_flip.py

The reference ships the pieces of flip testing but not their composition; the composition recorded
here is the one its config keys imply (TEST.FLIP_TEST, TEST.SHIFT_HEATMAP, config.py:118,120):
    Lf = logits of flip(x, 3)                                  img_utils.py:319-331
    Fb = flip_back(Lf viewed as [N, J, D*H, W], pairs)         transforms.py:5-19
    shift: Fb[..., 1:] = Fb[..., :-1].copy()
    coords = softmax_integral_tensor(0.5 * (L + Fb), ...)      integral_loss.py:71-86
Stored: flip of an index image batch, flip_back of index volumes (a pure gather, so the index map
pins it completely) and the merged coordinates for each case with the shift off and on."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)
from oracle import refshim  # noqa: E402
from tests import flip_cases as fc  # noqa: E402

r = refshim.ref()
il, iu = r.integral_loss, r.img_utils
import importlib  # noqa: E402
tr = importlib.import_module("lib.utils.transforms")

out = {"flip_images": iu.flip(torch.from_numpy(fc.index_images()), 3).numpy()}
for tag, (N, J, D, H, W, seed, scale, pairs) in fc.CASES.items():
    out["flip_back_" + tag] = tr.flip_back(fc.index_volume(tag), pairs).copy()
    L2 = fc.logits2N(tag)
    for shift in (0, 1):
        fb = tr.flip_back(L2[N:].reshape(N, J, D * H, W).copy(), pairs)
        if shift:
            fb[:, :, :, 1:] = fb[:, :, :, 0:-1].copy()
        merged = 0.5 * (L2[:N] + fb.reshape(N, J * D, H, W))
        coords = il.softmax_integral_tensor(torch.from_numpy(np.ascontiguousarray(merged)), J, True, W, H, D)
        out["coords_%s_shift%d" % (tag, shift)] = coords.numpy()
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "flip_test.npz"), **out)
print("wrote flip_test", {k: v.shape for k, v in out.items()})
