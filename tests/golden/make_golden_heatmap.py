"""Golden vectors for the heat-map decode: the UNMODIFIED reference lib/core/inference.py
get_max_preds (:12-40), get_final_preds' refinement (:43-68, with transform_preds replaced by the
identity so that the refined heat-map coordinates themselves are pinned) and get_depth_preds
(:144-170) on one fixed seeded set: 3 images x 5 joints of 48 x 64 maps with planted ties, border
maxima, a non-positive map and equal neighbours, and 16-bin depth logits.  Build container only:
    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_heatmap.py"""
import os
import sys
import types

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)
from oracle import refshim  # noqa: E402

N, J, H, W, D = 3, 5, 48, 64, 16
rng = np.random.default_rng(811)
yy, xx = np.mgrid[0:H, 0:W]
hm = np.empty((N, J, H, W), dtype=np.float32)
for n in range(N):
    for j in range(J):
        cy, cx = rng.uniform(2, H - 3), rng.uniform(2, W - 3)
        hm[n, j] = np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / 8.0) + 0.01 * rng.standard_normal((H, W))
hm[0, 0, 10, 20] = hm[0, 0, 30, 5] = 2.0                 # tie: the first index wins
hm[0, 1, 0, 33] = 3.0                                    # maximum on the top row
hm[0, 2, H - 1, 7] = 3.0                                 # bottom row
hm[0, 3, 17, 0] = 3.0                                    # left column
hm[0, 4, 22, W - 1] = 3.0                                # right column
hm[1, 0] = -np.abs(hm[1, 0]) - 0.5                       # maxval <= 0: coordinates zeroed
hm[1, 1, 20, 30] = 4.0                                   # equal neighbours: sign 0 in both axes
hm[1, 1, 20, 29] = hm[1, 1, 20, 31] = 1.0
hm[1, 1, 19, 30] = hm[1, 1, 21, 30] = 1.0
hm[1, 2, 1, 1] = 4.0                                     # one inside the border: refinement skipped
hm[1, 3, 2, 2] = 4.0                                     # the first refined position
depth = (3.0 * rng.standard_normal((N, J * D))).astype(np.float32)

r = refshim.ref()
preds, maxvals = r.inference.get_max_preds(hm.copy())
r.inference.transform_preds = lambda coords, center, scale, output_size: coords.copy()
S = types.SimpleNamespace
cfg = S(TEST=S(POST_PROCESS=True), MODEL=S(NUM_JOINTS=J, DEPTH_RES=D), DATASET=S(DEPTH_RANGE=2000))
refined, _ = r.inference.get_final_preds(cfg, hm.copy(), np.zeros((N, 2)), np.ones((N, 2)))
dpred = r.inference.get_depth_preds(cfg, depth.copy())
out = dict(hm=hm, depth=depth, preds=preds, maxvals=maxvals, refined=refined, depth_mm=dpred)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "heatmap_decode.npz"), **out)
print({k: (v.shape, v.dtype) for k, v in out.items()})
