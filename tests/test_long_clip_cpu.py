"""Pin the CPU oracle at T = 48 (past the 32 frames of the short-clip temporal-attention kernel) against the unmodified reference
UNetModel (tests/golden/unet_mc64_T48.npz, written by tools/make_golden_long_clip.py: shared image tokens, since L = 333 != 77 + 16 T)."""
import json
import os

import numpy as np
import torch

from oracle import lvdm_oracle as O
from oracle import synth


def test_unet_T48_oracle_matches_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "unet_mc64_T48.npz"), allow_pickle=False)
    assert g["x"].shape[2] == 48
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    sd = synth.synth_state_dict(shapes, seed=3)
    with torch.no_grad():
        y = O.unet_forward(sd, torch.from_numpy(g["x"]), torch.from_numpy(g["t"]), torch.from_numpy(g["ctx"]).float(),
                           torch.from_numpy(g["fs"]))
    np.testing.assert_allclose(y.numpy(), g["y"], rtol=0, atol=5e-5)
