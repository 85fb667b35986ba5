"""Generate tests/golden/unet_mc64_T48.npz by running the UNMODIFIED reference UNetModel on the CPU (build container only).

    python tools/make_golden_long_clip.py

The case of oracle/make_golden.py's `unet_*` fixtures at T = 48, past the 32 frames of the short-clip temporal-attention kernel:
model_channels 64, 8x8 latent, a context of 333 tokens (77 + 16 T != 333: the shared image-token branch), the same synthetic weights
(seed 3) and input draws (seed 5).  Only this file is written; the existing fixtures are left as they are.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ref_shims  # noqa: E402
from oracle.make_golden import OUT, _load_synth  # noqa: E402

NAME, OVER, T, H, W = "mc64_T48", dict(model_channels=64), 48, 8, 8


def main():
    m = ref_shims.build_unet(**OVER)
    shapes = _load_synth(m, seed=3)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 8, T, H, W, generator=g)
    ctx = torch.randn(1, 333, 1024, generator=g).half().float()      # fp16-representable: stored exactly as fp16 (file size)
    t = torch.tensor([499])
    fs = torch.tensor([10])
    with torch.no_grad():
        y = m(x, t, context=ctx, fs=fs)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"unet_{NAME}.npz")
    np.savez_compressed(path, shapes=shapes, kwargs=json.dumps(OVER), x=x.numpy(), ctx=ctx.numpy().astype(np.float16), t=t.numpy(),
                        fs=fs.numpy(), y=y.numpy())
    print(NAME, "out std", float(y.std()), "absmax", float(y.abs().max()), "->", path)


if __name__ == "__main__":
    main()
