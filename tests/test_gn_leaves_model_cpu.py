"""Executable specification of reproducible mode's GroupNorm statistics (ops.groupnorm_canonical, csrc/norm.cu: gn_leaves_kernel /
gn_leaves_combine_kernel, csrc/peer.cu: peer_leaves_kernel) in numpy float32.

A frame of HW pixels is cut into nc = ops.gn_leaf_chunks(HW) chunks of HW / nc contiguous pixels.  A leaf is the fp32 (sum, sumsq)
per group of one (sample, frame, chunk); its summation order is a function of the chunk's shape alone.  A per-frame (2-D) GroupNorm
sums its frame's leaves over the chunks in index order, a 5-D GroupNorm over frames, then chunks (fp64, rounded once to fp32).  The
checks below show that the frame layout, the site layouts of 2, 4 and 8 GPUs (25 frames: uneven frame ranges) and batch splits all
produce bit-identical statistics -- because each of them holds every chunk whole and the combine order is fixed."""
import numpy as np
import pytest

from viewcrafter_b200.ops import gn_leaf_chunks
from viewcrafter_b200.parallel import frame_ranges


def leaf(block):
    """[rows, C] fp32 -> [32, 2]: a fixed summation order that depends only on the block's shape."""
    rows, C = block.shape
    g = block.reshape(rows, 32, C // 32)
    s = np.add.reduce(np.add.reduce(g, axis=2, dtype=np.float32), axis=0, dtype=np.float32)
    q = np.add.reduce(np.add.reduce(g * g, axis=2, dtype=np.float32), axis=0, dtype=np.float32)
    return np.stack([s, q], -1)


def leaves(x, rows_per_leaf):
    """[R, C] rows -> [R / rows_per_leaf, 32, 2] (one leaf per block of rows, wherever the block sits)."""
    return np.stack([leaf(x[i:i + rows_per_leaf]) for i in range(0, x.shape[0], rows_per_leaf)])


def combine(lv):
    """[n, 32, 2] -> [32, 2] fp32: index-order fp64 sum."""
    acc = np.zeros((32, 2), np.float64)
    for v in lv:
        acc += v
    return acc.astype(np.float32)


def frame_layout_stats(x, per_frame):
    """x [B, T, HW, C] held whole (one GPU): the statistics of a per-frame or a 5-D GroupNorm."""
    B, T, HW, C = x.shape
    nc = gn_leaf_chunks(HW)
    lv = leaves(x.reshape(-1, C), HW // nc).reshape(B, T, nc, 32, 2)
    if per_frame:
        return np.stack([[combine(lv[b, t]) for t in range(T)] for b in range(B)])
    return np.stack([combine(lv[b].reshape(-1, 32, 2)) for b in range(B)])


def site_layout_stats(x, P):
    """The 5-D GroupNorm as P GPUs compute it: rank r holds [(b, t_all, hw_local)] with the pixels [r HW/P, (r+1) HW/P), computes the
    leaves of its rows, the ranks exchange them (exact copies) and every rank combines them in canonical (b, t, chunk) order."""
    B, T, HW, C = x.shape
    nc = gn_leaf_chunks(HW)
    assert nc % P == 0
    HWl, ncl = HW // P, nc // P
    per_rank = [leaves(x[:, :, r * HWl:(r + 1) * HWl].reshape(-1, C), HW // nc).reshape(B, T, ncl, 32, 2) for r in range(P)]
    canon = np.concatenate(per_rank, axis=2)                                         # [B, T, nc]: rank r's chunks at r * ncl
    out = [np.stack([combine(canon[b].reshape(-1, 32, 2)) for b in range(B)]) for _ in range(P)]
    for o in out[1:]:
        assert np.array_equal(o, out[0])                                             # every rank combines the same values
    return out[0]


def frame_sharded_per_frame_stats(x, P):
    """Per-frame GroupNorms on frame-sharded ranks: rank r holds frames frame_ranges(T, P)[r] of every sample and uses its own leaves."""
    B, T, HW, C = x.shape
    parts = [frame_layout_stats(x[:, f0:f1], True) for f0, f1 in frame_ranges(T, P) if f1 > f0]
    return np.concatenate(parts, axis=1)


def _x(B, T, HW, C, seed):
    r = np.random.default_rng(seed)
    return (r.standard_normal((B, T, HW, C)) * 1.5 + 0.3).astype(np.float16).astype(np.float32)


def test_chunk_count_rule():
    # the latent and U-Net level sizes of 576x1024 (72x128 latents) and 320x512 (40x64) clips, and the VAE's own resolutions
    for hw in (9216, 2304, 576, 144, 2560, 640, 160, 40, 589824, 147456, 36864, 9216, 163840, 40960, 10240, 2560):
        nc = gn_leaf_chunks(hw)
        assert hw % nc == 0 and nc % 8 == 0 and all(nc % P == 0 for P in (2, 4, 8))
        assert nc == 8 or hw // nc >= 256
    assert gn_leaf_chunks(589824) == 1024                      # one 576x1024 VAE frame: 1024 leaves of 576 rows fill the GPU
    assert gn_leaf_chunks(35) == 1 and gn_leaf_chunks(7 * 9) == 1


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("HW", [40, 64, 160])
def test_site_layouts_match_the_frame_layout(B, HW):
    x = _x(B, 25, HW, 64, seed=B * 1000 + HW)
    ref5 = frame_layout_stats(x, per_frame=False)
    ref2 = frame_layout_stats(x, per_frame=True)
    for P in (2, 4, 8):
        assert np.array_equal(site_layout_stats(x, P), ref5), P
        assert np.array_equal(frame_sharded_per_frame_stats(x, P), ref2), P


def test_batch_splits_match():
    x = _x(3, 25, 160, 64, seed=7)
    for per_frame in (False, True):
        whole = frame_layout_stats(x, per_frame)
        split = np.concatenate([frame_layout_stats(x[b:b + 1], per_frame) for b in range(3)])
        pair = np.concatenate([frame_layout_stats(x[:2], per_frame), frame_layout_stats(x[2:], per_frame)])
        assert np.array_equal(whole, split) and np.array_equal(whole, pair)
    # per-frame: one frame per call (per-frame VAE) vs all frames in one call
    one = np.concatenate([frame_layout_stats(x[:, t:t + 1], True) for t in range(25)], axis=1)
    assert np.array_equal(one, frame_layout_stats(x, True))


def test_odd_frames_use_one_chunk():
    x = _x(2, 5, 35, 64, seed=9)                              # HW % 8 != 0: nc = 1, a leaf is a whole frame (single GPU only)
    assert gn_leaf_chunks(35) == 1
    lv = leaves(x.reshape(-1, 64), 35)
    assert lv.shape == (10, 32, 2)
    assert np.array_equal(frame_layout_stats(x, True).reshape(10, 32, 2), np.stack([combine(lv[i:i + 1]) for i in range(10)]))
    assert np.array_equal(np.concatenate([frame_layout_stats(x[b:b + 1], False) for b in range(2)]), frame_layout_stats(x, False))


def test_channel_concat():
    """The ResBlock skip concat x1|x2: a leaf of the concatenated rows, group boundaries inside x2 and across the seam."""
    r = np.random.default_rng(11)
    x1 = r.standard_normal((2, 3, 64, 96)).astype(np.float16).astype(np.float32)
    x2 = r.standard_normal((2, 3, 64, 32)).astype(np.float16).astype(np.float32)
    x = np.concatenate([x1, x2], -1)
    whole = frame_layout_stats(x, True)
    split = np.concatenate([frame_layout_stats(x[b:b + 1], True) for b in range(2)])
    assert np.array_equal(whole, split)
    ref = x.reshape(2, 3, 64, 32, 4).astype(np.float64)
    assert np.allclose(whole[..., 0], ref.sum((2, 4)), rtol=1e-5, atol=1e-3)
    assert np.allclose(whole[..., 1], (ref * ref).sum((2, 4)), rtol=1e-5, atol=1e-3)
