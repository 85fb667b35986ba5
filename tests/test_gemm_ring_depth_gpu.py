"""Ring depths of the tap-GEMM tile widths whose depth the shared-memory output tile changed (GemmCfg<BN>::STAGES in
csrc/gemm_tap.cu): BN = 64 holds 8 stages.  Per-tile iteration counts straddle that depth, with the residual loaded by TMA
(contiguous and in place) and read directly (unaligned pitch), through the same operands, references and tolerance as
test_gemm_sweep_gpu.py."""
import pytest
import torch

from tests.test_gemm_sweep_gpu import Lin

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

DEPTH = {64: 8}                                          # GemmCfg<BN>::STAGES


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


@pytest.mark.parametrize("BN", sorted(DEPTH))
def test_ring_depth(ops, BN):
    """Iterations per tile S - 1, S, S + 1 and 2 S + 1 (S = ring stages), a two-source K split whose second slab is not a whole
    k-block, and every residual path.  3 m-tiles, the last one ragged."""
    S, N = DEPTH[BN], BN
    assert ops._lib.load().vc_gemm_tile_n(N, 0) == BN
    M = 128 * 3 - 37
    for K in (64 * (S - 1), 64 * S, 64 * S + 8, 64 * 2 * S + 24):
        case = Lin(M, K, N, seed=5000 + K)
        for res_kind in ("contig", "inplace", "p8"):
            case.check(ops, f"BN={BN} K={K} res={res_kind}", res_kind=res_kind)
    for K2 in (8, 72):
        Lin(M, 64 * (S - 1), N, seed=6000 + K2, K2=K2).check(ops, f"BN={BN} K1={64 * (S - 1)} K2={K2}")
