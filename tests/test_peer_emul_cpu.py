"""The shapes test_peer_kernels_gpu.py runs through the layout switch in the GEMM epilogue are shapes the product runs there
(parallel.fused_scatter_ok with the kernel's 4-rank limit): a patch that straddles a rank's pixel range or a frame would make TMA stores
with negative coordinates, which fault on hardware (test_peer_scatter_model_cpu.py).  And PeerFrameComm.scatter_plan decides with that
predicate and nothing else."""
import pytest

from tests import peer_emul as pe
from tests.test_peer_kernels_gpu import EXCHANGE_CASES, GRAPH_SCATTER, GRID_SCATTER, LEVEL, SCATTER_CASES
from viewcrafter_b200 import parallel


@pytest.mark.parametrize("producer,P,T,B,HW", SCATTER_CASES + GRID_SCATTER + [GRAPH_SCATTER])
def test_every_fused_scatter_case_is_a_product_shape(producer, P, T, B, HW):
    assert pe.scatter_case_ok(P, T, B, HW, LEVEL[HW][2])


def test_the_smallest_level_stays_on_the_exchange_kernel():
    cases = [c for c in EXCHANGE_CASES if c[3] == 144]
    assert any(c[0] == 2 for c in cases)
    for P, T, B, HW, Cc in cases:
        assert not pe.scatter_case_ok(P, T, B, HW, Cc), (P, T, B, HW, Cc)
        assert not parallel.fused_scatter_ok("aligned", 2, 4, parallel.frame_ranges(T, P), B, HW, Cc)


@pytest.mark.parametrize("fused,max_p", [("aligned", 2), ("aligned", 4), ("1", 4), ("0", 4)])
def test_scatter_plan_follows_the_predicate(monkeypatch, fused, max_p):
    monkeypatch.setattr(parallel, "_ScatterPlan", lambda comm, to_sites, B, HW, Cc: ("plan", to_sites, B, HW, Cc))
    n_plans = 0
    for P in (1, 2, 3, 4, 8):
        for T in (1, 3, 16, 25):
            for HW in (9216, 2304, 576, 144, 48, 64):
                for B in (1, 2, 3, 4, 5):
                    for Cc in (320, 640, 48):
                        comm = object.__new__(parallel.PeerFrameComm)
                        comm.world, comm.bmax, comm.fused, comm.fused_max_p = P, 4, fused, max_p
                        comm.ranges = parallel.frame_ranges(T, P)
                        ok = parallel.fused_scatter_ok(fused, max_p, 4, comm.ranges, B, HW, Cc)
                        got = comm.scatter_plan(True, B, HW, Cc)
                        assert (got is not None) == ok, (fused, max_p, P, T, HW, B, Cc)
                        n_plans += ok
    assert (n_plans > 0) == (fused != "0")
