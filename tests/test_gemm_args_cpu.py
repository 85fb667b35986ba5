"""Host-side argument checks that guard vector loads of the kernels.  The tap-GEMM epilogue reads the bias as float4, so a bias that
is not 16-byte aligned -- or per-z bias rows (bias_z_div) that start at bias + z * N with N % 4 != 0 -- must be refused before
anything reaches the driver; the LayerNorm / GroupNorm kernels read rows as 16-byte vectors.  The calls carry fake, otherwise valid
device pointers and run in a child process that sees no CUDA device, so nothing can be launched even by a library that lacks a
check."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHILD = r"""
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from viewcrafter_b200 import _lib
lib = _lib.load()

def desc(N, bias, bias_z_div=0, Z=1):
    d = _lib.GemmDesc()
    d.a, d.lda, d.w, d.out = 0x7f0000000000, 64, 0x7f0000100000, 0x7f0000200000
    d.X, d.Y, d.Z, d.bx, d.by = 256, 1, Z, 128, 1
    d.K, d.K1, d.N, d.num_taps, d.ldo = 64, 64, N, 1, N
    d.bias, d.bias_z_div = bias, bias_z_div
    return d

cases = {                  # the valid layouts first: an error text they leave behind cannot come from a rejected bias
    "aligned": desc(64, 0x7f0000300000),
    "aligned_per_z": desc(64, 0x7f0000300000, bias_z_div=1, Z=2),
    "one_row_ragged_n": desc(6, 0x7f0000300000),
    "misaligned": desc(64, 0x7f0000300004),
    "misaligned_8": desc(64, 0x7f0000300008),
    "per_z_ragged_n": desc(6, 0x7f0000300000, bias_z_div=1, Z=2),
}
res = {}
for name, d in cases.items():
    rc = lib.vc_gemm_tap(C.byref(d), None)
    res[name] = [rc, (lib.vc_last_error() or b"").decode()]
# norm kernels on rows that start 8 bytes past a 16-byte boundary
x, stats, ws = 0x7f0000400008, 0x7f0000500000, 0x7f0000600000
res["layernorm_stats"] = [lib.vc_layernorm_stats(x, 64, 320, 1e-5, stats, None), (lib.vc_last_error() or b"").decode()]
res["layernorm"] = [lib.vc_layernorm(x, 64, 320, stats, stats, 1e-5, ws, None), (lib.vc_last_error() or b"").decode()]
res["groupnorm_stats"] = [lib.vc_groupnorm_stats(x, 320, None, 0, 1, 64, stats, ws, 1 << 20, None), (lib.vc_last_error() or b"").decode()]
print("RESULT " + json.dumps(res))
"""


@pytest.fixture(scope="module")
def results():
    from viewcrafter_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert line, r.stdout + r.stderr
    return json.loads(line[-1][len("RESULT "):])


@pytest.mark.parametrize("case", ["misaligned", "misaligned_8", "per_z_ragged_n"])
def test_gemm_rejects_bias_the_epilogue_cannot_load(results, case):
    rc, msg = results[case]
    assert rc != 0 and "bias" in msg, (rc, msg)


@pytest.mark.parametrize("case", ["layernorm_stats", "layernorm", "groupnorm_stats"])
def test_norms_reject_misaligned_rows(results, case):
    """The LayerNorm / GroupNorm kernels read rows as 16-byte vectors: a misaligned tensor (e.g. a contiguous view that starts 8
    bytes into an allocation) is refused on the host instead of faulting on the device."""
    rc, msg = results[case]
    assert rc != 0 and "16-byte aligned" in msg, (rc, msg)


@pytest.mark.parametrize("case", ["aligned", "aligned_per_z", "one_row_ragged_n"])
def test_gemm_accepts_valid_bias(results, case):
    """Valid bias layouts pass the argument checks; without a device the call fails later, for a reason that is not the bias."""
    rc, msg = results[case]
    assert "bias" not in msg, (rc, msg)
