"""Grid-size invariance of the tap-GEMM: a fixed set of GEMMs whose outputs, GroupNorm records (gn_out) and LayerNorm statistics
(ln_out) are saved to the file given as the first argument.  Run with VC_SM_COUNT=k to cut every grid to k CTAs (read once per
process): with one CTA the smem ring wraps its phase many times and one CTA runs every tile, so the results must equal those of the
full grid bit for bit.  Cases have iteration counts below and above the ring depth and odd and even tile counts.  Prints one line
per case and GEMM_GRID_CHECK_OK.  Used by tests/test_gemm_sweep_gpu.py::test_results_do_not_depend_on_the_grid_size, which also
imports run_all() for the full-grid side."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def _t(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def run_all(ops):
    """name -> {"out", and "gn" / "ln" where the case emits them} (CPU tensors).  The caller forces the GroupNorm records
    (ops.GN_FROM_PRODUCER = 2) and keeps reproducible mode off."""
    res = {}

    def keep(name, out, ln=None):
        d = {"out": out.cpu()}
        part = ops.gn_part_of(out)
        if part is not None:
            d["gn"] = part.part.cpu()
        if ln is not None:
            d["ln"] = ln.cpu()
        res[name] = d
        print(f"{name}: absmax {float(out.float().abs().max()):.4g}{' gn' if 'gn' in d else ''}{' ln' if ln is not None else ''}")

    # BN = 128 (5 stages), 6 iterations per tile, 37 m-tiles (odd), bias + residual, LayerNorm statistics
    M = 128 * 37 - 37
    x, w, b, r = _t((M, 328), 1), _t((128, 328), 2, 328 ** -0.5), _t((128,), 3, dtype=torch.float32), _t((M, 128), 4)
    y, st = ops.linear(x, w, bias=b, res=r, ln_out=True)
    keep("linear_N128_it6_t37_ln", y, st)
    # BN = 160 (4 stages), 3 iterations, 20 m-tiles x 2 n-tiles (even), residual view (pitch % 16 == 8), GroupNorm records
    M = 128 * 20 - 37
    x, w = _t((M, 136), 5), _t((320, 136), 6, 136 ** -0.5)
    rb = _t((M, 328), 7)
    y = ops.linear(x, w, res=rb[:, :320], gn_out=True)
    keep("linear_N320_it3_t40_gn", y)
    # BN = 32 (8 stages), 1 iteration, 9 tiles (odd)
    M = 128 * 9 - 37
    keep("linear_N32_it1_t9", ops.linear(_t((M, 24), 8), _t((32, 24), 9, 24 ** -0.5), bias=_t((32,), 10, dtype=torch.float32)))
    # conv3x3, 9 x 2 iterations per tile, 3 frames x 3 row boxes x 2 n-tiles (even), per-frame bias rows, GroupNorm records
    frames, H, W, Ci = 3, 20, 16, 72
    wc = ops.pack_conv3x3(_t((320, Ci, 3, 3), 11, (9 * Ci) ** -0.5).cpu()).cuda()
    y = ops.conv3x3(_t((frames * H * W, Ci), 12), frames, H, W, wc, bias=_t((frames, 320), 13, dtype=torch.float32), bias_z_div=1,
                    res=_t((frames * H * W, 320), 14), gn_out=True)
    keep("conv3x3_it18_t18_gn", y)
    # temporal conv (BN = 96, 6 stages), 3 iterations, 3 batches x 6 m-tiles (even), residual
    B, T, HW, C = 3, 5, 130, 64
    w3 = ops.pack_conv_temporal(_t((96, C, 3, 1, 1), 15, (3 * C) ** -0.5).cpu()).cuda()
    keep("temporal_it3_t18", ops.conv_temporal(_t((B * T * HW, C), 16), B, T, HW, w3, bias=_t((96,), 17, dtype=torch.float32),
                                              res=_t((B * T * HW, 96), 18)))
    # GEGLU (BN = 128), 4 iterations, 8 m-tiles x 2 n-tiles
    M = 1000
    wg, bg = ops.pack_geglu(_t((256, 200), 19, 200 ** -0.5), _t((256,), 20, dtype=torch.float32))
    keep("geglu_it4_t16", ops.linear(_t((M, 200), 21), wg, bias=bg, geglu=True))
    # BN = 64 (7 stages), 15 iterations (2 S + 1), 5 m-tiles (odd), fp32 output
    M = 128 * 5 - 37
    keep("linear_N64_it15_t5_f32", ops.linear(_t((M, 64 * 14 + 8), 22), _t((64, 64 * 14 + 8), 23, 904 ** -0.5), res=_t((M, 64), 24),
                                              out_f32=True))
    torch.cuda.synchronize()
    return res


if __name__ == "__main__":
    from viewcrafter_b200 import ops
    ops.GN_FROM_PRODUCER, ops.GN_PARTS_MIN_MB, ops.REPRODUCIBLE = 2, 0.0, False
    print(f"VC_SM_COUNT={os.environ.get('VC_SM_COUNT', '(unset)')}")
    results = run_all(ops)
    torch.save(results, sys.argv[1])
    print("GEMM_GRID_CHECK_OK")
