"""Host side of the U-Net's FP8 mode: the weight quantisation (ops.pack_fp8) on every kind of packed weight, the C-ABI descriptor,
UNetModel.enable_fp8's scope and refusals, and the unchanged state_dict."""
import pytest
import torch

from viewcrafter_b200 import ops


def _expected(w_packed, taps):
    """e4m3 per output channel n over all taps: s = amax / 448 (1 if 0), q = float8_e4m3fn(clamp(w / s, +-448))."""
    rows, K = w_packed.shape
    w = w_packed.float().view(taps, rows // taps, K)
    amax = w.abs().amax(dim=(0, 2))
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return (w / s[None, :, None]).clamp(-448, 448).to(torch.float8_e4m3fn).view(rows, K), s


def _same(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def test_pack_fp8_rounding_and_zero_rows():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(9 * 40, 96, generator=g) * 0.05).half()
    w[7] = 0                                            # tap 0 of channel 7 ...
    w.view(9, 40, 96)[:, 11] = 0                        # ... and every tap of channel 11
    q, s = ops.pack_fp8(w, taps=9)
    q_ref, s_ref = _expected(w, 9)
    assert q.dtype == torch.float8_e4m3fn and q.shape == w.shape and s.shape == (40,)
    assert _same(q, q_ref) and torch.equal(s, s_ref)
    assert s[11] == 1.0 and (q.view(9, 40, 96)[:, 11].float() == 0).all()
    assert s[7] != 1.0                                  # the other taps of channel 7 set its scale
    wmax = w.float().view(9, 40, 96).abs().amax(dim=(0, 2))
    assert (q.float().view(9, 40, 96).abs().amax(dim=(0, 2))[wmax > 0] == 448).all()


def test_pack_fp8_folded_layernorm_and_colsum():
    g = torch.Generator().manual_seed(1)
    w, gamma, beta = torch.randn(192, 64, generator=g) * 0.1, torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g)
    w16, _, _ = ops.fold_layernorm(w, gamma, beta)
    q, s = ops.pack_fp8(w16)
    q_ref, s_ref = _expected(w16, 1)
    assert _same(q, q_ref) and torch.equal(s, s_ref)
    w8 = ops.Fp8Weight(q, s)
    assert torch.equal(ops.fp8_colsum(w8), (q.float() * s[:, None]).sum(1))


def test_pack_fp8_geglu_interleave_keeps_scale_order():
    g = torch.Generator().manual_seed(2)
    w, b = torch.randn(2 * 256, 64, generator=g), torch.randn(2 * 256, generator=g)
    w[3] *= 100                                         # a value row with a distinct scale
    gamma, beta = torch.ones(64), torch.zeros(64)
    wp, bp, cs = ops.pack_geglu_ln(w, b, gamma, beta)
    q, s = ops.pack_fp8(wp)
    idx = ops._geglu_index(512, "cpu")
    _, s_orig = _expected(ops.fold_layernorm(w, gamma, beta)[0], 1)
    assert torch.equal(s, s_orig[idx])                  # per-row scales follow the interleaved rows
    assert int(torch.argmax(s)) == int((idx == 3).nonzero())


def test_pack_fp8_upconv_presummed_taps():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(32, 48, 3, 3, generator=g)
    for p in ops.pack_upconv3x3(w):
        q, s = ops.pack_fp8(p, taps=4)
        q_ref, s_ref = _expected(p, 4)
        assert _same(q, q_ref) and torch.equal(s, s_ref)


def test_gemm_desc_abi_version_9():
    """ABI 9: the descriptor's FP8 fields, and the version both the binding and include/vc_b200.h declare (9 since ln_part records hold
    (sum, M2 about the chunk mean))."""
    import os
    import re
    from viewcrafter_b200 import _lib
    names = [f[0] for f in _lib.GemmDesc._fields_]
    assert names[-4:] == ["peer", "fp8", "w_scale", "a_amax"]
    assert _lib.ABI_VERSION == 9
    header = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vc_b200.h")
    with open(header) as f:
        assert int(re.search(r"#define VC_B200_ABI_VERSION (\d+)", f.read()).group(1)) == _lib.ABI_VERSION
    d = _lib.GemmDesc()
    assert d.fp8 == 0 and not d.w_scale and not d.a_amax
    assert "vc_absmax_f16" in _lib.SIGNATURES


def _small_unet():
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    torch.manual_seed(0)
    return UNetModel(**dict(UNET_PARAMS, model_channels=64)).eval()


def test_fp8_packs_scope():
    m = _small_unet()
    m.enable_fp8()                                      # CPU parameters: the packs are built on first use
    P8, P = m._packs(), m._packed
    W8 = ops.Fp8Weight
    assert not isinstance(P8["input"][0][0]["w"], W8)  # first conv (K = 8)
    assert not isinstance(P8["out_w"], W8)              # last conv (N = 4)
    res = P8["input"][1][0]
    assert isinstance(res["w1"], W8) and isinstance(res["w2"], W8) and all(isinstance(t[2], W8) for t in res["tconv"])
    sp = P8["input"][1][1]
    assert sp["kind"] == "S" and isinstance(sp["in_w"], W8) and isinstance(sp["out_w"], W8)
    Q, Q16 = sp["blocks"][0], P["input"][1][1]["blocks"][0]
    for k in ("qkv1", "o1_w", "q2", "o2_w", "ff1", "ff2_w"):
        assert isinstance(Q[k], W8), k
    assert Q["kv_txt"] is Q16["kv_txt"] and Q.get("kv_img") is Q16.get("kv_img")      # context K/V stay fp16
    assert torch.equal(Q["q2_cs"], ops.fp8_colsum(Q["q2"])) and torch.equal(Q["ff1_cs"], ops.fp8_colsum(Q["ff1"]))
    assert isinstance(P8["init_attn"][0]["in_w"], W8)
    kinds = {m_["kind"]: m_ for st in P8["input"] + P8["output"] for m_ in st}
    assert isinstance(kinds["D"]["w"], W8) and all(isinstance(w, W8) for w in kinds["U"]["w"])
    m.enable_fp8(False)
    assert m._packs() is P and m._packed8 is None


def test_enable_fp8_refusals_and_state_dict():
    m = _small_unet()
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    m.enable_fp8()
    sd1 = m.state_dict()
    assert sd0.keys() == sd1.keys() and all(torch.equal(sd0[k], sd1[k]) for k in sd0)
    m._packs()
    m.load_state_dict(sd0)
    assert m._packed8 is None and m.fp8_enabled()      # rebuilt from the new weights on the next forward
    prev = ops.set_reproducible(True)
    try:
        with pytest.raises(ValueError):
            _small_unet().enable_fp8()
    finally:
        ops.set_reproducible(prev)
    m2 = _small_unet()
    m2._comm = object()                                 # what parallel.shard_model sets for frame groups of several GPUs
    with pytest.raises(NotImplementedError):
        m2.enable_fp8()
