"""The attention error bound of `tests/attention_ref.py` is tight enough to catch real online-softmax mistakes.

`flash_model` restates the arithmetic of `flash_attn_d64_kernel` (viewcrafter_b200/csrc/attention.cu) in numpy: BNK-key tiles of K / V
(zero-filled past Nk, as TMA loads them), fp32 scores, masked keys set to -inf, the exp2-domain running max m with
alpha = 2^(m_old - m_new) rescaling l and O, e = 2^(s * scale * log2(e) - m) in fp32, P = fp16(e), l summed from the unrounded e,
O += P V in fp32 and one fp16 rounding of O / l (plus the accumulate target).  The correct model must sit at or below half the bound on
every rung at both tile widths; each mutant, a mistake an online softmax can make, must break the bound on a named rung.
"""
import math

import numpy as np
import pytest
import torch

from tests import attention_ref as ar

def flash_model(q, k, v, scale, bnk, mutant=None, base=None):
    """q [Nq, 64], k / v [Nk, 64] fp16 numpy arrays -> fp16 [Nq, 64]."""
    f32 = np.float32
    Nq, Nk = q.shape[0], k.shape[0]
    sl2 = f32(scale) * f32(1.4426950408889634)
    qf = q.astype(f32)
    m = np.full(Nq, -np.inf, f32)
    l = np.zeros(Nq, f32)
    o = np.zeros((Nq, 64), f32)
    with np.errstate(over="ignore", invalid="ignore"):
        for j in range(0, Nk, bnk):
            kt = np.zeros((bnk, 64), np.float16)
            vt = np.zeros((bnk, 64), np.float16)
            kt[:min(bnk, Nk - j)] = k[j:j + bnk]
            vt[:min(bnk, Nk - j)] = v[j:j + bnk]
            sc = (qf @ kt.astype(f32).T).astype(f32)
            valid = Nk - j
            if valid < bnk:
                sc[:, valid + (1 if mutant == "leak" else 0):] = -np.inf
            if mutant == "no-max":
                mn = np.zeros(Nq, f32)
                alpha = np.ones(Nq, f32)
            else:
                mn = np.maximum(m, sc.max(1) * sl2).astype(f32)
                alpha = np.exp2(m - mn).astype(f32)
            m = mn
            if mutant != "l-alpha":
                l = (l * alpha).astype(f32)
            if mutant != "o-alpha":
                o = (o * alpha[:, None]).astype(f32)
            e = np.exp2((sc.astype(np.float64) * np.float64(sl2) - mn[:, None]).astype(f32)).astype(f32)   # ex2(fma(s, sl2, -m))
            l = (l + e.sum(1, dtype=f32)).astype(f32)
            o = (o + e.astype(np.float16).astype(f32) @ vt.astype(f32)).astype(f32)
        out = (o / l[:, None]).astype(f32)
    if base is not None:
        out = (out + base.astype(f32)).astype(f32)
    return out.astype(np.float16)


def ratio(rung, Nq, Nk, bnk, mutant=None, accumulate=False, seed=0):
    q, k, v = ar.rung_qkv(rung, 1, Nq, Nk, 1, seed, device="cpu", bnk=bnk)
    q, k, v = q[0, :, 0], k[0, :, 0], v[0, :, 0]
    base = (torch.randn(Nq, 64, generator=torch.Generator().manual_seed(seed + 1)) * 4.0).half() if accumulate else None
    out = flash_model(q.numpy(), k.numpy(), v.numpy(), 0.125, bnk, mutant, None if base is None else base.numpy())
    o, p, mag = ar.attn_ref(q, k, v, 0.125)
    ref = o if base is None else o + base.double()
    return ar.worst_ratio(torch.from_numpy(out), ref, ar.attn_bound(o, p, mag, v, base=base))


@pytest.mark.parametrize("bnk", [64, 128])
@pytest.mark.parametrize("Nk", [1, 63, 77, 128, 200, 333])
def test_correct_model_within_half_the_bound(bnk, Nk):
    """accumulate=True rounds base + O / l once, and term (e) of the bound is that rounding alone: it can reach 1 but not pass it."""
    worst = {}
    for rung in ar.rungs_for(Nk, bnk):
        for acc in (False, True):
            worst[(rung, acc)] = ratio(rung, 48, Nk, bnk, accumulate=acc)
    bad = {k: v for k, v in worst.items() if not v <= (1.0 if k[1] else 0.5)}
    assert not bad, f"bnk={bnk} Nk={Nk}: {bad}"


@pytest.mark.parametrize("bnk", [64, 128])
@pytest.mark.parametrize("mutant,rung,Nk", [("no-max", "shift+30", 200), ("leak", "shift-30", 77), ("leak", "shift-30", 333),
                                            ("leak", "v-offset", 333), ("o-alpha", "late-max@last", 200),
                                            ("l-alpha", "late-max@last", 200), ("o-alpha", "ramp", 333), ("l-alpha", "ramp", 333)])
def test_mutant_breaks_the_bound(bnk, mutant, rung, Nk):
    r = ratio(rung, 48, Nk, bnk, mutant=mutant)
    assert r > 1.0, f"{mutant} on {rung} (Nk={Nk}, bnk={bnk}) stays within the bound: {r:.3g}"


def test_bound_refuses_rows_past_its_derivation():
    o = torch.zeros(1, 64, dtype=torch.float64)
    with pytest.raises(AssertionError):
        ar.attn_bound(o, torch.zeros(1, ar.MAX_NK + 1, dtype=torch.float64), torch.zeros(1, ar.MAX_NK + 1, dtype=torch.float64),
                      torch.zeros(ar.MAX_NK + 1, 64))


def test_softmax_bound_covers_an_exact_fp16_rounding():
    """The softmax_rows bound is at least the fp16 rounding of the exact probabilities, on every kind of row it is used for."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(8, 300, generator=g) * 40.0
    x[1, 5:] = -math.inf
    x[2] = 7.0
    x[3, 0] += 400.0
    ref = ar.softmax_ref(x, 0.05)
    err = (ref.half().double() - ref).abs()
    assert bool((err <= ar.softmax_bound(x, 0.05)).all())
