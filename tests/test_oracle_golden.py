"""Pin the CPU oracle (oracle/lvdm_oracle.py) against outputs of the UNMODIFIED reference.

tests/golden/*.npz were produced by oracle/make_golden.py running the reference modules from
/root/reference.  The reference itself ships no tests, so these fixtures are the pin.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lvdm_oracle as O
from oracle import synth


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name), allow_pickle=False)


def test_ddim_timesteps_bit_exact(golden_dir):
    g = _load(golden_dir, "schedule_kat.npz")
    for m, S in (("uniform_trailing", 50), ("uniform_trailing", 10), ("uniform_trailing", 3),
                 ("uniform_trailing", 1), ("uniform", 50), ("quad", 20)):
        assert np.array_equal(O.make_ddim_timesteps(m, S, 1000), g[f"ts_{m}_{S}"]), (m, S)
    # SURVEY.md §8c known answers
    assert list(O.make_ddim_timesteps("uniform_trailing", 50, 1000)[:3]) == [19, 39, 59]
    assert list(O.make_ddim_timesteps("uniform_trailing", 3, 1000)) == [332, 666, 999]


def test_model_schedule_bit_exact(golden_dir):
    g = _load(golden_dir, "schedule_kat.npz")
    for base in (0.3, 0.7):
        s = O.model_schedule(base_scale=base)
        assert np.array_equal(s["alphas_cumprod"].numpy(), g["alphas_cumprod"])
        assert np.array_equal(s["scale_arr"].numpy(), g[f"scale_arr_{base}"])
    assert s["alphas_cumprod"][999].item() == 0.0


def test_step_scalars_bit_exact(golden_dir):
    g = _load(golden_dir, "schedule_kat.npz")
    for base in (0.3, 0.7):
        s = O.model_schedule(base_scale=base)
        for S, eta in ((50, 1.0), (10, 1.0), (50, 0.0)):
            tab = O.ddim_tables(s, S, "uniform_trailing", eta)
            mine = np.stack([O.step_scalars(tab, i) for i in range(S)])
            ref = g[f"step_scalars_b{base}_S{S}_eta{eta}"]
            assert mine.dtype == np.float32 and np.array_equal(mine.view(np.uint32), ref.view(np.uint32)), (base, S, eta)


def test_timestep_embedding(golden_dir):
    g = _load(golden_dir, "schedule_kat.npz")
    e = O.timestep_embedding(torch.tensor([999, 499, 19, 0]), 320).numpy()
    assert np.array_equal(e, g["temb_999_320"])
    assert np.array_equal(O.timestep_embedding(torch.tensor([10]), 64).numpy(), g["temb_10_64"])


def _toy(x, t, c):
    return torch.tanh(0.7 * x * c["k"] + 0.05 * torch.sin(t.float())[:, None, None, None, None]) + 0.1 * c["b"]


@pytest.mark.parametrize("tag,S,base", [("S5", 5, 0.3), ("S50", 50, 0.7)])
def test_ddim_loop_matches_reference(golden_dir, tag, S, base):
    g = _load(golden_dir, "ddim_small.npz")
    sched = O.model_schedule(base_scale=base)
    x_T = torch.from_numpy(g[f"{tag}_x_T"])
    noises = [torch.from_numpy(n) for n in g[f"{tag}_noises"]]
    cond = {"k": torch.tensor([1.3]), "b": torch.from_numpy(g[f"{tag}_cond_b"])}
    unc = {"k": torch.tensor([0.4]), "b": torch.from_numpy(g[f"{tag}_uncond_b"])}
    out, inter = O.ddim_sample(_toy, sched, x_T.shape, S, cond, unc, x_T, noises)
    assert len(inter["x_inter"]) == int(g[f"{tag}_n_inter"])
    np.testing.assert_allclose(out.numpy(), g[f"{tag}_samples"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(inter["pred_x0"][-1].numpy(), g[f"{tag}_pred_x0_last"], rtol=0, atol=2e-5)


@pytest.mark.parametrize("name", ["mc64_T4", "mc64_T16", "mc128_T3"])
def test_unet_matches_reference(golden_dir, name):
    g = _load(golden_dir, f"unet_{name}.npz")
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    sd = synth.synth_state_dict(shapes, seed=3)
    with torch.no_grad():
        y = O.unet_forward(sd, torch.from_numpy(g["x"]), torch.from_numpy(g["t"]), torch.from_numpy(g["ctx"]).float(),
                           torch.from_numpy(g["fs"]))
    np.testing.assert_allclose(y.numpy(), g["y"], rtol=0, atol=5e-5)


def test_vae_decoder_matches_reference(golden_dir):
    g = _load(golden_dir, "vae_ch32.npz")
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    sd = {"decoder." + k: v for k, v in synth.synth_state_dict(shapes, seed=4).items()}
    sd.update({"post_quant_conv." + k: v for k, v in
               synth.synth_state_dict([("weight", (4, 4, 1, 1)), ("bias", (4,))], 4).items()})
    with torch.no_grad():
        y = O.vae_decode(sd, torch.from_numpy(g["z"]))
    np.testing.assert_allclose(y.numpy(), g["y"], rtol=0, atol=5e-5)


def _enc_sd(g):
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    sd = {"encoder." + k: v for k, v in synth.synth_state_dict(shapes, seed=14).items()}
    sd.update({"quant_conv." + k: v for k, v in synth.synth_state_dict([("weight", (8, 8, 1, 1)), ("bias", (8,))], 14).items()})
    return sd


def test_vae_encoder_matches_reference(golden_dir):
    """Encoder + quant_conv moments and the posterior sample of the unmodified reference (autoencoder.py:97-102,
    distributions.py:24-40)."""
    g = _load(golden_dir, "vae_enc_ch32.npz")
    sd = _enc_sd(g)
    with torch.no_grad():
        m = O.vae_encode_moments(sd, torch.from_numpy(g["x"]))
        z = O.posterior_sample(m, torch.from_numpy(g["noise"]))
    np.testing.assert_allclose(m.numpy(), g["moments"], rtol=0, atol=5e-5)
    np.testing.assert_allclose(z.numpy(), g["z"], rtol=0, atol=5e-5)


def test_resampler_matches_reference(golden_dir):
    """image_proj_model: Resampler.forward of the unmodified reference (resampler.py:96-145), reduced width, B=2."""
    g = _load(golden_dir, "resampler_d256.npz")
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    kw = json.loads(str(g["kwargs"]))
    sd = synth.synth_state_dict(shapes, seed=17)
    with torch.no_grad():
        y = O.resampler_forward(sd, torch.from_numpy(g["x"]), heads=kw["heads"], dim_head=kw["dim_head"])
    assert y.shape == (2, kw["num_queries"] * kw["video_length"], kw["output_dim"])
    np.testing.assert_allclose(y.numpy(), g["y"], rtol=0, atol=5e-5)


@pytest.mark.parametrize("tag,S,cfg_img", [("S5", 5, 2.5), ("S8", 8, None)])
def test_ddim_multicond_loop_matches_reference(golden_dir, tag, S, cfg_img):
    """Three-way CFG sampler: the unmodified lvdm/models/samplers/ddim_multiplecond.py on the toy denoiser."""
    g = _load(golden_dir, "ddim_multicond_small.npz")
    sched = O.model_schedule(base_scale=0.3)
    x_T = torch.from_numpy(g[f"{tag}_x_T"])
    noises = [torch.from_numpy(n) for n in g[f"{tag}_noises"]]
    cond = {"k": torch.tensor([1.3]), "b": torch.from_numpy(g[f"{tag}_cond_b"])}
    unc = {"k": torch.tensor([0.4]), "b": torch.from_numpy(g[f"{tag}_uncond_b"])}
    unc_img = {"k": torch.tensor([0.9]), "b": torch.from_numpy(g[f"{tag}_uncond_img_b"])}
    tab = O.ddim_tables(sched, S, "uniform_trailing", 1.0, fixed_prev_scale=False)
    assert np.array_equal(tab["scale_prev"].numpy(), g[f"{tag}_scale_prev"])           # the un-fixed [0] entry (ddim_multiplecond.py:33)
    out, inter = O.ddim_sample(_toy, sched, x_T.shape, S, cond, unc, x_T, noises, fixed_prev_scale=False, uncond_img=unc_img, cfg_img=cfg_img)
    assert len(inter["x_inter"]) == int(g[f"{tag}_n_inter"])
    np.testing.assert_allclose(out.numpy(), g[f"{tag}_samples"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(inter["pred_x0"][-1].numpy(), g[f"{tag}_pred_x0_last"], rtol=0, atol=2e-5)
