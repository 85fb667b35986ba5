"""viewcrafter_b200: H100-native (sm_90a) implementation of ViewCrafter's DDIM-denoise hot path.

Drop-in classes (same names / constructor kwargs / state-dict keys as the reference):
    viewcrafter_b200.unet.UNetModel             <- lvdm.modules.networks.openaimodel3d.UNetModel
    viewcrafter_b200.autoencoder.AutoencoderKL  <- lvdm.models.autoencoder.AutoencoderKL
    viewcrafter_b200.ddim.DDIMSampler           <- lvdm.models.samplers.ddim.DDIMSampler
    viewcrafter_b200.ddim_multiplecond.DDIMSampler <- lvdm.models.samplers.ddim_multiplecond.DDIMSampler
    viewcrafter_b200.resampler.Resampler        <- lvdm.modules.encoders.resampler.Resampler
    viewcrafter_b200.synthesis.image_guided_synthesis / get_latent_z <- utils.diffusion_utils (same names)
Added samplers (opt-in; DDIM stays the default):
    viewcrafter_b200.dpm_solver.DPMSolverSampler / DPMSolverSamplerMultiCond: DPM-Solver++(2M), image_guided_synthesis(sampler="dpmpp_2m")
    viewcrafter_b200.dpm_solver.DPMSolver3MSDESampler / DPMSolver3MSDESamplerMultiCond: DPM-Solver++(3M) SDE (eta = 1),
        image_guided_synthesis(sampler="dpmpp_3m_sde")
    viewcrafter_b200.fifo.FIFOSampler / FIFOSamplerMultiCond: FIFO-Diffusion diagonal denoising, clips of any length at the memory
        of one window, image_guided_synthesis(fifo=f)
All tensor work runs in libvc_b200.so (hand-written CUDA for sm_90a, C ABI in include/vc_b200.h).

set_reproducible(on) / VC_REPRODUCIBLE=1: reproducible mode (bit-identical results across batching, GPU count and SM count).
"""
__version__ = "0.1.0"

from .ops import reproducible, set_reproducible  # noqa: E402,F401
