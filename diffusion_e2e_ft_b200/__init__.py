"""diffusion_e2e_ft_b200 — H100-native single-step denoising engine (UNet2DConditionModel + AutoencoderKL
hot path of VisualComputingInstitute/diffusion-e2e-ft) behind the reference's module / pipeline API.

    from diffusion_e2e_ft_b200 import B200UNet2DConditionModel, B200AutoencoderKL, MarigoldPipeline

Arithmetic lives in libb200_e2eft.so (hand-written sm_90a CUDA, C ABI in include/b200_e2eft.h).
"""
from .lib import load as load_library, LIB_PATH, EXPORTS  # noqa: F401
from .unet import B200UNet2DConditionModel, UNet2DConditionOutput  # noqa: F401
from .vae import B200AutoencoderKL  # noqa: F401
from .pipelines import (DDIMScheduler, MarigoldPipeline, MarigoldDepthOutput,  # noqa: F401
                        DepthNormalEstimationPipeline, DepthNormalPipelineOutput, pyramid_noise_like)
from .clip_text import B200CLIPTextModel, EmptyPromptTokenizer  # noqa: F401
from .clip_vision import B200CLIPVisionModelWithProjection, CLIPImageProcessorConfig  # noqa: F401
from .ensemble import ensemble_normals, ensemble_normals_with_index, ensemble_depths  # noqa: F401

__version__ = "0.1.0"
