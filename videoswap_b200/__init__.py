"""videoswap_b200: H100-native (sm_90a) implementation of the denoising hot path of showlab/VideoSwap -- the
`AnimateDiffUNet3DModel` forward + classifier-free guidance + DDIM step, the CLIP text encoder of the prompts, the VAE
encode of the source frames, the VAE decode of the result, the DIFT features of tracked points and the propagation of
point drags through the layered atlas -- behind the reference's own Python surface.
See DESIGN.md / INTEGRATION.md.  Importing this package never touches `oracle/` and there is no CPU fallback."""
from . import formats  # noqa: F401
from .atlas import (IMLP_Hash, atlas_dims, init_atlas_model, process_displacement_propagation,  # noqa: F401
                    propagate_point_sequence)
from .dift import DIFT_Demo, SDFeaturizer, extract_point_embedding  # noqa: F401
from .pipeline import (SparsePointAdapter, TuneAVideoPipeline, TuneAVideoPipelineOutput, VideoSwapPipeline)  # noqa: F401
from .scheduler import DDIMInverseScheduler, DDIMScheduler  # noqa: F401
from .spec import (CLIPTextConfig, UNetConfig, VAEConfig, adapter_param_shapes, clip_text_param_shapes,  # noqa: F401
                   unet_param_shapes, vae_encoder_param_shapes, vae_param_shapes)
from .t2i_adapter import T2IAdapter, T2IAdapterConfig, t2i_adapter_param_shapes  # noqa: F401
from .text import CLIPTextModel, CLIPTextModelOutput  # noqa: F401
from .unet import AnimateDiffUNet3DModel, UNet3DConditionModel, UNet3DConditionOutput  # noqa: F401
from .vae import AutoencoderKL, AutoencoderKLOutput, DecoderOutput, DiagonalGaussianDistribution  # noqa: F401
from .weights import seeded_state_dict  # noqa: F401

# Name -> class lookup, mirroring videoswap/utils/registry.py (MODEL_REGISTRY / PIPELINE_REGISTRY) of the reference.
MODEL_REGISTRY = {"AnimateDiffUNet3DModel": AnimateDiffUNet3DModel, "UNet3DConditionModel": AnimateDiffUNet3DModel,
                  "SparsePointAdapter": SparsePointAdapter, "T2IAdapter": T2IAdapter}
PIPELINE_REGISTRY = {"VideoSwapPipeline": VideoSwapPipeline, "TuneAVideoPipeline": VideoSwapPipeline}


def build_model(name):
    return MODEL_REGISTRY[name]


def build_pipeline(name):
    return PIPELINE_REGISTRY[name]
