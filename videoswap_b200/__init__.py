"""videoswap_b200: H100-native (sm_90a) implementation of the denoising hot path of showlab/VideoSwap -- the
`AnimateDiffUNet3DModel` forward + classifier-free guidance + DDIM step -- behind the reference's own Python surface.
See DESIGN.md / INTEGRATION.md.  Importing this package never touches `oracle/` and there is no CPU fallback."""
from . import formats  # noqa: F401
from .pipeline import (SparsePointAdapter, TuneAVideoPipeline, TuneAVideoPipelineOutput, VideoSwapPipeline)  # noqa: F401
from .scheduler import DDIMInverseScheduler, DDIMScheduler  # noqa: F401
from .spec import UNetConfig, adapter_param_shapes, unet_param_shapes  # noqa: F401
from .unet import AnimateDiffUNet3DModel, UNet3DConditionModel, UNet3DConditionOutput  # noqa: F401
from .weights import seeded_state_dict  # noqa: F401

# Name -> class lookup, mirroring videoswap/utils/registry.py (MODEL_REGISTRY / PIPELINE_REGISTRY) of the reference.
MODEL_REGISTRY = {"AnimateDiffUNet3DModel": AnimateDiffUNet3DModel, "UNet3DConditionModel": AnimateDiffUNet3DModel,
                  "SparsePointAdapter": SparsePointAdapter}
PIPELINE_REGISTRY = {"VideoSwapPipeline": VideoSwapPipeline, "TuneAVideoPipeline": VideoSwapPipeline}


def build_model(name):
    return MODEL_REGISTRY[name]


def build_pipeline(name):
    return PIPELINE_REGISTRY[name]
