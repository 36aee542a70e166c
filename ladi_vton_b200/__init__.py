"""ladi_vton_b200 -- H100-native (sm_90a) engine for the LaDI-VTON try-on inference path.

Public surface mirrors the reference (miccunifi/ladi-vton): `StableDiffusionTryOnePipeline` (src/vto_pipelines/tryon_pipe.py),
`StableDiffusionInpaintPipeline` (diffusers 0.14, what src/train_inversion_adapter.py validates with),
`AutoencoderKL` (src/models/AutoencoderKL.py), `EMASC` (src/models/emasc.py), `UNet2DConditionModel` + `DDIMScheduler`
(diffusers 0.14, built in hubconf.py / src/inference.py), the hub constructors (`hub.py` <- hubconf.py) and the conditioning front-end
(`clip.py` <- src/utils/encode_text_word_embedding.py, the CLIP towers of src/inference.py:126-138,269-293).  All arithmetic runs in libladi_b200.so (include/ladi_b200.h);
there is no CPU or library fallback.
"""
from .adapter import InversionAdapter  # noqa: F401
from .clip import CLIPTextModel, CLIPVisionModel, CLIPVisionModelWithProjection, encode_text_word_embedding  # noqa: F401
from .pipeline import StableDiffusionInpaintPipeline, StableDiffusionPipelineOutput, StableDiffusionTryOnePipeline  # noqa: F401
from .scheduler import DDIMScheduler  # noqa: F401
from .unet import UNet2DConditionModel, unet_param_shapes  # noqa: F401
from .vae import EMASC, AutoencoderKL, vae_param_shapes  # noqa: F401
from .vgg import VGG19, VGGLoss  # noqa: F401
from .warp import ConvNet_TPS, UNetVanilla, generate_warped_cloth  # noqa: F401
