from editanything_b200.pipeline import (StableDiffusionControlNetInpaintMixingPipeline,  # noqa: F401
                                        StableDiffusionControlNetInpaintPipeline, StableDiffusionPipelineOutput,
                                        prepare_controlnet_conditioning_image, prepare_image, prepare_mask_image)
