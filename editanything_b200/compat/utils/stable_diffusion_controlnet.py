from editanything_b200.loading import ControlNetModel, ControlNetModel2  # noqa: F401
from editanything_b200.pipeline import StableDiffusionControlNetPipeline2  # noqa: F401  (sketch2image.py:21)
