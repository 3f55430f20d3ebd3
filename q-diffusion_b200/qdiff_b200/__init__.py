"""qdiff_b200: H100-native (sm_90a) drop-in for the `qdiff` package of Xiuyu-Li/q-diffusion (hot path only).

Exports mirror qdiff/__init__.py:1-5.  Compute lives in libqdiff_b200.so (sm_90a); importing this
package does not need a GPU, running a UNet does.
"""
from .adaptive_rounding import AdaRoundQuantizer
from .quant_block import BaseQuantBlock
from .quant_layer import QuantModule, UniformAffineQuantizer
from .quant_model import QuantModel
from .utils import convert_adaround, resume_cali_model

__all__ = ["AdaRoundQuantizer", "BaseQuantBlock", "QuantModule", "UniformAffineQuantizer", "QuantModel",
           "convert_adaround", "resume_cali_model"]
