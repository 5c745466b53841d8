"""quantized_distillation_b200 -- H100 (sm_90a) implementation of the
fake-quantization hot path of antspy/quantized_distillation.

    from quantized_distillation_b200 import quantization        # same names as the reference package
    quantized_distillation_b200.install_as_quantization()       # or: make `import quantization` resolve here

See DESIGN.md for the kernels and INTEGRATION.md for the drop-in recipe.
"""
import sys

from . import quantization  # noqa: F401
from .plan import QuantizationPlan  # noqa: F401

__version__ = "0.1.0"


def install_as_quantization() -> None:
    """Registers this package's ``quantization`` under the reference's top-level
    module name, so unmodified reference code (``import quantization``,
    ``import quantization.help_functions as qhf``) runs on the CUDA kernels."""
    sys.modules["quantization"] = quantization
    sys.modules["quantization.quant_functions"] = quantization.quant_functions
    sys.modules["quantization.help_functions"] = quantization.help_functions
