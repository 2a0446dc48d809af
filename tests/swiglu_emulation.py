"""The emulation of tests/dinov2_emulation.py (DinoEmulation, f16 and FP8 forms) with SwiGLU MLPs (vitb200_arch.activation = 4), for
tests.

    swiglu  h = f16(silu(x1) * x2) in float64, x1 | x2 the two halves of fc1's output (its rows in HF's order), silu(x) = x / (1 + e^-x)

fc2 then reads h [T][F] as it reads the GELU output.  Every other activation is DinoEmulation's."""
import numpy as np

from tests.dinov2_emulation import DinoEmulation
from tests.fp8_reference import _f16


class SwigluEmulation(DinoEmulation):
    """DinoEmulation with the file's SwiGLU MLPs."""

    def _act(self, h):
        if self.activation != "swiglu":
            return super()._act(h)
        x1, x2 = np.split(np.asarray(h, np.float64), 2, axis=-1)
        with np.errstate(over="ignore"):
            return _f16(x1 / (1.0 + np.exp(-x1)) * x2)
