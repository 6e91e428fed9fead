"""Alias of ffn_b200.inference.resegmentation_analysis."""
import sys as _sys
from ffn_b200.inference import resegmentation_analysis as _impl
_sys.modules[__name__] = _impl
