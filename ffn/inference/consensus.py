"""Alias of ffn_b200.inference.consensus."""
import sys as _sys
from ffn_b200.inference import consensus as _impl
_sys.modules[__name__] = _impl
