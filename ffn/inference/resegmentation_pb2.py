"""Alias of ffn_b200.inference.resegmentation_pb2."""
import sys as _sys
from ffn_b200.inference import resegmentation_pb2 as _impl
_sys.modules[__name__] = _impl
