"""Alias of ffn_b200.inference.consensus_pb2."""
import sys as _sys
from ffn_b200.inference import consensus_pb2 as _impl
_sys.modules[__name__] = _impl
