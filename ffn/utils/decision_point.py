"""Alias of ffn_b200.utils.decision_point."""
import sys as _sys
from ffn_b200.utils import decision_point as _impl
_sys.modules[__name__] = _impl
