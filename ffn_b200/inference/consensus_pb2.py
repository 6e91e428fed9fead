"""Drop-in for ffn/inference/consensus_pb2.py (runtime-built descriptors, see protos.py)."""
from .protos import ConsensusRequest  # noqa: F401
