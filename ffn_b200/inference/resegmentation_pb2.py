"""Drop-in for ffn/inference/resegmentation_pb2.py (runtime-built descriptors, see protos.py).

`EndpointSegmentationResult` is the name resegmentation_analysis.py:118 uses for the message that
resegmentation.proto:22 calls `EndpointResegmentationResult`; both names are the same class.
"""
from .protos import EndpointResegmentationResult, PairResegmentationResult  # noqa: F401

EndpointSegmentationResult = EndpointResegmentationResult
