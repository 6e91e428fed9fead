"""Import-compatibility shim: `ffn.inference.*`, `ffn.utils.*_pb2`, `ffn.training.model(s)` resolve
to the GPU-native implementations in `ffn_b200` so code written against google/ffn's inference
API (run_inference.py, notebooks constructing Runner / Canvas) runs unchanged."""
