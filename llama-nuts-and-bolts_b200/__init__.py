"""llama-nuts-and-bolts_b200 -- H100 (sm_90a) forward path behind the Go API of
adalkiran/llama-nuts-and-bolts.

Layout
  csrc/        CUDA kernels + the C-ABI (include/lnb.h) -> liblnb.so
  _capi.py     ctypes binding of every lnb_* symbol
  ml.py        host mirror of the reference's src/ml  (Tensor, LinearTransformation, MatMul, ...)
  model.py     host mirror of src/model               (ModelArgs, LlamaTransformer, InferenceContext)
  inference.py host mirror of src/inference           (InferenceEngine generate loop)
  synth.py     synthetic 8B checkpoint description (no real checkpoint exists offline)

The Go toolchain is absent from the build image, so this Python layer plays the role of the
cgo shims (INTEGRATION.md shows the Go side).  There is NO CPU fallback: importing the
package fails loudly if liblnb.so is missing, and every op raises if CUDA is unavailable.
"""
from . import _capi  # noqa: F401  (loads liblnb.so or raises)
from . import ml, model, inference, synth, torch_reader, vocabulary  # noqa: F401

__all__ = ["ml", "model", "inference", "synth", "_capi"]
