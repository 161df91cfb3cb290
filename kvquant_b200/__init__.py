"""kvquant_b200 -- H100-native (sm_90a) implementation of the KVQuant deployment hot path.

Layout
  csrc/            hand-written CUDA kernels + the C ABI (include/kvquant_b200.h)
  _lib.py          ctypes binding (no fallback: raises if libkvquant_b200.so is missing)
  quant_cuda.py    the reference's 34-op `quant_cuda` Python surface on top of the C ABI
  cache.py         QuantK / QuantV mirrors of the reference's cache managers + the native fused layer cache
  decode.py        LLaMA-shaped decode harness and the layer-group pipeline (NCCL P2P of the hidden vector)
  synth.py         synthetic activations / calibration artefacts (no weights or datasets offline)
"""
__version__ = "0.1.0"
