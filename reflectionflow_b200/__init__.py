"""reflectionflow_b200 — H100-native (sm_90a) FLUX.1-dev DiT hot path of
Diffusion-CoT/ReflectionFlow behind the reference's own call surface.

Layers (top to bottom):
  tts/            outer search loop (noise scaling, reflection rounds), verifier hooks, sharding
  pipeline.py     B200FluxPipeline.__call__ / generate()  (diffusers FluxPipeline surface)
  transformer.py  B200FluxTransformer2DModel.forward / tranformer_forward()
  _lib.py         ctypes binding of librf_b200.so (C ABI, include/rf_b200.h)
  csrc/           hand-written CUDA: wgmma GEMM, wgmma attention, bandwidth kernels, orchestrator
"""
from .config import FluxDiTConfig  # noqa: F401

__version__ = "0.1.0"
