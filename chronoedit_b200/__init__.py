"""chronoedit_b200 — H100-native (sm_90a) implementation of the ChronoEdit denoising hot path.

Public surface (drop-in for the objects `ChronoEditPipeline` registers, pipeline_chronoedit.py:175-183):
  ChronoEditTransformer3DModel   <- chronoedit_diffusers/transformer_chronoedit.py:298-476
  AutoencoderKLWan               <- diffusers AutoencoderKLWan (arithmetic twin: chronoedit/_src/tokenizers/wan2pt1.py)
  FlowUniPCMultistepScheduler    <- chronoedit/_src/models/fm_solvers_unipc.py (the per-step glue either side of the DiT call)
  UMT5EncoderModel, CLIPVisionModel <- the transformers classes the pipeline runs once per edit (pipeline_chronoedit.py:205-254)
All call hand-written CUDA kernels in lib/libchronoedit_b200.so through the C ABI of include/chronoedit_b200.h.
Importing this package does not need a GPU; running anything does (there is no CPU fallback).
"""
from ._lib import CEError, LIB_PATH, lib  # noqa: F401
from .autoencoder import AutoencoderKLWan  # noqa: F401
from .encoders import CLIPVisionModel, UMT5EncoderModel  # noqa: F401
from .scheduler import FlowUniPCMultistepScheduler  # noqa: F401
from .transformer import ChronoEditTransformer3DModel, Transformer2DModelOutput  # noqa: F401

__all__ = ["ChronoEditTransformer3DModel", "Transformer2DModelOutput", "AutoencoderKLWan", "FlowUniPCMultistepScheduler",
           "UMT5EncoderModel", "CLIPVisionModel", "CEError", "lib", "LIB_PATH"]
