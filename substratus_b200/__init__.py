"""substratus_b200 — H100-native engine for the Substratus ``Server`` CRD's serving container.

Only what the Server-CRD inference hot path needs (SURVEY.md §8): ``csrc/`` (sm_90a CUDA
kernels + the C ABI of ``include/ssb.h``), ``engine.py`` (ctypes mirror of the serve host's
view) and the serve host under ``host/``.  No CPU fallback.
"""
from .engine import Engine, SsbError, load_library, synth_fill_host  # noqa: F401

__all__ = ["Engine", "SsbError", "load_library", "synth_fill_host"]
