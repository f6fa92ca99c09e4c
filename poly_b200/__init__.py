"""poly_b200 -- H100 (sm_90a) implementation of bebop/poly's search/mash sketching
hot path plus the secondary search/align Smith-Waterman scorer and primers SantaLucia
Tm kernels.  Host-side mirrors of the reference's Go API live in mash / align /
primers; all compute happens in libpolyb200.so (hand-written CUDA, C ABI in
include/poly_b200.h)."""
from . import _lib  # noqa: F401

__all__ = ["mash", "align", "primers", "synth"]
__version__ = "0.1.0"
