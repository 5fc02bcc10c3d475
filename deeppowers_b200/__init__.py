"""deeppowers_b200 — H100-native FHE ciphertext arithmetic behind a C ABI (include/dpfhe.h).

The package holds only what the hot path needs: csrc/ (sm_90a kernels + the extern "C" ABI),
the in-tree build, the ctypes loader and a thin host-side mirror of the C++ wrapper.
"""
from .evaluator import Context, DpfheError, LinearLayer, MultiContext, PinnedBuffer, PolyEval, SlotSum, linear_bsgs_grouped, pinned_empty, public_seed, slotsum_steps  # noqa: F401
from ._lib import load as load_library, so_path  # noqa: F401
from .build import build as build_library  # noqa: F401

__all__ = ["Context", "DpfheError", "LinearLayer", "MultiContext", "PinnedBuffer", "PolyEval", "SlotSum", "linear_bsgs_grouped", "pinned_empty", "public_seed", "slotsum_steps", "load_library", "so_path", "build_library"]
