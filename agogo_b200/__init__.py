"""agogo_b200 — H100-native AlphaZero self-play engine behind gorgonia/agogo's API.

The compute lives in agogo_b200/libagogo_b200.so (hand-written sm_90a CUDA behind the C ABI of
include/agogo_b200.h).  There is no CPU fallback: loading the engine without the built library,
or creating an engine without a CUDA device, raises.
"""
from . import _capi  # noqa: F401
from ._capi import load, make_desc  # noqa: F401
