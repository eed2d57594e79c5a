"""hanabi_b200 — H100-native particle simulation backend behind Hanabi's authoring API.

The package is a binding over ``libhanabi_b200.so`` (C ABI in ``include/hanabi_b200.h``); importing it
fails loudly when the native library has not been built. There is no CPU execution path.
"""
from . import _native  # noqa: F401  (raises ImportError if the library is missing)
from ._native import HanabiError  # noqa: F401
from .runtime import Context, LoweredEffect, AttrField  # noqa: F401

__all__ = ["Context", "LoweredEffect", "AttrField", "HanabiError"]
