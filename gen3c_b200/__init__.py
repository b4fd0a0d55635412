"""gen3c_b200 — Hopper-native (sm_90a, H100) engine for GEN3C's two hot paths.

Path R (3D-cache render): ``gen3c_b200.warp`` / ``gen3c_b200.cache_3d``
Path D (7B DiT denoise step): ``gen3c_b200.dit`` / ``gen3c_b200.sampler`` / ``gen3c_b200.ops``
All compute lives in ``lib/libgen3c_b200.so`` (C ABI: ``include/gen3c_b200.h``); there is no CPU path.
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
__version__ = "0.1.0"
