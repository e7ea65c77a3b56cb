"""scenelib2_b200 — H100-native (sm_90a) implementation of the SceneLib2 EKF-MonoSLAM hot path.

Layout (hot path only, see DESIGN.md):
  csrc/      CUDA kernels + the C ABI (libsl2b200.so, declared in include/sl2b200.h)
  host/      C++ shim keeping the MonoSLAM / Kalman / Feature class surface over the C ABI
  lib.py     ctypes mirror of the C ABI (used by tests, bench.py and the smoke entry)
  synth.py   deterministic synthetic inputs for BASELINE configs C1..C5
"""
from . import synth  # noqa: F401
from .lib import Context, Sl2Config, Sl2Error, config_for_scene, default_config, load, load_scene  # noqa: F401

__all__ = ["synth", "Context", "Sl2Config", "Sl2Error", "config_for_scene", "default_config",
           "load", "load_scene"]
