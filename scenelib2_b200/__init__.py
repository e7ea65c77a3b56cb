"""scenelib2_b200 — H100-native (sm_90a) implementation of the SceneLib2 EKF-MonoSLAM hot path.

Layout (hot path only, see DESIGN.md):
  csrc/      CUDA kernels + the C ABI (libsl2b200.so, declared in include/sl2b200.h)
  host/      C++ shim keeping the MonoSLAM / Kalman / Feature class surface over the C ABI
  lib.py     ctypes mirror of the C ABI (used by tests, bench.py and the smoke entry)
  synth.py   deterministic synthetic inputs for BASELINE configs C1..C5
"""
from . import synth  # noqa: F401
from .lib import (STEP_RECORD_DTYPE, Context, Sl2Config, Sl2Error, Sl2SnapshotHeader, Sl2StepRecord,  # noqa: F401
                  Sl2StreamConfig, Sl2StreamSource, config_for_scene, default_config, load, load_scene, read_snapshot,
                  stream_config_for_scene)

__all__ = ["synth", "STEP_RECORD_DTYPE", "Context", "Sl2Config", "Sl2Error", "Sl2SnapshotHeader", "Sl2StepRecord",
           "Sl2StreamConfig", "Sl2StreamSource", "config_for_scene", "default_config", "load", "load_scene", "read_snapshot",
           "stream_config_for_scene"]
