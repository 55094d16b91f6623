"""kukeon_b200 — H100-native (sm_90a) model-hub weight loader for kukeon (the package keeps its original name).

The product is `libkukeon_gpuload.so` (C ABI in include/kukeon_gpuload.h, sources in kukeon_b200/csrc).
`gpupool` is the ctypes binding (twin of the Go `internal/gpupool` cgo shim); `modelhub` mirrors the
`modelhub.Pull/Load/Mount` Go surface.  Importing this package does not load the native library; the
first call does, and fails loudly if it is missing — there is no CPU fallback.
"""
from . import gpupool, modelhub, registry, schema  # noqa: F401

__all__ = ["gpupool", "modelhub", "registry", "schema"]
