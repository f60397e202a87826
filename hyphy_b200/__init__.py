"""hyphy_b200 -- GPU-native (H100) phylogenetic-likelihood engine (drop-in for HyPhy's ComputeBlock hot path).

The product is libhyphy_b200.so (C ABI in include/hyphy_b200.h, CUDA sm_90a kernels in hyphy_b200/csrc).
This package is the thin host-side mirror used by tests and bench.py; it never computes likelihoods on the CPU."""
from .engine import EngineError, Partition, LikelihoodFunction, load_library, device_count  # noqa: F401

__all__ = ["EngineError", "Partition", "LikelihoodFunction", "load_library", "device_count"]
