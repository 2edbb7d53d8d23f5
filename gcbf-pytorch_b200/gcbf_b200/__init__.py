"""gcbf_b200 -- H100-native (sm_90a) implementation of the gcbf-pytorch hot path.

Mirrors the reference package layout (`gcbf.nn`, `gcbf.controller`, `gcbf.algo`, `gcbf.env`) with the same class
names, constructor signatures, forward signatures and state-dict keys; the arithmetic runs in the hand-written
CUDA kernels of libgcbf_b200.so (see include/gcbf_b200.h).  Importing the package does not load the shared
library; the first CUDA op does, and fails loudly if it is missing (there is no CPU fallback).

`gcbf-pytorch_b200/dropin/` holds a `gcbf` alias package so that `from gcbf.nn import MLP` style imports of the
reference's trainer / scripts resolve to this implementation.
"""
__version__ = '0.1.0'
