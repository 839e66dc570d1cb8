"""caffe_mpi_b200 -- H100-native (sm_90a) data-parallel hot path of Caffe-MPI.

The product is ``libb2c.so`` (CUDA kernels + the C ABI declared in ``include/b2c.h``) and the C++
host layer in ``host/`` that mirrors the reference's ``caffe::Blob / Layer / Net / Solver`` surface
for this path.  This Python package is only the loader and a thin ctypes binding used by the
tests and by ``bench.py``; PyTorch supplies device memory, streams and ``torch.distributed``
plumbing.  There is no CPU fallback: importing works without a GPU (so the symbol table can be
checked), but every compute entry point fails loudly when the extension or a device is missing.
"""
from . import capi  # noqa: F401
from .capi import B2CError, ConvParams, ConvDesc, lib  # noqa: F401

__all__ = ["capi", "B2CError", "ConvParams", "ConvDesc", "lib"]
