"""crabml_b200 -- H100-native CUDA backend for crabml's quantized decode path.

The product is the C-ABI shared library (include/crabml_cuda.h -> crabml_b200/lib/libcrabml_cuda.so).
This Python package is a thin ctypes binding used by tests/ and bench.py; it mirrors the reference's
`Tensor` trait (crabml-core/src/tensor/api.rs:11-79).  There is no CPU fallback: importing works on a
CPU-only box (so the symbol table can be checked) but creating a device fails loudly without CUDA.
"""
from .capi import load_library, CudaError, TensorError  # noqa: F401
from .tensor import CudaTensor, CudaTensorDevice, TensorStrider  # noqa: F401
