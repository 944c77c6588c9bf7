"""Device attributes the GPU tests use to decide which side of a kernel's dispatch rule a case lands on.

The library picks code paths from the per-block opt-in shared-memory limit (``sqb_ctx::smem_optin``, from
``cudaDeviceProp::sharedMemPerBlockOptin``).  The tests read the same attribute through the CUDA runtime that is already
loaded by the library (and by torch), so that a case written for one branch can assert that it really takes it."""

from __future__ import annotations

import ctypes

H100_SMEM_OPTIN = 232448  # bytes: 227 KB per block on sm_90
_CUDA_DEV_ATTR_MAX_SHARED_MEMORY_PER_BLOCK_OPTIN = 97  # cudaDevAttrMaxSharedMemoryPerBlockOptin
_CUDA_DEV_ATTR_MULTIPROCESSOR_COUNT = 16  # cudaDevAttrMultiProcessorCount


def _attr(attr: int, device: int) -> int:
    from squidpy_b200 import _lib

    _lib.load()  # links libcudart.so.12: the name below resolves to the runtime already in the process
    rt = ctypes.CDLL("libcudart.so.12")
    v = ctypes.c_int(0)
    rc = rt.cudaDeviceGetAttribute(ctypes.byref(v), attr, int(device))
    if rc != 0:
        raise RuntimeError(f"cudaDeviceGetAttribute failed with cudaError {rc}")
    return v.value


def smem_optin(device: int = 0) -> int:
    """``cudaDeviceGetAttribute(cudaDevAttrMaxSharedMemoryPerBlockOptin, device)``."""
    return _attr(_CUDA_DEV_ATTR_MAX_SHARED_MEMORY_PER_BLOCK_OPTIN, device)


def sm_count(device: int = 0) -> int:
    """``cudaDeviceGetAttribute(cudaDevAttrMultiProcessorCount, device)``: the library launches per-SM CTA counts from it."""
    return _attr(_CUDA_DEV_ATTR_MULTIPROCESSOR_COUNT, device)
