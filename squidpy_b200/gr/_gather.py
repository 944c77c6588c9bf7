"""A dense block gathered on the device from a device-resident expression matrix (``sqb_dense_gather_device``): the input of
``ligrec`` and ``sepal`` when ``X`` lives in GPU memory.  The caller's matrix is read in place and never copied to the host."""

from __future__ import annotations

import ctypes as C
from typing import Any

import numpy as np

from .._device import DevMatrix, array_device, device_matrix, matrix_args
from .._lib import Context, check, default_context, load, pointer_device

OBS_MAJOR, GENE_MAJOR = 0, 1  # layout: observations x genes (ligrec), genes x observations (sepal)
CODE_DTYPES = {0: np.float32, 1: np.float64, 2: np.float16, 3: np.int32, 4: np.int64}


def device_context(m: Any, device: int | None) -> tuple[DevMatrix, Context]:
    """Describe the device matrix ``m`` (observations x genes of ``m.shape``) and the context on its device; ``device`` (or
    ``None``) must name that device."""
    d = device_matrix(m)
    on = array_device(d, pointer_device)
    if device is not None and int(device) != on:
        raise ValueError(f"`device={device}` does not match the device of the expression matrix, cuda:{on}.")
    return matrix_args(d, d.shape), default_context(on)


class Gathered:
    """``rows`` (ascending, or ``None`` for all) x ``cols`` (input column of every output column) of ``m``, gathered on the
    device in ``layout``, as float64 or in the input's own dtype; NaN written as 0 with ``nan_zero``."""

    def __init__(self, ctx: Context, m: DevMatrix, rows: np.ndarray | None, cols: np.ndarray, layout: int, *, nan_zero: bool,
                 keep_dtype: bool = False):
        self._lib = load()
        self.ctx = ctx
        r = None if rows is None else np.ascontiguousarray(rows, dtype=np.int64)
        c = np.ascontiguousarray(cols, dtype=np.int32)
        self.n_obs = m.shape[0] if r is None else int(r.size)
        self.n_genes = int(c.size)
        self.layout = layout
        self.dtype = np.dtype(CODE_DTYPES[m.code] if keep_dtype else np.float64)
        h = C.c_void_p()
        check(self._lib.sqb_dense_gather_device(ctx.handle, m.format, m.x, m.indptr, m.indptr_bits, m.indices, m.index_bits, m.nnz, m.code,
                                                m.shape[0], m.shape[1], m.strides[0], m.strides[1], None if r is None else r.ctypes.data,
                                                self.n_obs, c.ctypes.data, self.n_genes, layout, int(nan_zero) | (2 if keep_dtype else 0),
                                                m.stream, C.byref(h)))
        self._h = h

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    @property
    def shape(self) -> tuple[int, int]:
        return (self.n_obs, self.n_genes) if self.layout == OBS_MAJOR else (self.n_genes, self.n_obs)

    def download(self) -> np.ndarray:
        out = np.empty(self.shape, dtype=self.dtype)
        check(self._lib.sqb_dense_download(self._h, out.ctypes.data))
        return out

    def close(self) -> None:
        if self._h is not None:
            self._lib.sqb_dense_free(self._h)
            self._h = None

    def __enter__(self) -> Gathered:
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass
