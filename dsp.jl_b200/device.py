"""Device-resident arrays for pipelines (conv -> welch_pgram ...) that should not bounce through host memory.

`to_device(x)` copies a numpy array to HBM once; every front end of this package that receives a `DeviceArray`
runs the `*_exec_dev` entry point on it and returns a `DeviceArray` (array results) or host numpy (small results:
periodogram power).  This is the analogue of handing CuArrays to the Julia glue; the reference itself has no
device notion.  Memory comes from the library's own allocator (`dspb200_malloc`), so no other CUDA binding is needed.
"""
import ctypes as C

import numpy as np

from . import _lib


# freed blocks are kept for reuse (cudaMalloc / cudaFree of half-gigabyte buffers cost milliseconds and synchronise)
_POOL = {}
_POOL_BYTES = [0]
_POOL_LIMIT = 16 << 30


def _alloc(nbytes):
    lst = _POOL.get(nbytes)
    if lst:
        _POOL_BYTES[0] -= nbytes
        return lst.pop()
    p = C.c_void_p(None)
    _lib.check(_lib.lib.dspb200_malloc(C.byref(p), nbytes))
    return p.value


def _release(ptr, nbytes):
    if _POOL_BYTES[0] + nbytes <= _POOL_LIMIT:
        _POOL.setdefault(nbytes, []).append(ptr)
        _POOL_BYTES[0] += nbytes
    else:
        _lib.lib.dspb200_free(ptr)


def empty_cache():
    """Return every cached block to the driver."""
    for lst in _POOL.values():
        for ptr in lst:
            _lib.lib.dspb200_free(ptr)
    _POOL.clear()
    _POOL_BYTES[0] = 0


class DeviceArray:
    """Column-major (time-fastest) device array: `shape` follows numpy semantics of the host mirror (axis 0 = time)."""

    def __init__(self, shape, dtype, _base=None, _ptr=None):
        self.shape = tuple(int(v) for v in shape)
        self.dtype = np.dtype(dtype)
        _lib.np_dtype_code(self.dtype)
        self.size = int(np.prod(self.shape)) if self.shape else 1
        self.nbytes = self.size * self.dtype.itemsize
        self._base = _base
        if _ptr is None:
            self._alloc_bytes = max(self.nbytes, 16)
            self.ptr = _alloc(self._alloc_bytes)
            self._owner = True
        else:
            self.ptr = int(_ptr)
            self._owner = False

    @property
    def ndim(self):
        return len(self.shape)

    def __len__(self):
        return self.shape[0]

    def __getitem__(self, key):
        """Contiguous slices along time of a 1-D array (views, no copy): d[a:b]."""
        if self.ndim != 1 or not isinstance(key, slice) or key.step not in (None, 1):
            raise IndexError("DeviceArray supports d[a:b] on vectors only")
        a, b, _ = key.indices(self.shape[0])
        b = max(a, b)
        return DeviceArray((b - a,), self.dtype, _base=self, _ptr=self.ptr + a * self.dtype.itemsize)

    def overlaps(self, other):
        """True when `other` (a DeviceArray, or None) shares at least one byte of device memory with this array."""
        return (other is not None and self.nbytes > 0 and other.nbytes > 0 and self.ptr < other.ptr + other.nbytes
                and other.ptr < self.ptr + self.nbytes)

    def to_host(self, out=None):
        """Copy back to a (Fortran-ordered for 2-D) numpy array."""
        if out is None:
            out = np.empty(self.shape, dtype=self.dtype, order="F")
        if self.nbytes:
            _lib.check(_lib.lib.dspb200_memcpy_d2h(_lib.ptr(out), self.ptr, self.nbytes, None))
            _lib.check(_lib.lib.dspb200_stream_sync(None))
        return out

    def copy_from_host(self, x):
        x = np.asfortranarray(x, dtype=self.dtype)
        if x.size != self.size:
            raise ValueError("size mismatch")
        if self.nbytes:
            _lib.check(_lib.lib.dspb200_memcpy_h2d(self.ptr, _lib.ptr(x), self.nbytes, None))
            _lib.check(_lib.lib.dspb200_stream_sync(None))
        return self

    def copy_from_host_ptr(self, host_ptr, nbytes):
        """H2D from a raw (ideally pinned) host pointer, e.g. a torch pinned tensor's data_ptr()."""
        if nbytes > self.nbytes:
            raise ValueError("size mismatch")
        _lib.check(_lib.lib.dspb200_memcpy_h2d(self.ptr, host_ptr, nbytes, None))
        _lib.check(_lib.lib.dspb200_stream_sync(None))
        return self

    def __del__(self):
        try:
            if getattr(self, "_owner", False) and self.ptr:
                _release(self.ptr, self._alloc_bytes)
                self.ptr = 0
        except Exception:
            pass


def to_device(x):
    """Copy a numpy array (float32/float64/complex64/complex128; integers are promoted to float64) to the GPU."""
    x = np.asarray(x)
    if x.dtype.kind in "biu":
        x = x.astype(np.float64)
    d = DeviceArray(x.shape, x.dtype)
    return d.copy_from_host(x)


def to_host(d):
    return d.to_host() if isinstance(d, DeviceArray) else np.asarray(d)


def sync():
    _lib.check(_lib.lib.dspb200_stream_sync(None))
