"""jax.random (0.2.8, threefry2x32) subset used by the hot path, host side backed by libsmd.

Keys are numpy uint32[2] arrays exactly like ``jax.random.PRNGKey``; ``split`` runs the C++ host threefry in
libsmd (smd_threefry_split); ``normal`` / ``uniform`` generate on the GPU (smd_threefry_normal / _uniform)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import lib as _lib


def PRNGKey(seed: int) -> np.ndarray:
    seed = int(seed)
    return np.array([(seed >> 32) & 0xFFFFFFFF, seed & 0xFFFFFFFF], dtype=np.uint32)


def split(key, num: int = 2) -> np.ndarray:
    lib = _lib.load_library()
    k = (C.c_uint32 * 2)(int(key[0]), int(key[1]))
    out = (C.c_uint32 * (2 * num))()
    _lib.check(lib.smd_threefry_split(k, int(num), out))
    return np.array(list(out), dtype=np.uint32).reshape(num, 2)


def normal(key, shape, device=None, rows=None) -> torch.Tensor:
    """jax.random.normal(key, shape).  ``rows=(first, count)`` returns only rows [first, first + count) of the
    leading axis (a data-parallel rank's slice of the global draw; threefry is counter based)."""
    lib = _lib.load_library()
    shape = tuple(int(s) for s in shape)
    total = int(np.prod(shape))
    k = (C.c_uint32 * 2)(int(key[0]), int(key[1]))
    st = torch.cuda.current_stream().cuda_stream
    if rows is None:
        out = torch.empty(shape, dtype=torch.float32, device=device or "cuda")
        _lib.check(lib.smd_threefry_normal(k, out.data_ptr(), total, st))
        return out
    first, count = int(rows[0]), int(rows[1])
    per = total // shape[0]
    out = torch.empty((count,) + shape[1:], dtype=torch.float32, device=device or "cuda")
    _lib.check(lib.smd_threefry_normal_slice(k, out.data_ptr(), count * per, first * per, total, st))
    return out


def uniform(key, shape, minval: float = 0.0, maxval: float = 1.0, device=None, rows=None) -> torch.Tensor:
    """jax.random.uniform(key, shape, minval=minval, maxval=maxval).  ``rows=(first, count)`` as in ``normal``."""
    lib = _lib.load_library()
    shape = tuple(int(s) for s in shape)
    total = int(np.prod(shape))
    k = (C.c_uint32 * 2)(int(key[0]), int(key[1]))
    st = torch.cuda.current_stream().cuda_stream
    if rows is None:
        out = torch.empty(shape, dtype=torch.float32, device=device or "cuda")
        _lib.check(lib.smd_threefry_uniform(k, out.data_ptr(), total, C.c_float(minval), C.c_float(maxval), st))
        return out
    first, count = int(rows[0]), int(rows[1])
    per = total // shape[0]
    out = torch.empty((count,) + shape[1:], dtype=torch.float32, device=device or "cuda")
    _lib.check(lib.smd_threefry_uniform_slice(k, out.data_ptr(), count * per, first * per, total, C.c_float(minval),
                                              C.c_float(maxval), st))
    return out
