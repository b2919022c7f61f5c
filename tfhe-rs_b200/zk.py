"""Host-side mirror of tfhe-zk-pok's GPU MSM callers (``tfhe-zk-pok/src/gpu/
mod.rs``) over the zk-cuda-backend C ABI of include/tfhe_b200_zk.h.

  g1_msm_gpu / g2_msm_gpu      tfhe-zk-pok/src/gpu/mod.rs: the managed call on
                               a fresh stream, points in normal form, the result
                               normalized on the host; the identity is None
  msm_managed                  g{1,2}_msm_managed_wrapper, raw Montgomery result
  msm_device                   g{1,2}_msm_unmanaged_wrapper_async on torch
                               tensors and a gpu.CudaStreams stream, with
                               scratch sized by pippenger_scratch_size_g{1,2}

Arrays use the ABI layout.  A G1 point is G1_DTYPE (x, y: 7 x u64, infinity;
120 bytes), a G2 point G2_DTYPE (x, y: 2 x 7 x u64; 232 bytes), a scalar 5 x
u64 (any value below 2^320).  Field elements are little-endian limbs; the
MSMs take points in Montgomery form (R = 2^448) unless `points_in_montgomery`
is False on the managed call.  Arguments are checked before any GPU work and
bad ones raise ValueError.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import _lib

G1_DTYPE = np.dtype({"names": ["x", "y", "infinity"], "formats": [("<u8", (7,)), ("<u8", (7,)), "?"],
                     "offsets": [0, 56, 112], "itemsize": 120})
G2_DTYPE = np.dtype({"names": ["x", "y", "infinity"], "formats": [("<u8", (2, 7)), ("<u8", (2, 7)), "?"],
                     "offsets": [0, 112, 224], "itemsize": 232})
# homogeneous projective results: (X, Y, Z)
G1_PROJ_SHAPE, G2_PROJ_SHAPE = (3, 7), (3, 2, 7)
SCALAR_BITS = 320
_MASK = (1 << 64) - 1


class _Group:
    def __init__(self, name, dtype, proj_shape, degree):
        self.name, self.dtype, self.proj_shape, self.degree = name, dtype, proj_shape, degree

    def fn(self, pattern):
        return getattr(_lib.lib(), pattern.format(g=self.name))


G1 = _Group("g1", G1_DTYPE, G1_PROJ_SHAPE, 1)
G2 = _Group("g2", G2_DTYPE, G2_PROJ_SHAPE, 2)


def _group(group) -> _Group:
    if group in (G1, "g1", 1):
        return G1
    if group in (G2, "g2", 2):
        return G2
    raise ValueError(f"unknown group {group!r} (G1 or G2)")


# ---- Python integers <-> ABI arrays ----

def int_to_limbs(v: int, n: int = 7) -> np.ndarray:
    if not 0 <= v < 1 << (64 * n):
        raise ValueError(f"{v} does not fit {n} x u64 limbs")
    return np.array([(v >> (64 * i)) & _MASK for i in range(n)], dtype=np.uint64)


def limbs_to_int(a) -> int:
    return sum(int(w) << (64 * i) for i, w in enumerate(np.asarray(a, dtype=np.uint64).reshape(-1)))


def _coord(v, degree):
    return int_to_limbs(v) if degree == 1 else np.stack([int_to_limbs(v[0]), int_to_limbs(v[1])])


def points(group, pts: Sequence) -> np.ndarray:
    """ABI array of affine points given as (x, y) integer coordinates (Fp2
    coordinates as (c0, c1)) in whatever form the caller wants stored; None is
    the identity (infinity = true, coordinates 0)."""
    g = _group(group)
    out = np.zeros(len(pts), dtype=g.dtype)
    for i, p in enumerate(pts):
        if p is None:
            out[i]["infinity"] = True
        else:
            out[i]["x"], out[i]["y"] = _coord(p[0], g.degree), _coord(p[1], g.degree)
    return out


def scalars(values: Sequence[int]) -> np.ndarray:
    """(n, 5) uint64 scalars; every value must lie in [0, 2^320)."""
    out = np.zeros((len(values), 5), dtype=np.uint64)
    for i, v in enumerate(values):
        if not 0 <= int(v) < 1 << SCALAR_BITS:
            raise ValueError(f"scalar {v} is outside [0, 2^320)")
        out[i] = int_to_limbs(int(v), 5)
    return out


def _elem(a, degree):
    return limbs_to_int(a) if degree == 1 else (limbs_to_int(a[0]), limbs_to_int(a[1]))


def normalized_to_affine(group, proj: np.ndarray):
    """The (x, y) integers of a normalized projective result, None when Z = 0."""
    g = _group(group)
    proj = np.asarray(proj, dtype=np.uint64).reshape(g.proj_shape)
    if not proj[2].any():
        return None
    return _elem(proj[0], g.degree), _elem(proj[1], g.degree)


def normalize(group, proj: np.ndarray) -> np.ndarray:
    """g{1,2}_projective_from_montgomery_normalized_wrapper: Montgomery
    projective -> normal-form (X / Z, Y / Z, 1); Z = 0 stays 0."""
    g = _group(group)
    src = np.ascontiguousarray(proj, dtype=np.uint64).reshape(g.proj_shape)
    out = np.zeros(g.proj_shape, dtype=np.uint64)
    g.fn("{g}_projective_from_montgomery_normalized_wrapper")(out.ctypes.data, src.ctypes.data)
    return out


def _check_host(g, bases, ks):
    if not isinstance(bases, np.ndarray) or bases.dtype != g.dtype or bases.ndim != 1:
        raise ValueError(f"bases must be a 1-D numpy array of {g.name.upper()} ABI points")
    if not isinstance(ks, np.ndarray) or ks.dtype != np.uint64 or ks.ndim != 2 or ks.shape[1] != 5:
        raise ValueError("scalars must be an (n, 5) uint64 numpy array")
    if len(bases) != len(ks):
        raise ValueError(f"{len(bases)} bases but {len(ks)} scalars")
    if len(bases) >= 1 << 32:
        raise ValueError(f"n = {len(bases)} does not fit u32")


def _check_gpu(gpu_index):
    L = _lib.lib()
    count = L.cuda_get_number_of_gpus()
    if not 0 <= gpu_index < count:
        raise ValueError(f"gpu_index {gpu_index} exceeds available GPUs ({count})")
    return L


def msm_managed(group, bases: np.ndarray, ks: np.ndarray, gpu_index: int = 0, points_in_montgomery: bool = True,
                stream: Optional[int] = None) -> np.ndarray:
    """g{1,2}_msm_managed_wrapper on host arrays: the raw result (Montgomery
    projective, identity Z = 0).  n = 0 gives the identity without a call.
    `stream` is a cudaStream_t; by default a fresh one is created and destroyed."""
    g = _group(group)
    _check_host(g, bases, ks)
    out = np.zeros(g.proj_shape, dtype=np.uint64)
    if len(bases) == 0:
        return out
    L = _check_gpu(gpu_index)
    bases, ks = np.ascontiguousarray(bases), np.ascontiguousarray(ks)
    own = stream is None
    if own:
        stream = L.cuda_create_stream_ffi(gpu_index)
    tracker = C.c_uint64(0)
    try:
        g.fn("{g}_msm_managed_wrapper")(stream, gpu_index, out.ctypes.data, bases.ctypes.data, ks.ctypes.data,
                                         len(bases), points_in_montgomery, C.byref(tracker))
    finally:
        if own:
            L.cuda_destroy_stream(stream, gpu_index)
    return out


def _msm_gpu(g, bases, ks, gpu_index):
    raw = msm_managed(g, bases, ks, gpu_index, points_in_montgomery=False)
    if not raw[2].any():
        return None
    return normalized_to_affine(g, normalize(g, raw))


def g1_msm_gpu(bases: np.ndarray, ks: np.ndarray, gpu_index: int = 0):
    """tfhe-zk-pok's g1_msm_gpu: bases in normal form; the result as affine
    (x, y) integers, or None for the identity."""
    return _msm_gpu(G1, bases, ks, gpu_index)


def g2_msm_gpu(bases: np.ndarray, ks: np.ndarray, gpu_index: int = 0):
    """tfhe-zk-pok's g2_msm_gpu: as g1_msm_gpu, with Fp2 coordinates (c0, c1)."""
    return _msm_gpu(G2, bases, ks, gpu_index)


# ---- device-resident path ----

def words(group) -> int:
    """int64 words per point of a device point tensor (15 for G1, 29 for G2)."""
    return _group(group).dtype.itemsize // 8


def to_device(arr: np.ndarray, streams, stream_index: int = 0):
    """A host ABI array (points or scalars) as an int64 tensor of shape
    (n, words) on the stream's GPU."""
    import torch

    a = np.ascontiguousarray(arr)
    t = torch.from_numpy(a.view(np.int64).reshape(len(a), -1).copy())
    with torch.cuda.stream(streams.streams[stream_index]):
        return t.to(streams.device(stream_index), non_blocking=False)


def scratch_size(group, n: int, gpu_index: int = 0) -> int:
    g = _group(group)
    if not 0 < n < 1 << 32:
        raise ValueError(f"n = {n} must lie in [1, 2^32)")
    _check_gpu(gpu_index)
    return int(g.fn("pippenger_scratch_size_{g}_wrapper")(n, gpu_index))


def msm_device(group, d_points, d_scalars, streams, stream_index: int = 0, scratch=None) -> np.ndarray:
    """g{1,2}_msm_unmanaged_wrapper_async: d_points (n, words(group)) and
    d_scalars (n, 5) int64 tensors on the stream's GPU, points in Montgomery
    form; scratch a uint8 tensor of at least scratch_size(group, n) bytes
    (allocated on the stream when None).  Returns the raw result (Montgomery
    projective); the call has synchronized the stream."""
    import torch

    g = _group(group)
    dev = streams.device(stream_index)
    for name, t, w in (("points", d_points, words(g)), ("scalars", d_scalars, 5)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.int64 or t.dim() != 2 or t.shape[1] != w:
            raise ValueError(f"{name} must be an int64 tensor of shape (n, {w})")
        if t.device != dev or not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous on {dev}")
    n = d_points.shape[0]
    if d_scalars.shape[0] != n:
        raise ValueError(f"{n} points but {d_scalars.shape[0]} scalars")
    if n >= 1 << 32:
        raise ValueError(f"n = {n} does not fit u32")
    out = np.zeros(g.proj_shape, dtype=np.uint64)
    if n == 0:
        return out
    need = scratch_size(g, n, streams.gpu_indexes[stream_index])
    st = streams.streams[stream_index]
    if scratch is None:
        with torch.cuda.stream(st):
            scratch = torch.empty(need, dtype=torch.uint8, device=dev)
    elif (not isinstance(scratch, torch.Tensor) or scratch.device != dev or
          scratch.numel() * scratch.element_size() < need):
        raise ValueError(f"scratch must be a tensor of at least {need} bytes on {dev}")
    st.wait_stream(torch.cuda.current_stream(dev))
    g.fn("{g}_msm_unmanaged_wrapper_async")(streams.ptr(stream_index), streams.gpu_indexes[stream_index],
                                             out.ctypes.data, d_points.data_ptr(), d_scalars.data_ptr(), n,
                                             scratch.data_ptr())
    return out
