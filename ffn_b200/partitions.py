"""Partition map of a labelled volume on the device: compute_partitions (compute_partitions.py:115-204).

For every voxel of a labelled object, the fraction of identically labelled voxels in the (2r+1)^3 local object mask
(LOM) box around it, quantized by a list of thresholds; the result is what training coordinates are sampled from.
Counts are exact integers and the fraction is one float64 division, so the map equals the reference's bit for bit.
The computation runs in libffn_b200 (ffn_compute_partitions); there is no host fallback.
"""

from __future__ import annotations

import collections
import ctypes as C
import numbers

import numpy as np

from ffn_b200 import _lib

PartitionMap = collections.namedtuple('PartitionMap', ['corner', 'partitions', 'counts'])

_INT64_MAX = 2**63 - 1


def _radius(lom_radius):
  r = tuple(lom_radius)
  if len(r) != 3:
    raise ValueError('lom_radius must have 3 components (x, y, z), got %r' % (lom_radius,))
  for v in r:
    if not isinstance(v, numbers.Integral) or isinstance(v, bool):
      raise TypeError('lom_radius must hold integers, got %r' % (lom_radius,))
    if v < 0:
      raise ValueError('lom_radius must not be negative, got %r' % (lom_radius,))
    if v >= 2**31:
      raise ValueError('lom_radius too large: %r' % (lom_radius,))
  return tuple(int(v) for v in r)


def _whitelist_bits(id_whitelist, dtype):
  """The whitelisted values that are ids of `dtype`, as uint64 bit patterns (set membership by value)."""
  info = np.iinfo(dtype)
  bits = set()
  for w in id_whitelist:
    if isinstance(w, numbers.Integral):
      v = int(w)
    elif isinstance(w, numbers.Real) and float(w).is_integer():
      v = int(float(w))
    else:
      continue   # a string or a fraction equals no integer id
    if info.min <= v <= info.max:
      bits.add(v & (2**64 - 1))
  return np.array(sorted(bits), np.uint64)


def _spheres(exclusion_regions):
  """Exclusion regions (x, y, z, r) -> FfnExclusionSphere[]: int64 when all four values are integers (numpy's
  int64 arithmetic), float64 otherwise."""
  regions = list(exclusion_regions)
  arr = (_lib.ExclusionSphere * max(len(regions), 1))()
  for i, reg in enumerate(regions):
    vals = tuple(reg)
    if len(vals) != 4:
      raise ValueError('an exclusion region is (x, y, z, r), got %r' % (reg,))
    for v in vals:
      if not isinstance(v, numbers.Real):
        raise TypeError('exclusion region values must be numbers, got %r' % (reg,))
    s = arr[i]
    if all(isinstance(v, numbers.Integral) for v in vals):
      x, y, z, r = (int(v) for v in vals)
      if max(abs(x), abs(y), abs(z)) > _INT64_MAX:
        raise OverflowError('exclusion region %r does not fit in int64' % (reg,))
      s.integer = 1
      s.c_xyz[:] = (x, y, z)
      s.r2 = min(r * r, _INT64_MAX)
    else:
      s.f_xyz[:] = tuple(float(v) for v in vals[:3])
      r = vals[3]
      s.f_r2 = float(r * r) if isinstance(r, numbers.Integral) else float(r)**2
  return arr, len(regions)


def partition_map(seg_array, thresholds, lom_radius, id_whitelist=None, exclusion_regions=None, mask_configs=None,
                  min_size=10000, device=0, scratch_bytes=0) -> PartitionMap:
  """compute_partitions, with the 256-bin histogram of the partitions (`counts`, int64) computed alongside.

  `scratch_bytes` bounds the count scratch of one group of labels (8 bytes per voxel of their boxes grown by the
  radius); 0 takes a quarter of the free device memory.
  """
  if not isinstance(seg_array, np.ndarray) or not np.issubdtype(seg_array.dtype, np.integer):
    raise TypeError('seg_array must be a numpy array of integer ids, got %s'
                    % getattr(seg_array, 'dtype', type(seg_array)))
  if seg_array.ndim != 3:
    raise ValueError('seg_array must be 3-d, got shape %r' % (seg_array.shape,))
  if seg_array.size >= 2**31:
    raise ValueError('partition maps support volumes of fewer than 2^31 voxels, got %r' % (seg_array.shape,))
  r_xyz = _radius(lom_radius)
  th = np.array([float(t) for t in thresholds], np.float64)
  white = _whitelist_bits(id_whitelist, seg_array.dtype) if id_whitelist is not None else None
  spheres, n_spheres = _spheres(exclusion_regions) if exclusion_regions is not None else (None, 0)
  mask = None
  if mask_configs is not None:
    from ffn_b200.inference import storage
    built = storage.build_mask(mask_configs.masks, (0, 0, 0), seg_array.shape)
    if built is not None:
      mask = np.ascontiguousarray(built, dtype=np.uint8)
  ms = int(min(max(np.ceil(min_size), -2.0**62), 2.0**62))   # counts are integers: count < min_size <=> < ceil

  if np.issubdtype(seg_array.dtype, np.signedinteger):
    labels = np.ascontiguousarray(seg_array, dtype=np.int64).view(np.uint64).copy()
  else:
    labels = np.array(seg_array, dtype=np.uint64, order='C', copy=True)
  shape = seg_array.shape
  out = np.zeros([max(0, s - 2 * r) for s, r in zip(shape, r_xyz[::-1])], np.uint8)
  counts = np.zeros(256, np.int64)
  n_labels = C.c_int64(0)
  desc = _lib.PartitionDesc()
  desc.shape_zyx[:] = shape
  desc.lom_radius_zyx[:] = r_xyz[::-1]
  desc.min_size = ms
  desc.thresholds = th.ctypes.data
  desc.n_thresholds = th.size
  desc.use_whitelist = int(white is not None)
  desc.whitelist = white.ctypes.data if white is not None and white.size else None
  desc.n_whitelist = white.size if white is not None else 0
  desc.spheres = C.cast(spheres, C.c_void_p) if n_spheres else None
  desc.n_spheres = n_spheres
  desc.scratch_bytes = int(scratch_bytes)
  desc.n_labels_out = C.addressof(n_labels)
  lib = _lib.load()
  _lib.check(lib.ffn_compute_partitions(int(device), C.byref(desc), _lib.ptr(labels),
                                        _lib.ptr(mask) if mask is not None else None, _lib.ptr(out),
                                        _lib.ptr(counts)))
  if ms > 0:
    seg_array[labels.reshape(shape) == 0] = 0
  # The reference's quantization loop fails once it reaches its first label in these two cases.
  if n_labels.value and th.size == 0:
    raise IndexError('list index out of range')
  if n_labels.value and th.size + 1 > 255:
    raise OverflowError('Python integer %d out of bounds for uint8' % (th.size + 1))
  return PartitionMap(np.array(lom_radius), out, counts)


def compute_partitions(seg_array, thresholds, lom_radius, id_whitelist=None, exclusion_regions=None,
                       mask_configs=None, min_size=10000, device=0):
  """Computes quantized fractions of active voxels in a local object mask (compute_partitions.py:115-204).

  Args:
    seg_array: 3-d integer array of object ids (z, y, x), any signed or unsigned width; objects with fewer than
      `min_size` voxels are first set to 0 in place, as the reference's clear_dust does
    thresholds: activation voxel fractions; a voxel gets i + 1 for the first threshold (in list order) above its
      fraction, and len(thresholds) + 1 when there is none
    lom_radius: LOM radii as [x, y, z], non-negative integers
    id_whitelist: (optional) ids for which to compute the partition numbers, matched by value
    exclusion_regions: (optional) (x, y, z, r) spheres marked as excluded (255)
    mask_configs: (optional) MaskConfigs proto; any location whose LOM box holds a masked voxel becomes 255
    min_size: minimum number of voxels of an object to be partitioned
    device: CUDA device index (an H100)

  Returns:
    (corner as np.array(lom_radius) in (x, y, z), uint8 array of the VALID region, shape seg.shape - 2 r_zyx)

  Raises:
    TypeError: for a non-integer `seg_array` (the reference would accept floats) or non-integer radii
    ValueError: for a volume that is not 3-d, has 2^31 or more voxels, or a negative radius
    IndexError: empty `thresholds` with at least one label to partition, as in the reference
  """
  pm = partition_map(seg_array, thresholds, lom_radius, id_whitelist, exclusion_regions, mask_configs, min_size,
                     device)
  return pm.corner, pm.partitions


def partition_counts(counts):
  """The 256-bin histogram of a partition map -> np.array(np.unique(partitions, return_counts=True))."""
  counts = np.asarray(counts, np.int64)
  values = np.nonzero(counts)[0]
  return np.array([values, counts[values]])
