"""Result / checkpoint file formats and volume access.

Mirrors the parts of ffn/inference/storage.py the inference path touches: `OriginInfo` (:35),
`NumpyArray` (:55-71), `decorated_volume` (:74-112), `atomic_file` (:117-134),
`quantize_probability`/`dequantize_probability` (:137-151), `save_subvolume` (:154-171), the path
layout helpers (:174-241), `get_existing_subvolume_path` (:244-272), `threshold_segmentation`
(:275-288), `load_origins` (:291-299), `clip_subvolume_to_bounds` (:302-320), `build_mask`
(:323-411), `load_segmentation` (:414-488) and `load_segmentation_from_source` (:491-511).  File I/O
uses the local filesystem (the reference goes through `tf.io.gfile`).
"""

import collections
import contextlib
import glob
import json
import os
import re
import shutil
import tempfile

import numpy as np

from . import align
from . import segmentation

OriginInfo = collections.namedtuple('OriginInfo', ['start_zyx', 'iters', 'walltime_sec'])


class NumpyArray(np.ndarray):
  """ndarray with a `clear` method restoring the default value (host-side storage class)."""

  def __new__(cls, default_value=0, **kwargs):
    ret = super().__new__(cls, **kwargs)
    ret.default_value = default_value
    return ret

  def __init__(self, *args, **kwargs):
    del args, kwargs
    self.clear()

  def __array_finalize__(self, obj):
    self.default_value = getattr(obj, 'default_value', 0)

  def clear(self):
    self[...] = self.default_value


class _NpyVolume:
  """3d/4d array read from .npy / .npz — an offline stand-in where h5py is unavailable."""

  def __init__(self, arr):
    self._arr = arr
    self.shape = arr.shape
    self.ndim = arr.ndim
    self.dtype = arr.dtype

  def __getitem__(self, ind):
    return np.asarray(self._arr[ind])


def decorated_volume(settings, **kwargs):
  """DecoratedVolume proto -> array-like with __getitem__/shape/ndim (storage.py:74-112).

  `hdf5: "file.h5:dataset"` needs h5py.  As an extension for offline environments,
  `hdf5: "file.npy:"` and `hdf5: "file.npz:key"` are read with numpy.
  """
  del kwargs
  if settings.HasField('volinfo'):
    raise NotImplementedError('VolumeStore operations not available.')
  if settings.HasField('hdf5'):
    path = settings.hdf5.split(':')
    if len(path) != 2:
      raise ValueError('hdf5 volume_path should be specified as file_path:'
                       'hdf5_internal_dataset_path.  Got: ' + settings.hdf5)
    if path[0].endswith('.npy'):
      volume = _NpyVolume(np.load(path[0], mmap_mode='r'))
    elif path[0].endswith('.npz'):
      volume = _NpyVolume(np.load(path[0])[path[1]])
    else:
      try:
        import h5py  # pylint: disable=g-import-not-at-top
      except ImportError as e:
        raise ImportError('h5py is required to open %s' % settings.hdf5) from e
      volume = h5py.File(path[0], 'r')[path[1]]
  elif settings.HasField('tensorstore'):
    try:
      import tensorstore as ts  # pylint: disable=g-import-not-at-top
    except ImportError as e:
      raise ImportError('tensorstore is required for tensorstore volumes') from e
    store = ts.open(json.loads(settings.tensorstore)).result()

    class _Sync:
      shape, ndim, dtype = store.shape, store.ndim, store.dtype.numpy_dtype

      def __getitem__(self, ind):
        return np.array(store[ind])
    volume = _Sync()
  else:
    raise ValueError('A volume_path must be set.')
  if settings.HasField('decorator_specs'):
    raise ValueError('decorator_specs is only valid for volinfo volumes.')
  if volume.ndim not in (3, 4):
    raise ValueError('Volume must be 3d or 4d.')
  return volume


@contextlib.contextmanager
def atomic_file(path, mode='w+b'):
  """Writes to a temporary file and renames it over `path` (storage.py:117-134)."""
  directory = os.path.dirname(path) or '.'
  os.makedirs(directory, exist_ok=True)
  with tempfile.NamedTemporaryFile(mode=mode, dir=directory, delete=False, suffix='.tmp') as tmp:
    try:
      yield tmp
      tmp.flush()
    except BaseException:
      tmp.close()
      os.unlink(tmp.name)
      raise
  os.replace(tmp.name, path)


def quantize_probability(prob):
  """Probability -> uint8 in [1, 255]; 0 is reserved for NaN (storage.py:137-143)."""
  ret = np.digitize(prob, np.linspace(0.0, 1.0, 255))
  ret[np.isnan(prob)] = 0
  return ret.astype(np.uint8)


def dequantize_probability(prob):
  """Inverse of `quantize_probability` (storage.py:146-151)."""
  dq = 1.0 / 255
  ret = ((prob - 0.5) * dq).astype(np.float32)
  ret[prob == 0] = np.nan
  return ret


_DEFLATE_CHUNK = 4 << 20
_deflate_pool = None


def _pool():
  global _deflate_pool
  if _deflate_pool is None:
    from concurrent.futures import ThreadPoolExecutor
    _deflate_pool = ThreadPoolExecutor(max_workers=max(1, min(16, (os.cpu_count() or 2) - 1)), thread_name_prefix='ffn-deflate')
  return _deflate_pool


def _deflate_piece(view, level, last):
  """Raw-deflate one independent piece; not-last pieces end on a byte boundary without the final-block bit, so the
  concatenation of the pieces is ONE valid deflate stream (what pigz -i does).  zlib releases the GIL."""
  import zlib
  co = zlib.compressobj(level, zlib.DEFLATED, -15)
  return co.compress(view) + co.flush(zlib.Z_FINISH if last else zlib.Z_FULL_FLUSH)


def _npy_parts(arr):
  """The bytes of an .npy member as a list of buffers (header, data) without copying the data."""
  import io
  from numpy.lib import format as npy_format
  if arr.dtype.hasobject or arr.nbytes < (1 << 16):
    bio = io.BytesIO()
    npy_format.write_array(bio, arr, allow_pickle=True)
    return [bio.getvalue()]
  arr = np.ascontiguousarray(arr)
  bio = io.BytesIO()
  npy_format.write_array_header_1_0(bio, npy_format.header_data_from_array_1_0(arr))
  return [bio.getvalue(), memoryview(arr.reshape(-1).view(np.uint8))]


def savez_deflate(fd, compresslevel=3, **arrays):
  """Writes what np.savez_compressed writes — a zip archive of DEFLATE-compressed .npy members, readable by
  np.load — but compresses 4 MB pieces of every member on a thread pool (and at zlib level 3 instead of numpy's
  fixed 6): once the flood fill runs at 10^4 steps/s, single-threaded zlib over seg-*.npz / .prob was a sixth of
  Runner.run.  Members of 4 GB or more take the plain zipfile path (zip64)."""
  import struct
  import time
  import zlib
  members = []
  for name, value in arrays.items():
    parts = _npy_parts(np.asanyarray(value))
    if sum(len(x) for x in parts) >= 0xFFFFFFF0:
      return _savez_deflate_serial(fd, compresslevel, arrays)
    members.append((name + '.npy', parts))
  pool = _pool()
  jobs = []
  for name, parts in members:
    pieces = []
    for part in parts:
      view = memoryview(part)
      for off in range(0, max(len(view), 1), _DEFLATE_CHUNK):
        pieces.append(view[off:off + _DEFLATE_CHUNK])
    futs = [pool.submit(_deflate_piece, v, compresslevel, i == len(pieces) - 1) for i, v in enumerate(pieces)]

    def crc_of(parts=parts):
      crc = 0
      for part in parts:
        crc = zlib.crc32(part, crc)
      return crc
    jobs.append((name, parts, futs, pool.submit(crc_of)))
  t = time.localtime()
  dostime = (t.tm_hour << 11) | (t.tm_min << 5) | (t.tm_sec // 2)
  dosdate = ((max(t.tm_year, 1980) - 1980) << 9) | (t.tm_mon << 5) | t.tm_mday
  central = []
  offset = 0
  for name, parts, futs, crc_f in jobs:
    chunks = [f.result() for f in futs]
    csize = sum(len(x) for x in chunks)
    usize = sum(len(x) for x in parts)
    crc = crc_f.result() & 0xFFFFFFFF
    fname = name.encode('utf-8')
    if offset + csize >= 0xFFFFFFF0:
      raise ValueError('archive too large for the non-zip64 writer')
    fd.write(struct.pack('<IHHHHHIIIHH', 0x04034b50, 20, 0, 8, dostime, dosdate, crc, csize, usize, len(fname), 0))
    fd.write(fname)
    for x in chunks:
      fd.write(x)
    central.append(struct.pack('<IHHHHHHIIIHHHHHII', 0x02014b50, 20, 20, 0, 8, dostime, dosdate, crc, csize, usize,
                               len(fname), 0, 0, 0, 0, 0o600 << 16, offset) + fname)
    offset += 30 + len(fname) + csize
  cd = b''.join(central)
  fd.write(cd)
  fd.write(struct.pack('<IHHHHIIH', 0x06054b50, 0, 0, len(central), len(central), len(cd), offset, 0))


def _savez_deflate_serial(fd, compresslevel, arrays):
  import zipfile
  from numpy.lib import format as npy_format
  with zipfile.ZipFile(fd, mode='w', compression=zipfile.ZIP_DEFLATED, allowZip64=True, compresslevel=compresslevel) as zf:
    for name, value in arrays.items():
      arr = np.asanyarray(value)
      with zf.open(name + '.npy', 'w', force_zip64=True) as member:
        npy_format.write_array(member, arr, allow_pickle=True)


def save_subvolume(labels, origins, output_path, **misc_items):
  """seg-*.npz writer: segmentation (minimal uint dtype), origins, extra items (:154-171)."""
  seg = segmentation.reduce_id_bits(labels)
  os.makedirs(os.path.dirname(output_path), exist_ok=True)
  with atomic_file(output_path) as fd:
    savez_deflate(fd, segmentation=seg, origins=origins, **misc_items)


def legacy_subvolume_path(output_dir, corner, suffix):
  return os.path.join(output_dir, 'seg-%s.%s' % ('_'.join(str(x) for x in corner[::-1]), suffix))


def subvolume_path(output_dir, corner, suffix):
  """<out>/<x>/<y>/seg-<x>_<y>_<z>.<suffix> for a (z, y, x) corner (storage.py:189-202)."""
  return os.path.join(output_dir, str(corner[2]), str(corner[1]),
                      'seg-%s.%s' % ('_'.join(str(x) for x in corner[::-1]), suffix))


def get_corner_from_path(path):
  match = re.search(r'(\d+)_(\d+)_(\d+).npz', os.path.basename(path))
  if match is None:
    raise ValueError('Unrecognized path: %s' % path)
  return tuple(int(x) for x in match.groups())[::-1]


def get_existing_corners(segmentation_dir):
  corners = []
  for pattern in ('seg-*_*_*.npz', '*/*/seg-*_*_*.npz'):
    for path in glob.glob(os.path.join(segmentation_dir, pattern)):
      corners.append(get_corner_from_path(path))
  return corners


def checkpoint_path(output_dir, corner):
  return subvolume_path(output_dir, corner, 'cpoint')


def segmentation_path(output_dir, corner):
  return subvolume_path(output_dir, corner, 'npz')


def object_prob_path(output_dir, corner):
  return subvolume_path(output_dir, corner, 'prob')


def legacy_segmentation_path(output_dir, corner):
  return legacy_subvolume_path(output_dir, corner, 'npz')


def legacy_object_prob_path(output_dir, corner):
  return legacy_subvolume_path(output_dir, corner, 'prob')


def get_existing_subvolume_path(segmentation_dir, corner, allow_cpoint=False):
  for path in (segmentation_path(segmentation_dir, corner),
               legacy_segmentation_path(segmentation_dir, corner)):
    if os.path.exists(path):
      return path
  if allow_cpoint:
    path = checkpoint_path(segmentation_dir, corner)
    if os.path.exists(path):
      return path
  return None


def threshold_segmentation(segmentation_dir, corner, labels, threshold):
  prob_path = object_prob_path(segmentation_dir, corner)
  if not os.path.exists(prob_path):
    prob_path = legacy_object_prob_path(segmentation_dir, corner)
    if not os.path.exists(prob_path):
      raise ValueError('Cannot find probability map %s' % prob_path)
  with open(prob_path, 'rb') as f:
    data = np.load(f)
    if 'qprob' not in data:
      raise ValueError('Invalid FFN probability map.')
    prob = dequantize_probability(data['qprob'])
    labels[prob < threshold] = 0


def load_origins(segmentation_dir, corner):
  target_path = get_existing_subvolume_path(segmentation_dir, corner, False)
  if target_path is None:
    raise ValueError('Segmentation not found: %s, %s' % (segmentation_dir, corner))
  with open(target_path, 'rb') as f:
    data = np.load(f, allow_pickle=True)
    return data['origins'].item()


def clip_subvolume_to_bounds(corner, size, volume):
  """Clips a (z, y, x) box to the volume bounds (storage.py:302-320)."""
  volume_size = volume.shape[1:] if volume.ndim == 4 else volume.shape
  corner = np.asarray(corner)
  end = np.minimum(corner + np.asarray(size), np.asarray(volume_size))
  start = np.maximum(corner, 0)
  return start, np.maximum(end - start, 0)


def build_mask(masks, corner, subvol_size, mask_volume_map=None, image=None, alignment=None):
  """Boolean mask from MaskConfig protos (storage.py:323-411); True = excluded."""
  final_mask = None
  if mask_volume_map is None:
    mask_volume_map = {}
  if alignment is None:
    alignment = align.Alignment(corner, subvol_size)
  src_corner, src_size = alignment.expand_bounds(corner, subvol_size, forward=False)
  for config in masks:
    curr_mask = np.zeros(tuple(int(s) for s in subvol_size), dtype=bool)
    source_type = config.WhichOneof('source')
    if source_type == 'coordinate_expression':
      z, y, x = np.mgrid[[slice(int(c), int(c + s)) for c, s in zip(src_corner, src_size)]]
      bool_mask = eval(config.coordinate_expression.expression,  # pylint: disable=eval-used
                       {'np': np, 'x': x, 'y': y, 'z': z})
      curr_mask |= alignment.align_and_crop(src_corner, bool_mask, corner, subvol_size)
    else:
      if source_type == 'image':
        channels = config.image.channels
        mask = image
        if mask is None:
          raise ValueError('image mask requested but no image given')
      elif source_type == 'volume':
        channels = config.volume.channels
        key = config.volume.mask.SerializeToString()
        if key not in mask_volume_map:
          mask_volume_map[key] = decorated_volume(config.volume.mask)
        volume = mask_volume_map[key]
        clipped_corner, clipped_size = clip_subvolume_to_bounds(src_corner, src_size, volume)
        clipped_end = clipped_corner + clipped_size
        sel = tuple(slice(int(a), int(b)) for a, b in zip(clipped_corner, clipped_end))
        mask = volume[(slice(None),) + sel] if volume.ndim == 4 else volume[sel]
      else:
        raise ValueError('MaskConfig has no source')
      for chan_config in channels:
        channel_mask = mask[chan_config.channel] if mask.ndim == 4 else mask
        channel_mask = alignment.align_and_crop(src_corner, np.asarray(channel_mask), corner, subvol_size)
        if chan_config.values:
          bool_mask = np.isin(channel_mask, list(chan_config.values))
        else:
          bool_mask = (channel_mask >= chan_config.min_value) & (channel_mask <= chan_config.max_value)
        if chan_config.invert:
          bool_mask = np.logical_not(bool_mask)
        curr_mask |= bool_mask
    if config.invert:
      curr_mask = np.logical_not(curr_mask)
    final_mask = curr_mask if final_mask is None else (final_mask | curr_mask)
  return final_mask


def load_segmentation(segmentation_dir, corner, allow_cpoint=False, threshold=None, split_cc=True,
                      min_size=0, mask_config=None):
  """Loads a saved subvolume: (labels uint64, origins dict) (storage.py:414-488, simplified:
  connected-component splitting requires connectomics/skimage and is not performed)."""
  del split_cc, mask_config
  target_path = get_existing_subvolume_path(segmentation_dir, corner, allow_cpoint)
  if target_path is None:
    raise ValueError('Segmentation not found, %s, %r.' % (segmentation_dir, corner))
  with open(target_path, 'rb') as f:
    data = np.load(f, allow_pickle=True)
    if 'segmentation' in data:
      seg = data['segmentation']
    else:
      raise ValueError('FFN NPZ file %s does not contain valid segmentation.' % target_path)
    origins = _load_origins(data, target_path)
    output = seg.astype(np.uint64)
    if threshold is not None:
      threshold_segmentation(segmentation_dir, corner, output, threshold)
    if min_size:
      segmentation.clear_dust(output, min_size)
  return output, origins


def load_segmentation_from_source(source, corner):
  """Loads a saved subvolume as a SegmentationSource proto describes it (storage.py:491-511 with :414-488).

  Supports `directory`, `threshold` and `mask`.  Connected-component splitting and size filtering are not available:
  the source must set `split_cc: false`, and `min_size` must be unset or 0.

  Args:
    source: SegmentationSource proto
    corner: (z, y, x) subvolume corner

  Returns:
    (labels uint64, origins dict); an all-zero segmentation comes back with no origins, as in the reference

  Raises:
    NotImplementedError: if `split_cc` is unset or true, or `min_size` is above 0
    ValueError: when the segmentation (or the probability map a threshold needs) cannot be found
  """
  if not source.HasField('split_cc') or source.split_cc:
    raise NotImplementedError('SegmentationSource.split_cc must be set to false: connected-component splitting is '
                              'not available')
  if source.min_size:
    raise NotImplementedError('SegmentationSource.min_size must be unset or 0: size filtering after connected '
                              'components is not available')
  target_path = get_existing_subvolume_path(source.directory, corner)
  if target_path is None:
    raise ValueError('Segmentation not found, %s, %r.' % (source.directory, corner))
  with open(target_path, 'rb') as f:
    data = np.load(f, allow_pickle=True)
    if 'segmentation' in data:
      seg = data['segmentation']
    else:
      raise ValueError('FFN NPZ file %s does not contain valid segmentation.' % target_path)
    origins = _load_origins(data, target_path)
  if not np.any(seg):
    return np.zeros(seg.shape, dtype=np.uint64), {}
  output = seg.astype(np.uint64)
  if source.HasField('threshold'):
    threshold_segmentation(source.directory, corner, output, source.threshold)
  if source.HasField('mask'):
    mask = build_mask(source.mask.masks, corner, seg.shape)
    output[mask] = 0
  return output, origins


def _load_origins(data, path):
  """`origins` of a seg-*.npz.  Files written by the original (Python 2, internal) code base — e.g. the reference's
  shipped results/fib25/sample-training2.npz — pickle OriginInfo under its old module path with py2 strings: they
  are read with encoding='latin1' and the old module name mapped onto this package's OriginInfo."""
  try:
    return data['origins'].item()
  except (UnicodeDecodeError, ModuleNotFoundError, ImportError, AttributeError):
    pass
  import sys
  import types
  legacy = 'google3.research.neuromancer.segmentation.ffn.storage'
  added = []
  parts = legacy.split('.')
  for i in range(1, len(parts) + 1):
    name = '.'.join(parts[:i])
    if name not in sys.modules:
      sys.modules[name] = types.ModuleType(name)
      added.append(name)
  sys.modules[legacy].OriginInfo = OriginInfo
  try:
    with np.load(path, allow_pickle=True, encoding='latin1') as again:
      return again['origins'].item()
  finally:
    for name in added:
      sys.modules.pop(name, None)


def copy_file(src, dst):
  shutil.copyfile(src, dst)
