"""Time of the training coordinates (ffn_b200.coordinates.build_coordinates) on partition maps of Voronoi-phantom
ground truth of 256^3 and 600^3 voxels (compute_partitions with the README's 12 thresholds, lom_radius 16 and
min_size 1000), with the README's margin (35, 24, 24).

    python tools/coordinate_timing.py [--out DIR] [--workloads cube_256,cube_600] [--oracle-max-rows N]

Per workload, one call of each stage after a warm-up call of the device entry points, each ending in a device
synchronise:
  bucket_s     ffn_partition_rows on every volume (upload, kernels, download of the rows)
  shuffle_s    the host permutations and shuffle (numpy's RandomState)
  serialise_s  ffn_coordinate_records over every chunk (upload of the rows, kernels, download of the frames)
  deflate_s    the gzip member (CRC-32 and parallel deflate) of the frames, measured on up to 8 chunks and scaled
  write_s      serialise and deflate overlapped, as build_coordinates runs them, into a temporary file
  wall_s       build_coordinates end to end into a temporary file
and the kernel times of one bucketing call and one chunk from torch.profiler.  The numpy oracle (oracle/coordinates.py)
runs when the workload has at most --oracle-max-rows records; its rows are compared with the device's.
One JSON line per workload on stdout (and in DIR/coordinate_timing.jsonl).
"""

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from ffn_b200 import _lib  # noqa: E402
from ffn_b200 import coordinates  # noqa: E402
from ffn_b200 import partitions  # noqa: E402
from ffn_b200 import synthetic  # noqa: E402
from oracle import coordinates as oc  # noqa: E402

WORKLOADS = {'cube_256': (256, 256, 256), 'cube_600': (600, 600, 600)}
THRESHOLDS = [0.025, 0.05, 0.075, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]
RADIUS = [16, 16, 16]
MIN_SIZE = 1000
MARGIN = (35, 24, 24)
SEED = 0


def _gpu():
  try:
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30,
                         check=True).stdout.strip().split(', ')
  except (OSError, subprocess.SubprocessError):
    return {'gpu': None}
  return {'gpu': out[0], 'power_limit_w': float(out[1]), 'max_sm_clock_mhz': float(out[2])}


def kernel_times(fn):
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
  return {e.key: e.self_device_time_total * 1e-6 for e in prof.key_averages() if e.self_device_time_total > 0}


class _Null:
  def write(self, b):
    return len(b)


def partition_volume(shape):
  _, cells = synthetic.voronoi_phantom(shape, 7, return_cells=True)
  pm = partitions.partition_map(cells, THRESHOLDS, RADIUS, min_size=MIN_SIZE)
  full = np.full(shape, 255, np.uint8)
  r = RADIUS[::-1]
  full[r[0]:shape[0] - r[0], r[1]:shape[1] - r[1], r[2]:shape[2] - r[2]] = pm.partitions
  return full


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--workloads', default='cube_256,cube_600')
  ap.add_argument('--oracle-max-rows', type=int, default=50_000_000)
  args = ap.parse_args()
  info = _gpu()
  lib = _lib.load()
  lines = []
  for name in args.workloads.split(','):
    shape = WORKLOADS[name]
    vol = partition_volume(shape)
    rec = {'workload': name, 'shape': list(shape), 'margin_zyx': list(MARGIN), 'lom_radius': RADIUS}
    coordinates.partition_rows(vol[:40, :40, :40], MARGIN)   # warm-up of the device and its modules
    t0 = time.perf_counter()
    rows, counts = coordinates.partition_rows(vol, MARGIN)
    rec['bucket_s'] = time.perf_counter() - t0
    rec['crop_voxels'] = int(counts.sum())
    rec['kept_voxels'] = len(rows)
    rec['partitions'] = int((counts[:255] > 0).sum())
    rec['bucket_kernels_s'] = kernel_times(lambda: coordinates.partition_rows(vol, MARGIN))
    ends = np.cumsum(counts)
    parts = [rows[ends[v] - counts[v]:ends[v]] for v in np.flatnonzero(counts[:255])]
    np.random.seed(SEED)
    t0 = time.perf_counter()
    shuffled = coordinates.resample_and_shuffle(parts)
    rec['shuffle_s'] = time.perf_counter() - t0
    rec['records'] = len(shuffled)
    del parts, rows
    extent = coordinates.crop_box(vol.shape, MARGIN)[1]

    # serialise alone: every chunk into one reused buffer
    table, blob, max_name = coordinates._record_table(['vol'], [extent], MARGIN)
    desc = _lib.CoordinateDesc()
    desc.volumes = C.cast(table, C.c_void_p)
    desc.n_volumes = 1
    desc.names = blob.ctypes.data
    desc.names_bytes = blob.size
    chunk = coordinates.CHUNK_ROWS
    buf = np.empty(chunk * (130 + max_name), np.uint8)
    nbytes = C.c_int64(0)
    total, sample, sample_bytes = 0, [], 0
    t0 = time.perf_counter()
    for start in range(0, len(shuffled), chunk):
      part = shuffled[start:start + chunk]
      _lib.check(lib.ffn_coordinate_records(0, C.byref(desc), _lib.ptr(part), len(part), _lib.ptr(buf), buf.size,
                                            C.byref(nbytes)))
      total += nbytes.value
      if len(sample) < 8:
        sample.append(buf[:nbytes.value].copy())
    rec['serialise_s'] = time.perf_counter() - t0
    rec['uncompressed_bytes'] = total
    rec['serialise_kernels_s'] = kernel_times(lambda: lib.ffn_coordinate_records(
        0, C.byref(desc), _lib.ptr(shuffled[:chunk]), min(chunk, len(shuffled)), _lib.ptr(buf), buf.size,
        C.byref(nbytes)))
    t0 = time.perf_counter()
    w = coordinates.GzipMemberWriter(_Null())
    for s in sample:
      w.write(s)
      sample_bytes += s.size
    w.close()
    rec['deflate_s'] = (time.perf_counter() - t0) * total / max(sample_bytes, 1)
    del sample

    with tempfile.TemporaryDirectory() as tmp:
      path = os.path.join(tmp, 'coords.gz')
      with open(path, 'wb') as fd:
        t0 = time.perf_counter()
        coordinates.write_records(fd, shuffled, ['vol'], [extent], MARGIN)
        fd.flush()
        rec['write_s'] = time.perf_counter() - t0
      rec['file_bytes'] = os.path.getsize(path)
      del shuffled
      np.random.seed(SEED)
      t0 = time.perf_counter()
      coordinates.build_coordinates([('vol', vol)], MARGIN, path)
      rec['wall_s'] = time.perf_counter() - t0
    if rec['records'] <= args.oracle_max_rows:
      np.random.seed(SEED)
      t0 = time.perf_counter()
      want, _ = oc.coordinate_rows([vol], MARGIN)
      rec['oracle_rows_s'] = time.perf_counter() - t0
      np.random.seed(SEED)
      got, _ = coordinates.coordinate_rows([vol], MARGIN)
      rec['oracle_equal'] = bool(got.shape == want.shape and (got == want).all())
      del want, got
    else:
      rec['oracle_rows_s'] = None
    rec.update(info)
    print(json.dumps(rec), flush=True)
    lines.append(rec)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'coordinate_timing.jsonl'), 'w') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
