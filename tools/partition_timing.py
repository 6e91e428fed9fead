"""Time of the partition map (ffn_b200.partitions.compute_partitions) on Voronoi-phantom ground truth of 256^3 and
600^3 voxels (the cube size the reference's sample workflow recommends), with the README's 12 thresholds, lom_radius
16 and min_size 1000.

    python tools/partition_timing.py [--out DIR] [--reps 3] [--host-reps 1] [--host-max-voxels N]

Device: wall time of the synchronous call (pageable upload of the labels, kernels, download of the result), median
of --reps after a warm-up, then the kernel and copy times of one more call from torch.profiler.  Host: the numpy
oracle (oracle/partitions.py), median of --host-reps, on the workloads of at most --host-max-voxels voxels (its
`seg == label` per label makes it labels x voxels), and whether it equals the device result.
One JSON line per workload on stdout (and in DIR/partition_timing.jsonl).
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from ffn_b200 import partitions  # noqa: E402
from ffn_b200 import synthetic  # noqa: E402
from oracle import partitions as op  # noqa: E402

WORKLOADS = [('cube_256', (256, 256, 256)), ('cube_600', (600, 600, 600))]
THRESHOLDS = [0.025, 0.05, 0.075, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]
RADIUS = [16, 16, 16]
MIN_SIZE = 1000


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


def median_time(fn, seg, reps):
  """Median wall time of fn(copy of seg) over reps calls; the copy is made outside the timed region."""
  ts, res = [], None
  for _ in range(reps):
    work = seg.copy()
    t0 = time.perf_counter()
    res = fn(work)
    ts.append(time.perf_counter() - t0)
  return float(np.median(ts)), ts, res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--host-reps', type=int, default=1)
  ap.add_argument('--host-max-voxels', type=int, default=256**3)
  args = ap.parse_args()
  info = _gpu()
  device = lambda s: partitions.compute_partitions(s, THRESHOLDS, RADIUS, min_size=MIN_SIZE)[1]   # noqa: E731
  host = lambda s: op.compute_partitions(s, THRESHOLDS, RADIUS, min_size=MIN_SIZE)[1]   # noqa: E731
  lines = []
  for name, shape in WORKLOADS:
    _, seg = synthetic.voronoi_phantom(shape, 7, return_cells=True)
    rec = {'workload': name, 'shape': list(shape), 'labels': int(np.unique(seg).size - 1), 'lom_radius': RADIUS,
           'min_size': MIN_SIZE}
    device(seg.copy())   # warm-up
    rec['device_s'], rec['device_s_all'], got = median_time(device, seg, args.reps)
    ks = kernel_times(lambda: device(seg.copy()))
    rec['kernels_s'] = ks
    rec['kernel_total_s'] = sum(v for k, v in ks.items() if 'Memcpy' not in k and 'Memset' not in k)
    if args.host_reps > 0 and seg.size <= args.host_max_voxels:
      rec['host_s'], rec['host_s_all'], want = median_time(host, seg, args.host_reps)
      rec['host_impl'] = 'numpy oracle'
      rec['equal'] = bool(got.shape == want.shape and (got == want).all())
    rec.update(info)
    print(json.dumps(rec), flush=True)
    lines.append(rec)
    del seg
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'partition_timing.jsonl'), 'w') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
