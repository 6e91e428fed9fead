"""Time of connected-component clean-up (clean_up_and_count with split_cc) on Voronoi-phantom cells cut along a
family of planes, with ids above 2^32 (the first segmentation of `synthetic.consensus_pair`): the 256x512x512 volume
of BASELINE configs[4] and a 512^3 volume, at 6- and 26-connectivity, min_size 1000.

    python tools/clean_up_timing.py [--out DIR] [--reps 3] [--host-reps 1] [--profile]

Device: wall time of the synchronous call (pageable upload, kernels, download of the labels and the id table),
median of --reps after a warm-up.  --profile instead sums the kernel and copy times of one call with torch.profiler
(run it as a separate command).  Host: the scipy oracle (oracle/clean_up.py), median of --host-reps, and whether it
equals the device result (array, id map and counts).  One JSON line per workload on stdout (and in
DIR/clean_up_timing[_profile].jsonl), with the GPU's name and power limit read in the same run.
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

from ffn_b200 import synthetic  # noqa: E402
from ffn_b200.inference import segmentation  # noqa: E402
from oracle import clean_up as ocu  # noqa: E402

WORKLOADS = [('configs4', (256, 512, 512)), ('iso_512', (512, 512, 512))]
CONNECTIVITY = (1, 3)
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
  ts = []
  for _ in range(reps):
    work = seg.copy()
    t0 = time.perf_counter()
    res = fn(work)
    ts.append(time.perf_counter() - t0)
  return float(np.median(ts)), ts, work, res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--host-reps', type=int, default=1)
  ap.add_argument('--profile', action='store_true')
  ap.add_argument('--skip-device', action='store_true', help='host timing only (no GPU needed)')
  ap.add_argument('--shape', default=None, help='z,y,x: one workload of this shape instead of the default two')
  args = ap.parse_args()
  info = _gpu()
  workloads = WORKLOADS if args.shape is None else [('custom', tuple(int(v) for v in args.shape.split(',')))]
  lines = []
  for name, shape in workloads:
    seg, _ = synthetic.consensus_pair(shape, seed=3, big_ids=True)
    for c in CONNECTIVITY:
      device = lambda x: segmentation.clean_up_and_count(x, True, c, MIN_SIZE)   # noqa: E731
      rec = {'workload': name, 'shape': list(shape), 'connectivity': c, 'min_size': MIN_SIZE,
             'ids_in': int(np.unique(seg).size)}
      if args.profile:
        device(seg.copy())
        rec['kernels_s'] = kernel_times(lambda: device(seg.copy()))
      else:
        got = None
        if not args.skip_device:
          device(seg.copy())   # warm-up
          rec['device_s'], rec['device_s_all'], got, got_res = median_time(device, seg, args.reps)
          rec['ids_out'] = len(got_res[1])
        if args.host_reps > 0:
          host = lambda x: ocu.clean_up_and_count(x, True, c, MIN_SIZE)   # noqa: E731
          rec['host_s'], rec['host_s_all'], want, want_res = median_time(host, seg, args.host_reps)
          rec['host_impl'] = 'scipy oracle'
          if got is not None:
            rec['equal'] = bool(np.array_equal(got, want) and got_res == want_res)
      rec.update(info)
      print(json.dumps(rec), flush=True)
      lines.append(rec)
    del seg
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'clean_up_timing%s.jsonl' % ('_profile' if args.profile else '')), 'w') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
