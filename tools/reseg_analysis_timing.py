"""Time of evaluate_pair_resegmentations on the device against the scipy oracle, per point and per batch.

    python tools/reseg_analysis_timing.py [--points 300] [--out DIR]

Workload: decision points of the 256x512x512 configs[4]-like Voronoi volume (tools/decision_point_timing.py) at voxel
size (z, y, x) = (40, 16, 16), one synthetic result file per point (oracle.reseg_analysis.write_synthetic_results) with
resegmentation radius (20, 40, 40) and the manual's analysis radius (17, 34, 34): a 35x69x69 analysis box.  Reports
  read_s      reading the files and cropping the segmentation alone (the thread pool of the batch call)
  device_s    wall time of the whole batch call (median of --reps), reading included
  kernels_s   device time per kernel of one batch call, from torch.profiler (a separate call)
  oracle_s    scipy / numpy host time of the oracle on --oracle-points of the same points
with the card's name, power limit and SM clock.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from decision_point_timing import kernel_times, labels  # noqa: E402
from ffn_b200.inference import resegmentation_analysis as ra  # noqa: E402
from ffn_b200.utils import decision_point as dp  # noqa: E402
from oracle import reseg_analysis as ora  # noqa: E402

RADIUS, ANALYSIS, VOXEL_ZYX = (20, 40, 40), (17, 34, 34), (40, 16, 16)


def _gpu():
  out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                        '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30,
                       check=True).stdout.strip().split(', ')
  return {'gpu': out[0], 'power_limit_w': float(out[1]), 'sm_clock_mhz': int(out[2]), 'sm_clock_max_mhz': int(out[3])}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--points', type=int, default=300)
  ap.add_argument('--oracle-points', type=int, default=60)
  ap.add_argument('--reps', type=int, default=5)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  seg = labels((256, 512, 512), (2.5, 1.0, 1.0))
  points = dp.find_decision_points(seg, VOXEL_ZYX[::-1])
  rng = np.random.RandomState(0)
  keys = list(points)
  items = [(a, b, tuple(int(v) for v in points[(a, b)][1])) for a, b in (keys[i] for i in rng.permutation(len(keys)))]
  tmp = tempfile.mkdtemp(prefix='reseg_timing_')
  paths = ora.write_synthetic_results(seg, items[:2 * args.points], RADIUS, tmp, seed=1)[:args.points]
  vol = seg[np.newaxis]
  call = lambda: ra.evaluate_pair_resegmentations(paths, vol, RADIUS, ANALYSIS, VOXEL_ZYX)  # noqa: E731
  rec = {'workload': 'configs4_voronoi_pairs', 'points': len(paths), 'analysis_box_zyx': [2 * a + 1 for a in ANALYSIS],
         'voxel_size_zyx': list(VOXEL_ZYX)}
  got = call()   # warm-up
  rec['scored'] = sum(not isinstance(g, Exception) for g in got)
  ts, tr = [], []
  for _ in range(args.reps):
    t0 = time.perf_counter()
    ra._gather(lambda f: ra._load_pair(f, vol, RADIUS, ANALYSIS), paths)   # pylint: disable=protected-access
    tr.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    call()
    ts.append(time.perf_counter() - t0)
  rec.update({'read_s': float(np.median(tr)), 'device_s': float(np.median(ts)), 'device_s_all': ts})
  rec['device_ms_per_point'] = 1e3 * rec['device_s'] / len(paths)
  kt = kernel_times(call)
  rec['kernels_s'] = kt
  rec['kernels_total_s'] = float(sum(kt.values()))
  n = min(args.oracle_points, len(paths))
  t0 = time.perf_counter()
  for p in paths[:n]:
    try:
      ora.evaluate_pair_resegmentation(p, vol, RADIUS, ANALYSIS, VOXEL_ZYX)
    except ora.InvalidBaseSegmentatonError:
      pass
  rec['oracle_points'] = n
  rec['oracle_ms_per_point'] = 1e3 * (time.perf_counter() - t0) / n
  rec.update(_gpu())
  print(json.dumps(rec), flush=True)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'reseg_analysis_timing.json'), 'w') as f:
      json.dump(rec, f, indent=1)


if __name__ == '__main__':
  main()
