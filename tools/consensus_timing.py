"""Time of split consensus (split_segmentation_by_intersection) on two Voronoi-phantom segmentations that disagree as
a forward and a reverse run do (`synthetic.consensus_pair`: the same cells cut along different planes, pairwise merges
in the second, ids above 2^32 in the first): the 256x512x512 volume of BASELINE configs[4] and a 512^3 volume.

    python tools/consensus_timing.py [--out DIR] [--reps 3] [--host-reps 3] [--profile] [--reference DIR]

Device: wall time of the synchronous call (pageable upload of both arrays, kernels, download of the result), median
of --reps after a warm-up.  --profile instead sums the kernel and copy times of one call with torch.profiler (run it
as a separate command).  Host: the numpy oracle (oracle/consensus.py), median of --host-reps, and whether it equals
the device result; with --reference, the reference's own split_segmentation_by_intersection instead.
One JSON line per workload on stdout (and in DIR/consensus_timing[_profile].jsonl).
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
from oracle import consensus as oc  # noqa: E402

WORKLOADS = [('configs4', (256, 512, 512)), ('iso_512', (512, 512, 512))]
MIN_SIZE = 50


def _gpu():
  try:
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30,
                         check=True).stdout.strip().split(', ')
  except (OSError, subprocess.SubprocessError):
    return {'gpu': None}
  return {'gpu': out[0], 'power_limit_w': float(out[1]), 'max_sm_clock_mhz': float(out[2])}


def reference_split(reference):
  sys.path.insert(0, os.path.join(REPO, 'tests', 'golden'))
  import make_golden as mg
  mg.install_stubs()
  sys.path.insert(0, reference)
  import importlib.util
  spec = importlib.util.spec_from_file_location('ref_segmentation', os.path.join(reference, 'ffn/inference/segmentation.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod.split_segmentation_by_intersection


def kernel_times(fn):
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
  return {e.key: e.self_device_time_total * 1e-6 for e in prof.key_averages() if e.self_device_time_total > 0}


def median_time(fn, a, reps):
  """Median wall time of fn(copy of a) over reps calls; the copy is made outside the timed region."""
  ts = []
  for _ in range(reps):
    work = a.copy()
    t0 = time.perf_counter()
    fn(work)
    ts.append(time.perf_counter() - t0)
  return float(np.median(ts)), ts, work


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--host-reps', type=int, default=3)
  ap.add_argument('--profile', action='store_true')
  ap.add_argument('--skip-device', action='store_true', help='host timing only (no GPU needed)')
  ap.add_argument('--reference', default=None)
  args = ap.parse_args()
  info = _gpu()
  host = reference_split(args.reference) if args.reference else oc.split_segmentation_by_intersection
  device = lambda x: segmentation.split_segmentation_by_intersection(x, b, MIN_SIZE)   # noqa: E731
  lines = []
  for name, shape in WORKLOADS:
    a, b = synthetic.consensus_pair(shape, seed=3, big_ids=True)
    rec = {'workload': name, 'shape': list(shape), 'min_size': MIN_SIZE, 'ids_a': int(np.unique(a).size),
           'ids_b': int(np.unique(b).size)}
    if args.profile:
      device(a.copy())
      rec['kernels_s'] = kernel_times(lambda: device(a.copy()))
    else:
      got = None
      if not args.skip_device:
        device(a.copy())   # warm-up
        rec['device_s'], rec['device_s_all'], got = median_time(device, a, args.reps)
        rec['ids_out'] = int(np.unique(got).size)
      if args.host_reps > 0:
        rec['host_s'], rec['host_s_all'], want = median_time(lambda x: host(x, b, MIN_SIZE), a, args.host_reps)
        rec['host_impl'] = 'reference' if args.reference else 'numpy oracle'
        if got is not None:
          rec['equal'] = bool((got == want).all())
    rec.update(info)
    print(json.dumps(rec), flush=True)
    lines.append(rec)
    del a, b
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'consensus_timing%s.jsonl' % ('_profile' if args.profile else '')), 'w') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
