"""Device time of find_decision_points on Voronoi-cell labels: the 256x512x512 volume of BASELINE configs[4] at voxel
size xyz (16, 16, 40), and a 512^3 isotropic volume; with a host cost comparison.

    python tools/decision_point_timing.py [--out DIR] [--reps 3] [--skip-host] [--profile] [--reference DIR]

The labels tile a small Voronoi phantom's cells (membranes are background, so every call expands into gaps) with
distinct ids per tile; generating a 512^3 phantom directly takes minutes on the host.  Device times are the wall
time of the synchronous call (label copy and upload, kernels, result copy), median of --reps after a warm-up.
--profile instead sums the kernel and copy times of one call with torch.profiler (run it as a separate command).

Host comparison: a scipy feature-transform watershed_expand (one exact EDT with indices: the nearest labelled voxel,
with scipy's own choice on ties) followed by the numpy pair search of oracle/decision_points.py, or by the
reference's find_decision_points when --reference names a reference checkout.  It is a cost comparison only: its
ties differ from the smallest-id rule, so its result is not compared.
One JSON line per measurement on stdout (and in DIR/decision_point_timing.jsonl).
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
from scipy import ndimage

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from ffn_b200 import synthetic  # noqa: E402
from ffn_b200.utils import decision_point as dp  # noqa: E402
from oracle import decision_points as odp  # noqa: E402

WORKLOADS = [   # name, shape zyx, voxel size xyz, phantom voxel size zyx
    ('configs4_aniso', (256, 512, 512), (16, 16, 40), (2.5, 1.0, 1.0)),
    ('iso_512', (512, 512, 512), (1, 1, 1), (1.0, 1.0, 1.0)),
]


def _gpu():
  out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                       capture_output=True, text=True, timeout=30, check=True).stdout.strip().split(', ')
  return {'gpu': out[0], 'power_limit_w': float(out[1])}


def labels(shape, phantom_voxel):
  _, cells = synthetic.voronoi_phantom((64, 128, 128), seed=3, voxel_size_zyx=phantom_voxel, cell_volume=20000.0,
                                       return_cells=True)
  ncell = int(cells.max())
  reps = [int(np.ceil(s / t)) for s, t in zip(shape, cells.shape)]
  seg = np.zeros(shape, dtype=np.uint64)
  t = 0
  for iz in range(reps[0]):
    for iy in range(reps[1]):
      for ix in range(reps[2]):
        z0, y0, x0 = iz * 64, iy * 128, ix * 128
        blk = seg[z0:z0 + 64, y0:y0 + 128, x0:x0 + 128]
        c = cells[:blk.shape[0], :blk.shape[1], :blk.shape[2]].astype(np.uint64)
        blk[...] = np.where(c > 0, c + np.uint64(t * ncell), np.uint64(0))
        t += 1
  return seg


def host_points(seg, voxel_size, reference=None):
  if reference:
    sys.path.insert(0, os.path.join(REPO, 'tests', 'golden'))
    import make_golden as mg
    mg.install_stubs()
    sys.modules['connectomics.segmentation.labels'].watershed_expand = scipy_watershed_expand
    sys.path.insert(0, reference)
    from ffn.utils import decision_point as ref_dp   # the reference's module (the repo's ffn/ shim otherwise)
    return ref_dp.find_decision_points(seg, voxel_size)
  expanded, edt = scipy_watershed_expand(seg, voxel_size)
  return odp.points_of_expansion(expanded, edt)


def scipy_watershed_expand(seg, voxel_size, max_distance=None):
  edt, idx = ndimage.distance_transform_edt(seg == 0, sampling=tuple(voxel_size)[::-1], return_indices=True)
  expanded = seg[tuple(idx)]
  if max_distance is not None:
    expanded[edt > max_distance] = 0
  return expanded, edt


def kernel_times(fn):
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
  return {e.key: e.self_device_time_total * 1e-6 for e in prof.key_averages() if e.self_device_time_total > 0}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--skip-host', action='store_true')
  ap.add_argument('--profile', action='store_true')
  ap.add_argument('--reference', default=None)
  args = ap.parse_args()
  info = _gpu()
  lines = []
  for name, shape, vs, pvs in WORKLOADS:
    seg = labels(shape, pvs)
    rec = {'workload': name, 'shape': list(shape), 'voxel_size_xyz': list(vs), 'ids': int(np.unique(seg).size - 1)}
    call = lambda: dp.find_decision_points(seg, vs)   # noqa: E731
    if args.profile:
      call()
      rec['kernels_s'] = kernel_times(call)
    else:
      got = call()   # warm-up
      ts = []
      for _ in range(args.reps):
        t0 = time.perf_counter()
        got = call()
        ts.append(time.perf_counter() - t0)
      rec.update({'pairs': len(got), 'device_s': float(np.median(ts)), 'device_s_all': ts})
      if not args.skip_host:
        t0 = time.perf_counter()
        host = host_points(seg, vs, args.reference)
        rec['host_cost_s'] = time.perf_counter() - t0
        rec['host_pairs'] = len(host)
        rec['host_impl'] = 'reference' if args.reference else 'scipy feature transform + oracle pair search'
    rec.update(info)
    print(json.dumps(rec), flush=True)
    lines.append(rec)
    del seg
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'decision_point_timing%s.jsonl' % ('_profile' if args.profile else '')),
              'w') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
