"""Device vs host time of the peak_local_max seed policies (PolicyPeaks2d on the 256x512x512 serial-section
volume of BASELINE configs[4], PolicyFillEmptySpace on a 512^3 canvas), and the tie-break noise upload alone.

    python tools/seed_policy_timing.py [--out DIR] [--reps 3] [--skip-host]

The volumes tile a small Voronoi phantom (generating a 512^3 phantom takes minutes on the host); the policies' cost
does not depend on the content beyond the number of peaks, which is printed.  Device times are wall time of the
synchronous ffn_canvas_seed_policy call (allocation, noise upload, kernels, coordinate copy); per-kernel and copy
times of one call come from torch.profiler, and the noise upload is also timed alone, as a pageable host-to-device copy of the same array.  One JSON line per measurement on stdout
(and in DIR/seed_policy_timing.jsonl).
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ffn_b200 import _lib, engine as eng, synthetic, tf_checkpoint  # noqa: E402
from ffn_b200.inference import seed  # noqa: E402


class _HostCanvas:
  def __init__(self, image, segmentation):
    self.image, self.segmentation, self.restrictor = image, segmentation, None
    self.shape, self.margin, self.voxel_size_zyx = image.shape, np.zeros(3, int), (1, 1, 1)


def _gpu():
  try:
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                         capture_output=True, text=True, timeout=30).stdout.strip().split(', ')
    return {'gpu': out[0], 'power_limit_w': float(out[1])}
  except Exception:  # pylint: disable=broad-except
    return {'gpu': None, 'power_limit_w': None}


def _tile(small, shape):
  reps = [int(np.ceil(s / t)) for s, t in zip(shape, small.shape)]
  return np.ascontiguousarray(np.tile(small, reps)[:shape[0], :shape[1], :shape[2]])


def _upload(host_array):
  import torch
  out = torch.from_numpy(host_array).to('cuda:0')
  torch.cuda.synchronize()
  return out


def _kernel_time(fn):
  """Sum of the GPU kernel durations of one call (torch.profiler sees the library's kernels through CUPTI)."""
  try:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      fn()
    return {e.key: e.self_device_time_total * 1e-6 for e in prof.key_averages() if e.self_device_time_total > 0}
  except Exception as e:  # pylint: disable=broad-except
    return 'profiler unavailable: %s' % e


def _median_time(fn, reps):
  fn()                                            # warm-up (module load, first allocations)
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter()
    out = fn()
    ts.append(time.perf_counter() - t0)
  return float(np.median(ts)), out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--skip-host', action='store_true')
  args = ap.parse_args()
  repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(repo, 'tests', 'golden', 'fib25_convstack.npz'))
  engine = eng.Engine(w, b, (17, 33, 33), (4, 8, 8))
  info = _gpu()
  lines = []

  def emit(rec):
    rec.update(info)
    print(json.dumps(rec), flush=True)
    lines.append(rec)

  small, cells = synthetic.voronoi_phantom((64, 128, 128), seed=3, sigma=(0.5, 1, 1), voxel_size_zyx=(4, 1, 1),
                                           cell_volume=20000.0, return_cells=True)
  for kind, policy, shape in (('peaks_2d', 'PolicyPeaks2d', (256, 512, 512)),
                              ('fill_empty', 'PolicyFillEmptySpace', (512, 512, 512))):
    vol = _tile(small, shape)
    seg = np.zeros(shape, dtype=np.int32)
    if kind == 'fill_empty':
      c = _tile(cells, shape)
      seg[(c % 2 == 1)] = 1                        # about half of the cells labelled
      del c
    noise = np.random.RandomState(seed=42).rand(*(shape[1:] if kind == 'peaks_2d' else shape))
    md, thr = (7, 2.5) if kind == 'peaks_2d' else (2, 0.5)
    cv = eng.DeviceCanvas(engine, vol, eng.make_options(), 128.0, 33.0, keep_probability_maps=False)
    cv.write(_lib.ARRAY_SEGMENTATION, seg)
    t_dev, dev = _median_time(lambda: cv.seed_policy(kind, md, thr, 0, noise), args.reps)
    kernels_s = _kernel_time(lambda: cv.seed_policy(kind, md, thr, 0, noise))
    cv.close()
    t_up, _ = _median_time(lambda: _upload(noise), args.reps)
    rec = {'policy': policy, 'shape': list(shape), 'peaks': int(dev.shape[0]), 'device_s': t_dev, 'kernels_s': kernels_s,
           'noise_upload_s': t_up, 'noise_bytes': int(noise.nbytes)}
    if not args.skip_host:
      image = (vol.astype(np.float32) - np.float32(128)) / np.float32(33)
      host_cv = _HostCanvas(image, seg)
      t0 = time.perf_counter()
      pol = getattr(seed, policy)(host_cv)
      host = pol.remaining()
      rec['host_s'] = time.perf_counter() - t0
      rec['host_equals_device'] = bool(np.array_equal(host, dev))
      rec['speedup'] = rec['host_s'] / t_dev
      del image, host_cv
    emit(rec)
    del vol, seg, noise
  engine.close()
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'seed_policy_timing.jsonl'), 'w') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
