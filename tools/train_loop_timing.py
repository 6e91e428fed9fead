"""Training steps per second of Trainer.train (the example loop on the device) against Trainer.step fed precomputed
host batches, at the FIB-25 geometry (33^3 field of view, depth 12, deltas 8, batch 4) on a Voronoi phantom.

    python tools/train_loop_timing.py [--out DIR] [--steps 100] [--reps 3] [--profile]

Each repeat times --steps steps with a host clock around calls that end in a device synchronisation, after a warm-up;
the median and the spread over --reps repeats are reported for both policies (fixed, max_pred_moves) and for
Trainer.step on batches the loop produced beforehand (no loop work between steps, but the host copies step() makes).
--profile instead records Trainer.train with torch.profiler and reports the example-loop kernels' device time per step
(run it as a separate command).  One JSON line on stdout (and in DIR), with the GPU's name and power limit read in the
same run.
"""

import argparse
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

FOV, DELTAS, BATCH = (33, 33, 33), (8, 8, 8), 4
LOOP_KERNELS = ('exk::resume', 'exk::load', 'exk::crop', 'exk::paste', 'sum_loss')


def _gpu():
  import subprocess
  out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                       capture_output=True, text=True, timeout=30, check=True).stdout.strip().split(', ')
  return {'gpu': out[0], 'power_limit_w': float(out[1])}


def setup(policy, seed=0):
  from ffn_b200 import tf_checkpoint
  from ffn_b200.synthetic import voronoi_phantom
  from ffn_b200.training import examples as ex
  from ffn_b200.training.trainer import Trainer
  image, cells = voronoi_phantom((160, 160, 160), seed, return_cells=True)
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(REPO, 'tests', 'golden', 'fib25_convstack.npz'))
  moves = ex.patch_moves(policy, 1)
  half = np.array(FOV) // 2 + np.array(DELTAS) * moves
  rng = np.random.RandomState(seed)
  centers = np.stack([rng.randint(h, 160 - h, 4096) for h in half[::-1]], 1)
  stream = ex.ExampleStream(np.zeros(len(centers)), centers, (1, 2), (0, 1, 2), seed=seed)
  loop = ex.ExampleLoop({'vol': (image, cells.astype(np.int64))}, stream, FOV, DELTAS, BATCH, policy,
                        image_mean=128.0, image_stddev=33.0)
  trainer = Trainer(w, b, FOV, optimizer='adam', learning_rate=1e-4, batch_size=BATCH)
  return trainer, loop


def _median(fn, steps, reps):
  times = []
  for _ in range(reps):
    t0 = time.perf_counter()
    fn()
    times.append(time.perf_counter() - t0)
  rates = sorted(steps / t for t in times)
  return {'steps_per_s': rates[len(rates) // 2], 'min': rates[0], 'max': rates[-1]}


def timing(args):
  out = {}
  for policy in ('fixed', 'max_pred_moves'):
    trainer, loop = setup(policy)
    trainer.train(loop, 10)
    out['train_' + policy] = _median(lambda: trainer.train(loop, args.steps), args.steps, args.reps)
    if policy == 'fixed':
      batches = [loop.next()[:3] for _ in range(args.steps)]
      trainer.step(*batches[0])

      def steps():
        for s, im, lb in batches:
          trainer.step(s, im, lb)
      out['step_host_batches'] = _median(steps, args.steps, args.reps)
    loop.close()
    trainer.close()
  return out


def profile(args):
  import torch
  from torch.profiler import ProfilerActivity
  out = {}
  for policy in ('fixed', 'max_pred_moves'):
    trainer, loop = setup(policy)
    trainer.train(loop, 10)
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
      trainer.train(loop, args.steps)
    loop_us = total_us = 0.0
    for ev in prof.key_averages():
      t = getattr(ev, 'device_time_total', None)
      if t is None:
        t = ev.cuda_time_total
      total_us += t
      if any(k in ev.key for k in LOOP_KERNELS):
        loop_us += t
    out[policy] = {'loop_kernels_us_per_step': loop_us / args.steps, 'all_kernels_us_per_step': total_us / args.steps}
    loop.close()
    trainer.close()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--steps', type=int, default=100)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--profile', action='store_true')
  args = ap.parse_args()
  res = dict(_gpu(), fov=FOV, deltas=DELTAS, batch=BATCH, depth=12, steps=args.steps)
  res.update(profile(args) if args.profile else timing(args))
  line = json.dumps(res)
  print(line)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'train_loop_timing%s.json' % ('_profile' if args.profile else '')), 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
