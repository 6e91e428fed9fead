"""Cost of train.py's training state at the FIB-25 geometry (33^3 field of view, depth 12, deltas 8, batch 4, adam), for
both policies: the blob sizes, the state file's size, saving (get_state of the trainer, the loop and the stream, and
writing train_state-<step>.npz) and restoring (reading the file, then set_state), each the median of --reps runs with a
host clock around calls that end in a device synchronisation.

    python tools/train_state_timing.py [--out DIR] [--reps 7]

One JSON line on stdout (and in DIR), with the GPU's name and power limit read in the same run.
"""

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))


def _median_ms(fn, reps):
  times = []
  for _ in range(reps):
    t0 = time.perf_counter()
    fn()
    times.append(time.perf_counter() - t0)
  times.sort()
  return {'median_ms': 1e3 * times[len(times) // 2], 'min_ms': 1e3 * times[0], 'max_ms': 1e3 * times[-1]}


def timing(args):
  import train
  import train_loop_timing as tlt
  out = {}
  for policy in ('fixed', 'max_pred_moves'):
    trainer, loop = tlt.setup(policy)
    losses = trainer.train(loop, 20).tolist()
    with tempfile.TemporaryDirectory() as d:
      path = train.save_state(d, trainer, loop, losses, {})
      res = {'trainer_blob_bytes': int(trainer.get_state().size), 'loop_blob_bytes': int(loop.get_state()['device'].size),
             'state_file_bytes': os.path.getsize(path)}
      res['save'] = _median_ms(lambda: train.save_state(d, trainer, loop, losses, {}), args.reps)
      res['restore'] = _median_ms(lambda: train.restore_state(train.load_state(path, {}), trainer, loop), args.reps)
      res['get_state_only'] = _median_ms(lambda: (trainer.get_state(), loop.get_state()), args.reps)
      blobs = trainer.get_state(), loop.get_state()
      res['set_state_only'] = _median_ms(lambda: (trainer.set_state(blobs[0]), loop.set_state(blobs[1])), args.reps)
      # the restored objects continue as an untouched pair does
      t2, l2 = tlt.setup(policy)
      t2.train(l2, 20)
      res['continues_bit_for_bit'] = bool(np.array_equal(trainer.train(loop, 5), t2.train(l2, 5)))
      t2.close()
      l2.close()
    out[policy] = res
    loop.close()
    trainer.close()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--reps', type=int, default=7)
  args = ap.parse_args()
  import train_loop_timing as tlt
  res = dict(tlt._gpu(), fov=tlt.FOV, deltas=tlt.DELTAS, batch=tlt.BATCH, depth=12, optimizer='adam')
  res.update(timing(args))
  line = json.dumps(res)
  print(line)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'train_state_timing.json'), 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
