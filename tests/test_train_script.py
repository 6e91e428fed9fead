"""train.py's flags and its checks before any device work: the learning-rate schedule follows optimizer.py (decay only
when both --learning_rate_decay_factor and --decay_steps are given, --decay_steps passed through), and a coordinate
naming a volume without data or labels is refused.  CPU only (each run is a subprocess, so the script's absl flags stay
out of this process)."""

import gzip
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from test_examples_oracle import _example

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCHEDULE = r'''
import json, sys
import train
from ffn_b200.training.trainer import decayed_learning_rate
train.FLAGS(['train.py'] + sys.argv[1:])
o = train.trainer_options()
print(json.dumps({'options': o, 'lr': [float(decayed_learning_rate(o['learning_rate'], s,
                                                                  o['learning_rate_decay_factor'],
                                                                  o['decay_steps'])) for s in (0, 3, 4, 9, 1000)]}))
'''


def _run(args, script=None, cwd=REPO):
  cmd = [sys.executable] + (['-c', script] if script else [os.path.join(REPO, 'train.py')]) + list(args)
  return subprocess.run(cmd, capture_output=True, text=True, cwd=cwd, env=dict(os.environ, PYTHONPATH=REPO))


def _schedule(*args):
  res = _run(args, _SCHEDULE)
  assert res.returncode == 0, res.stderr[-2000:]
  return json.loads(res.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize('args', [(), ('--learning_rate_decay_factor=0.5',), ('--decay_steps=4',),
                                  ('--learning_rate_decay_factor=0.5', '--num_epochs_per_decay=0.1')])
def test_no_decay_without_both_flags(args):
  got = _schedule('--learning_rate=0.01', *args)
  assert got['lr'] == [float(np.float32(0.01))] * 5


def test_decay_steps_passed_through():
  got = _schedule('--learning_rate=0.01', '--learning_rate_decay_factor=0.5', '--decay_steps=4', '--optimizer=adam')
  assert got['options']['decay_steps'] == 4 and got['options']['learning_rate_decay_factor'] == 0.5
  assert got['options']['optimizer'] == 'adam'
  lr = np.float32(0.01)
  want = [lr, lr, np.float32(lr * np.float32(0.5)), np.float32(lr * np.float32(0.25)),
          np.float32(lr * np.power(np.float32(0.5), np.float32(250), dtype=np.float32))]
  assert got['lr'] == [float(v) for v in want]


def test_unknown_volume_name_is_refused(tmp_path):
  np.save(str(tmp_path / 'image.npy'), np.zeros((40, 40, 40), np.uint8))
  np.save(str(tmp_path / 'labels.npy'), np.ones((40, 40, 40), np.int64))
  with gzip.open(str(tmp_path / 'coords'), 'wb') as f:
    for name in (b'vol', b'other'):
      data = _example((20, 20, 20), name)
      f.write(struct.pack('<Q', len(data)) + b'\0' * 4 + data + b'\0' * 4)
  res = _run(['--train_coords', str(tmp_path / 'coords'), '--data_volumes', 'vol:%s:' % (tmp_path / 'image.npy'),
              '--label_volumes', 'vol:%s:' % (tmp_path / 'labels.npy'), '--image_mean', '128', '--image_stddev', '33',
              '--model_args', '{"depth": 1, "fov_size": [9, 9, 9], "deltas": [2, 2, 2]}',
              '--train_dir', str(tmp_path / 'train')], cwd=str(tmp_path))
  assert res.returncode != 0
  assert "coordinates name volumes without data or labels: ['other']" in res.stderr
  assert not (tmp_path / 'train').exists()
