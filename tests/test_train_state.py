"""Resuming train.py runs, on the CPU: the example stream's state round trip, the state files' retention and choice, the
run fingerprint's refusals before any device work, and --init_checkpoint's depth check (npz and TF checkpoints).
train.py runs as a subprocess, so that its absl flags stay out of this process."""

import gzip
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from test_examples_oracle import _example

from ffn_b200 import _lib, tf_checkpoint
from ffn_b200.training import examples as ex

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, 'tests', 'golden')
FIB25_NPZ = os.path.join(GOLDEN, 'fib25_convstack.npz')
# The index of the reference's FIB-25 TF1 checkpoint (its variable names, dtypes, shapes and offsets).  Its 2.5 MB data
# shard is not kept: fib25_tf_checkpoint rebuilds it from fib25_convstack.npz.  The depth check reads the index only.
FIB25_TF = os.path.join(GOLDEN, 'model.ckpt-27465036')


def fib25_tf_checkpoint(directory):
  """A copy of the FIB-25 TF1 checkpoint in `directory`: the reference's index, and a data shard holding each
  ConvStack variable's fib25_convstack.npz array at the offset the index gives it (zeros elsewhere).  Returns the
  prefix."""
  entries = tf_checkpoint.list_variables(FIB25_TF)
  w, b = tf_checkpoint.load_convstack_npz(FIB25_NPZ)
  layers = ['conv%d_%s' % (i, h) for i in range(12) for h in 'ab'] + ['conv_lom']
  arrays = {}
  for name, wi, bi in zip(layers, w, b):
    arrays['seed_update/%s/weights' % name] = wi
    arrays['seed_update/%s/biases' % name] = bi
  data = bytearray(max(e['offset'] + e['size'] for e in entries.values()))
  for name, a in arrays.items():
    e = entries[name]
    assert e['dtype'] == 1 and tuple(e['shape']) == a.shape and e['size'] == a.nbytes, name
    data[e['offset']:e['offset'] + e['size']] = a.astype('<f4').tobytes()
  prefix = os.path.join(str(directory), 'model.ckpt-27465036')
  with open(FIB25_TF + '.index', 'rb') as f, open(prefix + '.index', 'wb') as g:
    g.write(f.read())
  with open(prefix + '.data-00000-of-00001', 'wb') as f:
    f.write(bytes(data))
  return prefix


def _python(script, *args, cwd=REPO):
  return subprocess.run([sys.executable, '-c', script] + list(args), capture_output=True, text=True, cwd=cwd,
                        env=dict(os.environ, PYTHONPATH=REPO))


@pytest.mark.parametrize('permutable,reflectable', [((1, 2), (0, 1, 2)), ((0, 1, 2), ())])
def test_stream_state_round_trip_across_epochs(permutable, reflectable):
  rng = np.random.RandomState(3)
  vol, centers = rng.randint(0, 3, 7), rng.randint(0, 100, (7, 3))
  a = ex.ExampleStream(vol, centers, permutable, reflectable, seed=11)
  a.take(5)
  state = a.get_state()
  want = a.take(12)   # crosses two epoch boundaries
  b = ex.ExampleStream(vol, centers, permutable, reflectable, seed=99)
  b.take(3)
  b.set_state(state)
  np.testing.assert_array_equal(b.take(12), want)
  # a state taken exactly at an epoch boundary, and one before the first draw
  for n in (2, 0):
    c = ex.ExampleStream(vol, centers, permutable, reflectable, seed=5)
    c.take(n)
    s = c.get_state()
    d = ex.ExampleStream(vol, centers, permutable, reflectable, seed=6)
    d.set_state(s)
    np.testing.assert_array_equal(d.take(9), c.take(9))


def test_stream_state_refusals():
  a = ex.ExampleStream(np.zeros(4), np.zeros((4, 3)), seed=1)
  a.take(2)
  s = a.get_state()
  other = ex.ExampleStream(np.zeros(5), np.zeros((5, 3)), seed=1)
  with pytest.raises(ValueError, match='not a permutation'):
    other.set_state(s)
  with pytest.raises(ValueError, match='position'):
    a.set_state(dict(s, pos=np.int64(5)))
  np.testing.assert_array_equal(a.take(6), ex.ExampleStream(np.zeros(4), np.zeros((4, 3)), seed=1).take(8)[2:])


_FAKES = r'''
import json, os, sys
import numpy as np
import train
from ffn_b200 import _lib

class Stream:
  def get_state(self):
    return {'pos': np.int64(1), 'order': np.arange(3)}

class Loop:
  stream = Stream()
  def get_state(self):
    return {'device': np.zeros(8, np.uint8), 'pending': np.zeros(2, _lib.EXAMPLE_COORD_DTYPE), 'consumed': np.int64(4)}

class Trainer:
  global_step = 0
  def get_state(self):
    return np.full(16, self.global_step % 256, np.uint8)

d = sys.argv[1]
t = Trainer()
for step in (10, 20, 30, 40, 50, 60, 70, 80):
  t.global_step = step
  train.save_state(d, t, Loop(), [0.5] * step, {'batch_size': 4})
open(os.path.join(d, 'train_state-90.npz.tmp.npz'), 'w').close()   # a killed write
open(os.path.join(d, 'model.ckpt-900.npz'), 'w').close()
print(json.dumps({'files': sorted(os.listdir(d)), 'newest': train.newest_state(d),
                  'missing': train.newest_state(os.path.join(d, 'nothing'))}))
'''


def test_state_retention_and_newest(tmp_path):
  res = _python(_FAKES, str(tmp_path))
  assert res.returncode == 0, res.stderr[-3000:]
  got = json.loads(res.stdout.strip().splitlines()[-1])
  states = ['train_state-%d.npz' % s for s in (40, 50, 60, 70, 80)]
  assert sorted(f for f in got['files'] if f.startswith('train_state-') and f.endswith('0.npz')) == sorted(states)
  assert not [f for f in got['files'] if '.tmp' in f and f != 'train_state-90.npz.tmp.npz']
  assert got['newest'] == str(tmp_path / 'train_state-80.npz') and got['missing'] is None
  with np.load(str(tmp_path / 'train_state-80.npz')) as z:
    assert int(z['step']) == 80 and len(z['losses']) == 80 and int(z['loop_consumed']) == 4
    assert json.loads(str(z['fingerprint'])) == {'batch_size': 4}
    assert z['loop_pending'].dtype == _lib.EXAMPLE_COORD_DTYPE and int(z['stream_pos']) == 1


def _data(tmp_path, shape=(40, 40, 40), n_records=2):
  np.save(str(tmp_path / 'image.npy'), np.zeros(shape, np.uint8))
  np.save(str(tmp_path / 'labels.npy'), np.ones(shape, np.int64))
  with gzip.open(str(tmp_path / 'coords'), 'wb') as f:
    for _ in range(n_records):
      data = _example((20, 20, 20), b'vol')
      f.write(struct.pack('<Q', len(data)) + b'\0' * 4 + data + b'\0' * 4)


def _flags(tmp_path, *extra):
  return ['--train_coords', str(tmp_path / 'coords'), '--data_volumes', 'vol:%s:' % (tmp_path / 'image.npy'),
          '--label_volumes', 'vol:%s:' % (tmp_path / 'labels.npy'), '--image_mean', '128', '--image_stddev', '33',
          '--model_args', '{"depth": 1, "fov_size": [9, 9, 9], "deltas": [2, 2, 2]}',
          '--train_dir', str(tmp_path / 'train')] + list(extra)


# Writes the state file a run of these flags would leave at step 50 (its fingerprint only), as main() computes it.
_SAVED = r'''
import json, os, sys
import numpy as np
import train
from ffn_b200.training import inputs
train.FLAGS(['train.py'] + sys.argv[1:])
F = train.FLAGS
images, labels = train.parse_volumes(F.data_volumes), train.parse_volumes(F.label_volumes)
centers, names = inputs.load_coordinates(F.train_coords)
args = json.loads(F.model_args)
fp = train.run_fingerprint(args, images, labels, len(centers))
os.makedirs(F.train_dir)
np.savez(os.path.join(F.train_dir, 'train_state-50.npz'), fingerprint=np.array(json.dumps(fp, sort_keys=True)),
         step=np.int64(50))
'''


def _run_train(tmp_path, *args):
  return subprocess.run([sys.executable, os.path.join(REPO, 'train.py')] + list(args), capture_output=True, text=True,
                        cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=REPO))


@pytest.mark.parametrize('change,flag', [
    (('--batch_size', '2'), '--batch_size'), (('--fov_policy', 'max_pred_moves'), '--fov_policy'),
    (('--fov_moves', '2'), '--fov_moves'), (('--noshuffle_moves',), '--shuffle_moves'), (('--seed', '3'), '--seed'),
    (('--seed_pad', '0.1'), '--seed_pad'), (('--threshold', '0.8'), '--threshold'),
    (('--permutable_axes', '0,1,2'), '--permutable_axes'), (('--reflectable_axes', '0'), '--reflectable_axes'),
    (('--optimizer', 'adam'), '--optimizer'), (('--image_stddev', '30'), '--image_stddev'),
    (('--model_args', '{"depth": 2, "fov_size": [9, 9, 9], "deltas": [2, 2, 2]}'), '--model_args'),
    (('volume shape',), '--data_volumes / --label_volumes'), (('records',), '--train_coords'),
])
def test_fingerprint_refused_before_device_work(tmp_path, change, flag):
  _data(tmp_path)
  res = _python(_SAVED, *_flags(tmp_path), cwd=str(tmp_path))
  assert res.returncode == 0, res.stderr[-3000:]
  if change == ('volume shape',):
    _data(tmp_path, shape=(40, 40, 41))
    change = ()
  elif change == ('records',):
    _data(tmp_path, n_records=3)
    change = ()
  before = sorted(os.listdir(str(tmp_path / 'train')))
  res = _run_train(tmp_path, *_flags(tmp_path, '--max_steps', '100', *change))
  assert res.returncode != 0
  assert '%s differs from the run saved in' % flag in res.stderr, res.stderr[-3000:]
  assert sorted(os.listdir(str(tmp_path / 'train'))) == before


def test_resume_past_max_steps_writes_nothing(tmp_path):
  """A run already at --max_steps exits at once, with the flags that may change between runs changed."""
  _data(tmp_path)
  assert _python(_SAVED, *_flags(tmp_path), cwd=str(tmp_path)).returncode == 0
  before = sorted(os.listdir(str(tmp_path / 'train')))
  res = _run_train(tmp_path, *_flags(tmp_path, '--max_steps', '50', '--learning_rate', '0.5', '--momentum', '0.5',
                                     '--checkpoint_secs', '1', '--init_checkpoint', FIB25_NPZ))
  assert res.returncode == 0, res.stderr[-3000:]
  assert 'nothing to train' in res.stderr and '--init_checkpoint %s ignored' % FIB25_NPZ in res.stderr
  assert sorted(os.listdir(str(tmp_path / 'train'))) == before


@pytest.mark.parametrize('path,depth,msg', [
    (FIB25_NPZ, 9, 'holds 25 weight arrays; a network of depth 9'),
    (FIB25_TF, 9, 'has more residual modules'),
    (FIB25_TF, 13, 'has fewer residual modules'),
])
def test_init_checkpoint_of_another_depth_is_refused(tmp_path, path, depth, msg):
  _data(tmp_path)
  args = _flags(tmp_path, '--init_checkpoint', path, '--max_steps', '0')
  args[args.index('--model_args') + 1] = json.dumps({'depth': depth, 'fov_size': [33, 33, 33], 'deltas': [8, 8, 8]})
  res = _run_train(tmp_path, *args)
  assert res.returncode != 0
  assert msg in res.stderr, res.stderr[-3000:]
  assert not (tmp_path / 'train').exists()


def test_fib25_tf_checkpoint_equals_npz(tmp_path):
  """The FIB-25 TF1 checkpoint, laid out by the reference's own index, reads at depth 12 as the npz fixture bit for
  bit: every layer under its scope and name, in layer order."""
  w, b = tf_checkpoint.load_convstack_weights(fib25_tf_checkpoint(tmp_path), 12)
  ww, bb = tf_checkpoint.load_convstack_npz(FIB25_NPZ)
  assert len(w) == len(ww) == 25
  for x, y in zip(w + b, ww + bb):
    assert x.dtype == y.dtype and x.shape == y.shape
    np.testing.assert_array_equal(x, y)
