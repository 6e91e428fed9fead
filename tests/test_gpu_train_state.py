"""Saving and restoring training state on the device: the trainer's and the example loop's blobs continue bit for bit
after a restore into fresh objects, their refusals change nothing, and train.py resumes across processes and starts
from saved weights.  GPU."""

import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import examples_oracle as eo
from test_gpu_examples import case_loop, small_net
from test_train_state import fib25_tf_checkpoint
from ffn_b200 import _lib, tf_checkpoint
from ffn_b200.training import examples as ex
from ffn_b200.training.trainer import Trainer

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIB25_NPZ = os.path.join(REPO, 'tests', 'golden', 'fib25_convstack.npz')

# exk::State of ffn_b200/csrc/example_kernels.cuh, the first payload section of an example loop blob
STATE_DTYPE = np.dtype([('off', '<i4', (3,)), ('k', '<i4'), ('head', '<i4'), ('tail', '<i4'), ('active', '<i4'),
                        ('pad', '<i4'), ('example', '<i8')])


def fnv1a64(data) -> int:
  h = 0xcbf29ce484222325
  for b in bytes(data):
    h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
  return h


def payload_at(blob) -> int:
  return 32 + 8 * int(np.frombuffer(blob[12:16].tobytes(), '<u4')[0])


def resign(blob):
  blob[24:32] = np.frombuffer(struct.pack('<Q', fnv1a64(blob[32:])), np.uint8)
  return blob


def loop_states(blob, batch):
  o = payload_at(blob)
  return np.frombuffer(blob[o:o + STATE_DTYPE.itemsize * batch].tobytes(), STATE_DTYPE).copy()


def with_states(blob, states):
  out = blob.copy()
  o = payload_at(out)
  out[o:o + states.nbytes] = np.frombuffer(states.tobytes(), np.uint8)
  return resign(out)


def with_ecoords(blob, batch, coords):
  out = blob.copy()
  o = payload_at(out) + STATE_DTYPE.itemsize * batch
  out[o:o + coords.nbytes] = np.frombuffer(coords.tobytes(), np.uint8)
  return resign(out)


def loop_ecoords(blob, batch):
  o = payload_at(blob) + STATE_DTYPE.itemsize * batch
  return np.frombuffer(blob[o:o + _lib.EXAMPLE_COORD_DTYPE.itemsize * batch].tobytes(), _lib.EXAMPLE_COORD_DTYPE).copy()


def assert_same_tracker(a, b):
  for f in ('steps', 'fov_voxels', 'patches', 'eval_voxels', 'patch_loss', 'coords'):
    assert getattr(a, f) == getattr(b, f), f
  np.testing.assert_array_equal(a.prediction_counts, b.prediction_counts)
  assert a.moves.keys() == b.moves.keys()
  for r in a.moves:
    np.testing.assert_array_equal(a.moves[r], b.moves[r])
  assert len(a.planes) == len(b.planes)
  for pa, pb in zip(a.planes, b.planes):
    for x, y in zip(pa, pb):
      for u, v in zip(x, y):
        np.testing.assert_array_equal(u, v)


def assert_same_weights(ta, tb):
  wa, wb = ta.weights(), tb.weights()
  for a, b in zip(wa[0] + wa[1], wb[0] + wb[1]):
    np.testing.assert_array_equal(a, b)


def restored_loop(c, state, pos):
  loop = case_loop(c)
  loop.stream.pos = pos
  loop.set_state(state)
  return loop


@pytest.mark.parametrize('optimizer', ['sgd', 'momentum', 'adam'])
def test_trainer_round_trip(optimizer):
  c = eo.case_setup(eo.cases()[0])
  kw = dict(fov_zyx=c['fov'], optimizer=optimizer, learning_rate=0.05, learning_rate_decay_factor=0.5, decay_steps=4,
            batch_size=4)
  ta = Trainer(*small_net(2, 5), **kw)
  warm = case_loop(c)
  ta.train(warm, 6)
  blob = ta.get_state()
  tb = Trainer(*small_net(2, 6), **kw)
  tb.set_state(blob)
  assert tb.global_step == 6 and tb.current_learning_rate() == ta.current_learning_rate()
  la, lb = case_loop(c), case_loop(c)
  np.testing.assert_array_equal(ta.train(la, 9), tb.train(lb, 9))
  assert ta.global_step == tb.global_step == 15
  assert ta.current_learning_rate() == tb.current_learning_rate()
  assert_same_weights(ta, tb)
  np.testing.assert_array_equal(ta.get_state(), tb.get_state())
  for o in (ta, tb, warm, la, lb):
    o.close()


@pytest.mark.parametrize('i', range(len(eo.cases())))
def test_loop_round_trip(i):
  """Saves at step boundaries (one with a max_pred_moves element mid-example with a queued move) and once between
  next() and update(); every restored loop continues as the saved one, which itself stays equal to the oracle."""
  c = eo.case_setup(eo.cases()[i])
  coords = eo.as_coords(c['rows'])
  o = eo.ExampleLoopOracle(c['volumes'], c['offset_scale'], c['fov'], c['deltas'], c['batch'], c['policy'],
                           c['fov_moves'], ex.seed_logits(0.05), ex.thresholds(c['threshold']), c['shifts'])
  main = case_loop(c)
  rng = np.random.RandomState(c['logit_seed'])
  followers = []
  queued = False
  pos = 0
  for step in range(eo.N_STEPS):
    want = o.next(coords[pos:])
    pos += want[5]
    got = main.next()
    for k, g, w in zip(('seed', 'image', 'labels', 'offsets', 'example'), got, want):
      np.testing.assert_array_equal(g, w, err_msg='%s at step %d' % (k, step))
    for f in followers:
      for k, g, w in zip(('seed', 'image', 'labels', 'offsets', 'example'), f.next(), got):
        np.testing.assert_array_equal(g, w, err_msg='restored loop: %s at step %d' % (k, step))
    if step == 13:   # between next() and update(): the paste uses the restored offsets
      followers.append(restored_loop(c, main.get_state(), main.stream.pos))
    lg = eo.step_logits(rng, c)
    o.update(lg)
    for lp in [main] + followers:
      lp.update(lg)
    state = main.get_state()
    st = loop_states(state['device'], c['batch'])
    mid = c['policy'] == 'max_pred_moves' and bool(((st['head'] < st['tail']) & (st['active'] == 1)).any())
    if step in (2, 21) or (mid and not queued):
      queued |= mid
      followers.append(restored_loop(c, state, main.stream.pos))
  assert queued or c['policy'] == 'fixed'
  assert len(followers) >= 3
  for f in followers:
    np.testing.assert_array_equal(f.seeds(), main.seeds())
    assert f.consumed == main.consumed
    assert_same_tracker(f.tracker(), main.tracker())
    f.close()
  np.testing.assert_array_equal(main.seeds(), o.seeds())
  main.close()


def _stream_loop(c, seed):
  stream = ex.ExampleStream(c['rows'][:, 0], c['rows'][:, 1:4], c['permutable'], c['reflectable'], seed=seed)
  vols = {'vol%d' % i: v for i, v in enumerate(c['volumes'])}
  os_map = {'vol%d' % i: v for i, v in enumerate(c['offset_scale'])}
  return ex.ExampleLoop(vols, stream, c['fov'], c['deltas'], c['batch'], c['policy'], c['fov_moves'], 0.05,
                        c['threshold'], c['shifts'], os_map)


@pytest.mark.parametrize('policy', ['fixed', 'max_pred_moves'])
def test_train_split_by_save_and_restore(policy):
  """train(2n) equals train(n), a save, both handles closed, a restore into new objects and train(n)."""
  c = eo.case_setup([k for k in eo.cases() if k[3] == policy][0])
  kw = dict(fov_zyx=c['fov'], optimizer='adam', learning_rate=0.01, learning_rate_decay_factor=0.7, decay_steps=10,
            batch_size=c['batch'])
  n = 37
  ta, la = Trainer(*small_net(2, 5), **kw), _stream_loop(c, 7)
  want = ta.train(la, 2 * n)
  tb, lb = Trainer(*small_net(2, 5), **kw), _stream_loop(c, 7)
  first = tb.train(lb, n)
  saved = tb.get_state(), lb.get_state(), lb.stream.get_state()
  tb.close()
  lb.close()
  tc, lc = Trainer(*small_net(2, 9), **kw), _stream_loop(c, 8)
  tc.set_state(saved[0])
  lc.stream.set_state(saved[2])
  lc.set_state(saved[1])
  second = tc.train(lc, n)
  np.testing.assert_array_equal(np.concatenate([first, second]), want)
  assert tc.global_step == ta.global_step == 2 * n
  assert_same_weights(ta, tc)
  np.testing.assert_array_equal(lc.seeds(), la.seeds())
  assert_same_tracker(lc.tracker(), la.tracker())
  assert lc.consumed == la.consumed
  np.testing.assert_array_equal(lc.entries(8), la.entries(8))
  for o in (ta, la, tc, lc):
    o.close()


def test_trainer_refusals():
  c = eo.case_setup(eo.cases()[0])
  kw = dict(fov_zyx=c['fov'], learning_rate=0.05, batch_size=4)
  src = Trainer(*small_net(2, 5), optimizer='sgd', **kw)
  src.train(case_loop(c), 2)
  blob = src.get_state()
  flipped = blob.copy()
  flipped[-5] ^= 1
  target, twin = (Trainer(*small_net(2, 6), optimizer='sgd', **kw) for _ in range(2))
  for t, b, msg in ((Trainer(*small_net(1, 6), optimizer='sgd', **kw), blob, 'another depth'),
                    (Trainer(*small_net(2, 6), optimizer='adam', **kw), blob, 'another optimizer'),
                    (target, blob[:-1], 'truncated'), (target, blob[:20], 'truncated'),
                    (target, flipped, 'checksum'), (target, blob[::-1].copy(), 'bad magic')):
    with pytest.raises(RuntimeError, match=msg):
      t.set_state(b)
  la, lb = case_loop(c), case_loop(c)
  np.testing.assert_array_equal(target.train(la, 3), twin.train(lb, 3))
  assert target.global_step == twin.global_step == 3
  assert_same_weights(target, twin)


def _variant(c, **kw):
  v = dict(c)
  v.update(kw)
  return v


def test_loop_refusals():
  c = eo.case_setup(eo.cases()[0])
  src = case_loop(c)
  rng = np.random.RandomState(1)
  for _ in range(5):
    src.next()
    src.update(eo.step_logits(rng, c))
  state = src.get_state()
  blob = state['device']
  b = c['batch']
  vols = list(c['volumes'])
  vols[0] = (vols[0][0][:, :, :-1], vols[0][1][:, :, :-1])
  max_pred = _variant(c, policy='max_pred_moves')
  others = ((_variant(c, batch=2), 'another batch'), (_variant(c, fov=(9, 9, 9)), 'another field of view'),
            (max_pred, 'another policy'), (_variant(c, shifts=c['shifts'][::-1].copy()), 'another shift list'),
            (_variant(c, volumes=vols), 'another volume 0 image shape'))
  for v, msg in others:
    loop = case_loop(v)
    with pytest.raises(RuntimeError, match=msg):
      loop.set_state(state)
    loop.close()

  target, twin = case_loop(c), case_loop(c)
  flipped = blob.copy()
  flipped[len(blob) // 2] ^= 0x10
  st = loop_states(blob, b)
  assert (st['active'] == 1).all()
  bad = []
  for field, value, msg in (('k', len(c['shifts']) + 2, 'k = '), ('k', -1, 'k = '), ('tail', 10**6, 'tail'),
                            ('head', st['tail'][1] + 1, 'head'), ('off', (0, 0, 99), 'offset')):
    s = st.copy()
    s[field][1] = value
    bad.append((with_states(blob, s), msg))
  ec = loop_ecoords(blob, b)
  ec['center_xyz'][2] = (0, 0, 0)
  bad.append((with_ecoords(blob, b, ec), 'leaves volume'))
  ec = loop_ecoords(blob, b)
  ec['volume'][0] = 9
  bad.append((with_ecoords(blob, b, ec), 'unknown volume'))
  for data, msg in [(blob[:-1], 'truncated'), (np.concatenate([blob, blob[:3]]), 'truncated'),
                    (flipped, 'checksum')] + bad:
    with pytest.raises(RuntimeError, match=msg):
      target.set_state(dict(state, device=data))
  # a re-signed but unchanged blob passes: the refusals above are the fields', not the signing's
  twin_state = case_loop(c)
  twin_state.set_state(dict(state, device=resign(blob.copy())))
  twin_state.close()
  rng = np.random.RandomState(2)
  for step in range(6):
    for k, g, w in zip(('seed', 'image', 'labels', 'offsets', 'example'), target.next(), twin.next()):
      np.testing.assert_array_equal(g, w, err_msg='%s at step %d' % (k, step))
    lg = eo.step_logits(rng, c)
    target.update(lg)
    twin.update(lg)
  np.testing.assert_array_equal(target.seeds(), twin.seeds())
  assert_same_tracker(target.tracker(), twin.tracker())
  assert target.consumed == twin.consumed
  for o in (src, target, twin):
    o.close()


@pytest.fixture(scope='module')
def phantom(tmp_path_factory):
  from ffn_b200 import coordinates
  from ffn_b200.synthetic import voronoi_phantom
  d = tmp_path_factory.mktemp('phantom')
  image, cells = voronoi_phantom((128, 128, 128), 3, return_cells=True, cell_volume=20000.0)
  np.save(str(d / 'image.npy'), image)
  np.save(str(d / 'labels.npy'), cells.astype(np.int64))
  part = np.full(cells.shape, 255, np.uint8)
  lattice = np.s_[24:104:4, 24:104:4, 24:104:4]
  part[lattice] = np.where(cells[lattice] > 0, cells[lattice] % 4, 255)
  np.random.seed(0)
  coordinates.build_coordinates([('vol', part)], (24, 24, 24), str(d / 'coords'))
  return d


def _train_py(data, train_dir, *args):
  cmd = [sys.executable, os.path.join(REPO, 'train.py'), '--train_coords', str(data / 'coords'),
         '--data_volumes', 'vol:%s:' % (data / 'image.npy'), '--label_volumes', 'vol:%s:' % (data / 'labels.npy'),
         '--image_mean', '128', '--image_stddev', '33', '--train_dir', str(train_dir)] + list(args)
  return subprocess.run(cmd, capture_output=True, text=True, cwd=str(data), env=dict(os.environ, PYTHONPATH=REPO))


def _same_npz(a, b):
  with np.load(str(a)) as x, np.load(str(b)) as y:
    assert sorted(x.files) == sorted(y.files)
    for k in x.files:
      assert x[k].dtype == y[k].dtype and x[k].shape == y[k].shape, k
      assert x[k].tobytes() == y[k].tobytes(), k


def test_train_py_resumes_across_processes(phantom, tmp_path):
  """--max_steps 120 in one run equals 60 then 120 in two (50 steps per call, so the calls split differently)."""
  flags = ['--model_args', '{"depth": 2, "fov_size": [17, 17, 17], "deltas": [4, 4, 4]}', '--optimizer', 'adam',
           '--learning_rate', '0.003', '--batch_size', '4', '--fov_policy', 'max_pred_moves']
  one, two = tmp_path / 'one', tmp_path / 'two'
  res = _train_py(phantom, one, '--max_steps', '120', *flags)
  assert res.returncode == 0, res.stderr[-3000:]
  res = _train_py(phantom, two, '--max_steps', '60', *flags)
  assert res.returncode == 0, res.stderr[-3000:]
  assert (two / 'train_state-60.npz').exists() and 'Resuming' not in res.stderr
  res = _train_py(phantom, two, '--max_steps', '120', *flags)
  assert res.returncode == 0, res.stderr[-3000:]
  assert 'Resuming from step 60' in res.stderr
  assert (one / 'losses.npy').read_bytes() == (two / 'losses.npy').read_bytes()
  assert len(np.load(str(two / 'losses.npy'))) == 120
  _same_npz(one / 'model.ckpt-120.npz', two / 'model.ckpt-120.npz')
  before = sorted(os.listdir(str(two)))
  res = _train_py(phantom, two, '--max_steps', '180', *flags[:-3], '2', *flags[-2:])
  assert res.returncode != 0
  assert '--batch_size differs from the run saved in' in res.stderr, res.stderr[-3000:]
  assert sorted(os.listdir(str(two))) == before


@pytest.mark.parametrize('kind', ['npz', 'tf'])
def test_train_py_init_checkpoint(phantom, tmp_path, kind):
  path = FIB25_NPZ if kind == 'npz' else fib25_tf_checkpoint(tmp_path)
  fib25 = '{"depth": 12, "fov_size": [33, 33, 33], "deltas": [8, 8, 8]}'
  res = _train_py(phantom, tmp_path / 'train', '--init_checkpoint', path, '--model_args', fib25, '--max_steps', '0')
  assert res.returncode == 0, res.stderr[-3000:]
  assert 'Starting from the weights of %s' % path in res.stderr
  w, b = tf_checkpoint.load_convstack_npz(str(tmp_path / 'train' / 'model.ckpt-0.npz'))
  ww, bb = tf_checkpoint.load_convstack_npz(FIB25_NPZ)
  assert len(w) == len(ww) == 25
  for x, y in zip(w + b, ww + bb):
    assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
  res = _train_py(phantom, tmp_path / 'nine', '--init_checkpoint', path, '--model_args', fib25.replace('12', '9'),
                  '--max_steps', '0')
  assert res.returncode != 0 and 'depth 9' in res.stderr, res.stderr[-3000:]
  assert not (tmp_path / 'nine').exists()
