"""The device example loop against the oracle bit for bit, Trainer.train against next/step/update, the refusals,
destroy order and train.py end to end.  GPU."""

import os
import subprocess
import sys

import numpy as np
import pytest

import examples_oracle as eo
from ffn_b200 import _lib
from ffn_b200.training import examples as ex
from ffn_b200.training.trainer import Trainer

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Rows:
  """An ExampleStream stand-in that hands out fixed entries in order."""

  def __init__(self, coords, permutable=(0, 1, 2), reflectable=(0, 1, 2)):
    self.coords, self.pos = coords, 0
    self.permutable, self.reflectable = np.array(permutable), np.array(reflectable)

  def take(self, n):
    out = self.coords[self.pos:self.pos + n]
    self.pos += n
    assert len(out) == n
    return out


def case_loop(c, coords=None):
  vols = {'vol%d' % i: v for i, v in enumerate(c['volumes'])}
  os_map = {'vol%d' % i: v for i, v in enumerate(c['offset_scale'])}
  rows = _Rows(eo.as_coords(c['rows']) if coords is None else coords, c['permutable'], c['reflectable'])
  return ex.ExampleLoop(vols, rows, c['fov'], c['deltas'], c['batch'], c['policy'], c['fov_moves'], 0.05,
                        c['threshold'], c['shifts'], os_map)


@pytest.mark.parametrize('i', range(len(eo.cases())))
def test_device_loop_equals_oracle(i):
  c = eo.case_setup(eo.cases()[i])
  o = eo.ExampleLoopOracle(c['volumes'], c['offset_scale'], c['fov'], c['deltas'], c['batch'], c['policy'],
                           c['fov_moves'], ex.seed_logits(0.05), ex.thresholds(c['threshold']), c['shifts'])
  loop = case_loop(c)
  coords = eo.as_coords(c['rows'])
  rng = np.random.RandomState(c['logit_seed'])
  pos = 0
  for step in range(eo.N_STEPS):
    want = o.next(coords[pos:])
    pos += want[5]
    before = loop.consumed
    got = loop.next()
    for k, g, w in zip(('seed', 'image', 'labels', 'offsets', 'example'), got, want):
      np.testing.assert_array_equal(g, w, err_msg='%s at step %d' % (k, step))
    assert loop.consumed - before == want[5]
    lg = eo.step_logits(rng, c)
    o.update(lg)
    loop.update(lg)
  np.testing.assert_array_equal(loop.seeds(), o.seeds())
  loop.close()


def small_net(depth, seed):
  rng = np.random.RandomState(seed)
  ws = [(rng.standard_normal((3, 3, 3, 2 if i == 0 else 32, 32)) * 0.05).astype(np.float32) for i in range(2 * depth)]
  ws.append((rng.standard_normal((1, 1, 1, 32, 1)) * 0.1).astype(np.float32))
  bs = [np.zeros(32, np.float32) for _ in range(2 * depth)] + [np.array([0.5], np.float32)]
  return ws, bs


@pytest.mark.parametrize('optimizer,policy', [('sgd', 'fixed'), ('adam', 'max_pred_moves')])
def test_train_equals_next_step_update(optimizer, policy):
  case = [k for k in eo.cases() if k[3] == policy][0]
  c = eo.case_setup(case)
  c['batch'] = 3
  ws, bs = small_net(2, 5)
  kw = dict(fov_zyx=c['fov'], optimizer=optimizer, learning_rate=0.05, learning_rate_decay_factor=0.5,
            decay_steps=4, batch_size=4)
  ta, tb = Trainer(ws, bs, **kw), Trainer(ws, bs, **kw)
  la, lb = case_loop(c), case_loop(c)
  losses = np.concatenate([ta.train(la, 7), ta.train(la, 5)])
  want = []
  for _ in range(12):
    seed, image, labels, _, _ = lb.next()
    logits, loss = tb.step(seed, image, labels)
    lb.update(logits)
    want.append(loss)
  np.testing.assert_array_equal(losses, np.array(want))
  assert la.consumed == lb.consumed and ta.global_step == tb.global_step == 12
  wa, wb = ta.weights(), tb.weights()
  for a, b in zip(wa[0] + wa[1], wb[0] + wb[1]):
    np.testing.assert_array_equal(a, b)
  np.testing.assert_array_equal(la.seeds(), lb.seeds())
  for t in (ta, tb):
    t.close()


def _basic():
  c = eo.case_setup(eo.cases()[0])
  return c, {'vol%d' % i: v for i, v in enumerate(c['volumes'])}, {'vol%d' % i: v for i, v in
                                                                   enumerate(c['offset_scale'])}


def test_refusals():
  c, vols, osm = _basic()
  coords = eo.as_coords(c['rows'])
  rows = lambda co: _Rows(co, c['permutable'], c['reflectable'])
  mk = lambda **k: ex.ExampleLoop(vols, rows(coords), c['fov'], c['deltas'], k.pop('batch', 4), 'fixed', 1,
                                  k.pop('seed_pad', 0.05), k.pop('threshold', 0.9), None, osm)
  for kw, msg in (({'seed_pad': 1.0}, 'seed_pad'), ({'seed_pad': 0.0}, 'seed_pad'),
                  ({'threshold': 0.95}, 'fresh seed'), ({'batch': 33}, 'batch')):
    with pytest.raises(RuntimeError, match=msg):
      mk(**kw)
  mk(threshold=0.9499999).close()
  with pytest.raises(RuntimeError, match='equal patch extents'):
    ex.ExampleLoop(vols, _Rows(coords), (7, 7, 9), c['deltas'], 2, 'fixed', 1, 0.05, 0.9, None, osm)
  with pytest.raises(TypeError, match='uint8'):
    ex.ExampleLoop({'vol0': (vols['vol0'][0].astype(np.float32), vols['vol0'][1])}, _Rows(coords), c['fov'],
                   c['deltas'], 2, offset_scale=osm)
  with pytest.raises(TypeError, match='integers'):
    ex.ExampleLoop({'vol0': (vols['vol0'][0], vols['vol0'][1].astype(np.float32))}, _Rows(coords), c['fov'],
                   c['deltas'], 2, offset_scale=osm)
  with pytest.raises(ValueError, match='2\\^63'):
    big = vols['vol0'][1].astype(np.uint64)
    big[0, 0, 0] = 2**63
    ex.ExampleLoop({'vol0': (vols['vol0'][0], big)}, _Rows(coords), c['fov'], c['deltas'], 2, offset_scale=osm)
  # stream entries: an unknown volume, a crop leaving its volume, a disallowed permutation
  for field, value, msg in (('volume', 7, 'unknown volume'), ('center_xyz', (0, 0, 0), 'leaves volume'),
                            ('permutation_zyx', (1, 0, 2), 'not permutable')):
    bad = coords.copy()
    bad[field][1] = value
    loop = mk()
    loop.stream = rows(bad)
    with pytest.raises(RuntimeError, match=msg):
      loop.next()
    loop.close()
  # a trainer of another field of view, a batch above its max_batch
  ws, bs = small_net(1, 0)
  loop = mk()
  for kw, msg in (({'fov_zyx': (9, 9, 9), 'batch_size': 4}, 'field of view'),
                  ({'fov_zyx': c['fov'], 'batch_size': 2}, 'max_batch')):
    t = Trainer(ws, bs, **kw)
    with pytest.raises(RuntimeError, match=msg):
      t.train(loop, 1)
    t.close()
  loop.close()


@pytest.mark.parametrize('trainer_first', [True, False])
def test_destroy_order(trainer_first):
  c, vols, osm = _basic()
  ws, bs = small_net(1, 0)
  t = Trainer(ws, bs, fov_zyx=c['fov'], batch_size=4)
  loop = ex.ExampleLoop(vols, _Rows(eo.as_coords(c['rows'])), c['fov'], c['deltas'], 4, offset_scale=osm)
  t.train(loop, 2)
  first, second = (t, loop) if trainer_first else (loop, t)
  first.close()
  if second is loop:
    loop.next()
  else:
    z = np.zeros((4,) + c['fov'], np.float32)
    t.step(z, z, z)
  second.close()


def test_reader_reads_what_build_coordinates_writes(tmp_path):
  """inputs.load_coordinates against a protobuf parse of the same file, record for record, over several files."""
  from test_coordinates import read_coordinates
  from ffn_b200 import coordinates
  from ffn_b200.training import inputs
  rng = np.random.RandomState(4)
  want_c, want_n = [], []
  for k, names in enumerate((['alpha', 'Zellkörper_体積'], ['beta'])):
    vols = [(n, rng.choice(np.array([0, 1, 2, 3, 255], np.uint8), size=(14 + i, 16, 18))) for i, n in enumerate(names)]
    path = str(tmp_path / ('coords-%d' % k))
    np.random.seed(k)
    coordinates.build_coordinates(vols, (2, 3, 4), path)
    c, n = read_coordinates(path)
    want_c.append(c)
    want_n += [x.decode('utf-8') for x in n]
  centers, names = inputs.load_coordinates(str(tmp_path / 'coords-*'))
  np.testing.assert_array_equal(centers, np.concatenate(want_c))
  assert names == want_n and len(names) > 100


def test_train_py_end_to_end(tmp_path):
  from ffn_b200 import coordinates, engine as eng, tf_checkpoint
  from ffn_b200.synthetic import voronoi_phantom
  from ffn_b200.training import inputs
  image, cells = voronoi_phantom((128, 128, 128), 3, return_cells=True, cell_volume=20000.0)
  np.save(str(tmp_path / 'image.npy'), image)
  np.save(str(tmp_path / 'labels.npy'), cells.astype(np.int64))
  part = np.full(cells.shape, 255, np.uint8)   # a sparse lattice of training coordinates keeps the file small
  lattice = np.s_[24:104:4, 24:104:4, 24:104:4]
  part[lattice] = np.where(cells[lattice] > 0, cells[lattice] % 4, 255)
  np.random.seed(0)
  coordinates.build_coordinates([('vol', part)], (24, 24, 24), str(tmp_path / 'coords'))
  centers, names = inputs.load_coordinates(str(tmp_path / 'coords'))
  assert len(centers) > 0 and set(names) == {'vol'}
  assert (centers >= 24).all() and (centers < 104).all()
  env = dict(os.environ, PYTHONPATH=REPO)
  cmd = [sys.executable, os.path.join(REPO, 'train.py'), '--train_coords', str(tmp_path / 'coords'),
         '--data_volumes', 'vol:%s:' % (tmp_path / 'image.npy'), '--label_volumes', 'vol:%s:' % (tmp_path / 'labels.npy'),
         '--model_args', '{"depth": 2, "fov_size": [17, 17, 17], "deltas": [4, 4, 4]}', '--image_mean', '128',
         '--image_stddev', '33', '--train_dir', str(tmp_path / 'train'), '--max_steps', '200', '--optimizer', 'adam',
         '--learning_rate', '0.003', '--batch_size', '4']
  res = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), env=env)
  assert res.returncode == 0, res.stderr[-3000:]
  losses = np.load(str(tmp_path / 'train' / 'losses.npy'))
  assert len(losses) == 200 and np.isfinite(losses).all()
  assert losses[-50:].mean() < losses[:50].mean(), (losses[:50].mean(), losses[-50:].mean())
  w, b = tf_checkpoint.load_convstack_npz(str(tmp_path / 'train' / 'model.ckpt-200.npz'))
  e = eng.Engine(w, b, (17, 17, 17), (4, 4, 4), device=0)
  cv = eng.DeviceCanvas(e, image, eng.make_options(), 128.0, 33.0)
  st = cv.segment_at((64, 64, 64), max_steps=20)
  assert st.iters >= 1
  cv.close()
  e.close()
