"""The device tracker (ffn_examples_tracker) against the tracker oracle bit for bit, Trainer.train against
n x (next, step, update) with the tracker read, reset and refusals, and train.py's event file.  GPU."""

import ctypes as C
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

import examples_oracle as eo
import tracker_oracle as to
from ffn_b200 import _lib
from ffn_b200.training import summary
from ffn_b200.training import tracker as tk
from ffn_b200.training.trainer import Trainer
from test_gpu_examples import case_loop, small_net

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = 2.0**-53


def loss_bound(o):
  """Device and oracle both sum float64 terms max(x, 0) - x z + log1p(exp(-|x|)), each within 8 u |m| of exact
  (m = max(x, 0) + |x z| + log1p(exp(-|x|)); u for the product, the difference and the sum, 2 u each for exp and
  log1p in CUDA's and the host's libm, passed on at most 1:1), in different orders: each sum of N terms adds at most
  (N - 1) u of the sum of |terms|, and the division u.  The patch means are added in the same order, each addition
  within u of the running sum."""
  n = int(np.prod(o.eval))
  return 2 * U64 * (n + 8 + o.patches) * o.loss_mag + 1e-300


def assert_same(got, want, o, msg):
  for k in ('steps', 'fov_voxels', 'patches', 'eval_voxels'):
    assert getattr(got, k) == getattr(want, k), (msg, k)
  np.testing.assert_array_equal(got.prediction_counts, want.prediction_counts, err_msg=msg)
  assert sorted(got.moves) == sorted(want.moves), msg
  for r in got.moves:
    np.testing.assert_array_equal(got.moves[r], want.moves[r], err_msg='%s radius %d' % (msg, r))
  assert abs(got.patch_loss - want.patch_loss) <= loss_bound(o), (msg, got.patch_loss, want.patch_loss)
  assert got.coords == want.coords, msg
  assert len(got.planes) == len(want.planes), msg
  for gp, wp in zip(got.planes, want.planes):
    for (gl, gg), (wl, wg) in zip(gp, wp):
      np.testing.assert_array_equal(gl, wl, err_msg=msg)
      np.testing.assert_array_equal(gg, wg, err_msg=msg)


@pytest.mark.parametrize('i', range(len(to.cases())))
def test_device_tracker_equals_oracle(i):
  c = eo.case_setup(to.cases()[i])
  o = to.make(c)
  loop = case_loop(c)
  coords = eo.as_coords(c['rows'])
  rng = np.random.RandomState(c['logit_seed'])
  pos = 0
  for step in range(eo.N_STEPS):
    pos += o.next(coords[pos:])[5]
    loop.next()
    lg = to.step_logits(rng, c)
    o.update(lg)
    loop.update(lg)
    reset = (step + 1) % to.SUMMARY_EVERY == 0
    assert_same(loop.tracker(reset=reset), o.state(), o, '%s step %d' % (c['tag'], step))
    if reset:
      o.reset()
  loop.close()


@pytest.mark.parametrize('policy', ['fixed', 'max_pred_moves'])
def test_train_leaves_the_same_tracker(policy):
  case = [k for k in to.cases() if k[3] == policy][0]
  c = eo.case_setup(case)
  c['batch'] = 3
  ws, bs = small_net(2, 5)
  kw = dict(fov_zyx=c['fov'], optimizer='adam', learning_rate=0.05, batch_size=4)
  ta, tb, tc = Trainer(ws, bs, **kw), Trainer(ws, bs, **kw), Trainer(ws, bs, **kw)
  la, lb, lc = case_loop(c), case_loop(c), case_loop(c)
  losses_a = np.concatenate([ta.train(la, 7), ta.train(la, 5)])
  for _ in range(12):
    seed, image, labels, _, _ = lb.next()
    logits, _ = tb.step(seed, image, labels)
    lb.update(logits)
  a, b = la.tracker(), lb.tracker()
  assert a.patches > 0
  for k in ('steps', 'fov_voxels', 'patches', 'eval_voxels', 'patch_loss', 'coords'):
    assert getattr(a, k) == getattr(b, k), k
  np.testing.assert_array_equal(a.prediction_counts, b.prediction_counts)
  for r in a.moves:
    np.testing.assert_array_equal(a.moves[r], b.moves[r])
  for pa, pb in zip(a.planes, b.planes):
    for x, y in zip(pa, pb):
      np.testing.assert_array_equal(np.array(x), np.array(y))
  # reading and resetting between calls changes nothing the loop or the trainer computes
  losses_c = []
  for n in (4, 3, 5):
    if losses_c:
      lc.tracker(reset=True)
    losses_c.append(tc.train(lc, n))
  np.testing.assert_array_equal(np.concatenate(losses_c), losses_a)
  assert la.consumed == lc.consumed
  np.testing.assert_array_equal(la.seeds(), lc.seeds())
  for x, y in zip(sum(ta.weights(), []), sum(tc.weights(), [])):
    np.testing.assert_array_equal(x, y)
  # the reset state counts only the last call
  last = lc.tracker()
  assert last.steps == 5
  for t in (ta, tb, tc):
    t.close()
  for loop in (la, lb, lc):
    loop.close()


def test_reset_and_refusals():
  c = eo.case_setup(to.cases()[0])
  loop = case_loop(c)
  rng = np.random.RandomState(c['logit_seed'])
  for _ in range(eo.N_STEPS):
    loop.next()
    loop.update(to.step_logits(rng, c))
  s = loop.tracker(reset=True)
  assert s.patches > 0 and s.planes and sum(m.sum() for m in s.moves.values()) > 0
  e = loop.tracker()
  assert e.steps == e.patches == e.eval_voxels == 0 and e.patch_loss == 0.0 and not e.planes and not e.coords
  assert not e.prediction_counts.any() and all(not m.any() for m in e.moves.values())
  assert tk.summaries(e, ['vol0', 'vol1']) == []
  lib = _lib.load()
  counts, n = _lib.TrackerCounts(), C.c_int32()
  moves = np.zeros((16, 3), np.int64)
  planes = np.zeros((16, 10000), np.float32)
  coords = np.zeros(16, _lib.EXAMPLE_COORD_DTYPE)
  calls = [
      ((None, C.byref(counts), _lib.ptr(moves), 16, None, None, C.byref(n), 0), 'null examples'),
      ((loop.handle, None, _lib.ptr(moves), 16, None, None, C.byref(n), 0), 'null argument'),
      ((loop.handle, C.byref(counts), None, 16, None, None, C.byref(n), 0), 'null argument'),
      ((loop.handle, C.byref(counts), _lib.ptr(moves), 16, None, None, None, 0), 'null argument'),
      ((loop.handle, C.byref(counts), _lib.ptr(moves), max(loop.radii), None, None, C.byref(n), 0), 'radii'),
      ((loop.handle, C.byref(counts), _lib.ptr(moves), 16, _lib.ptr(planes), None, C.byref(n), 0), 'both'),
      ((loop.handle, C.byref(counts), _lib.ptr(moves), 16, None, _lib.ptr(coords), C.byref(n), 0), 'both'),
  ]
  for args, msg in calls:
    assert lib.ffn_examples_tracker(*args) != 0
    assert msg in lib.ffn_last_error().decode(), (msg, lib.ffn_last_error())
  # without planes the counts are still read
  assert lib.ffn_examples_tracker(loop.handle, C.byref(counts), _lib.ptr(moves), 16, None, None, C.byref(n), 0) == 0
  loop.close()


def test_train_py_writes_summaries(tmp_path):
  from ffn_b200 import coordinates
  from ffn_b200.synthetic import voronoi_phantom
  image, cells = voronoi_phantom((128, 128, 128), 3, return_cells=True, cell_volume=20000.0)
  np.save(str(tmp_path / 'image.npy'), image)
  np.save(str(tmp_path / 'labels.npy'), cells.astype(np.int64))
  part = np.full(cells.shape, 255, np.uint8)
  lattice = np.s_[24:104:4, 24:104:4, 24:104:4]
  part[lattice] = np.where(cells[lattice] > 0, cells[lattice] % 4, 255)
  np.random.seed(0)
  coordinates.build_coordinates([('vol', part)], (24, 24, 24), str(tmp_path / 'coords'))
  for policy in ('fixed', 'max_pred_moves'):
    train_dir = tmp_path / policy
    cmd = [sys.executable, os.path.join(REPO, 'train.py'), '--train_coords', str(tmp_path / 'coords'),
           '--data_volumes', 'vol:%s:' % (tmp_path / 'image.npy'),
           '--label_volumes', 'vol:%s:' % (tmp_path / 'labels.npy'),
           '--model_args', '{"depth": 2, "fov_size": [17, 17, 17], "deltas": [4, 4, 4]}', '--image_mean', '128',
           '--image_stddev', '33', '--train_dir', str(train_dir), '--max_steps', '100', '--optimizer', 'adam',
           '--learning_rate', '0.003', '--batch_size', '4', '--summary_rate_secs', '0', '--fov_policy', policy]
    res = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=REPO))
    assert res.returncode == 0, res.stderr[-3000:]
    assert 'eval/patch_loss' in res.stderr
    paths = glob.glob(str(train_dir / 'events.out.tfevents.*'))
    assert len(paths) == 1
    events = summary.read_events(paths[0])
    assert events[0].file_version == 'brain.Event:2'
    assert [e.step for e in events[1:]] == [50, 100]
    tags = {v.tag: v for v in events[-1].summary.value}
    want = ['eval/patch_loss', 'eval/patches', 'moves/total', 'fov/masked_voxel_fraction', 'fov/average_weight',
            'masked_voxel_fraction', 'pixel_loss', 'optimizer_loss', 'learning_rate']
    want += ['eval/all/%s' % m for m in ('accuracy', 'precision', 'recall', 'specificity', 'f1')]
    want += ['moves/all/%s' % t for t in tk.MOVE_TYPES]
    for r in (0, 4, 5, 6):
      want += ['moves/r=%d/%s' % (r, t) for t in ('correct', 'spurious', 'missed', 'total')]
    want += ['final_%s/0' % a for a in ('xy', 'xz', 'yz')]
    assert not set(want) - set(tags), set(want) - set(tags)
    assert tags['eval/patches'].simple_value > 0
    for t in ('eval/all/accuracy', 'eval/all/precision', 'eval/all/recall', 'eval/all/specificity', 'eval/all/f1',
              'moves/all/correct', 'moves/all/missed', 'moves/all/spurious', 'fov/masked_voxel_fraction',
              'masked_voxel_fraction'):
      assert 0.0 <= tags[t].simple_value <= 1.0, t
    assert tags['fov/average_weight'].simple_value == 1.0
    img = tags['final_xy/0'].image
    assert (img.height, img.width) == (25, 75) and img.encoded_image_string[:4] == b'\x89PNG'
