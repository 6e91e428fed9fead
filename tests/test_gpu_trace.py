"""The movement-queue pop events of the device event trace against the hybrid oracle.

With the trace on, the device logs one event per candidate it takes off the queue, in queue order:
EV_POP_DONE (its lattice cell is done), EV_POP_THRESHOLD (seed below the move threshold), EV_POP_INVALID (at the
border or already labelled) or EV_POP_VALID (returned by the pop: stepped on, skipped by the movement restrictor,
or the one in hand when the object ends as 'seed_got_too_weak').  The oracle loop (`ff.Canvas`, driven by the
same GPU network) logs the same classes from its `FaceMaxPolicy.pop`.  Turning the trace on must not change
any result.
"""

import os

import numpy as np
import pytest

from oracle import flood_fill as ff

pytestmark = pytest.mark.gpu

FOV, DELTAS = (33, 33, 33), (8, 8, 8)
EV_POP_VALID, EV_POP_INVALID, EV_POP_THRESHOLD, EV_POP_DONE = 2, 3, 4, 5


class _PopLogPolicy(ff.FaceMaxPolicy):
  """FaceMaxPolicy.pop that records the class of every candidate it takes off the queue."""

  def __init__(self, canvas, deltas, score_threshold):
    super().__init__(canvas, deltas, score_threshold)
    self.log = []

  def pop(self):
    counters = self.canvas.counters
    while self.queue:
      _, coord = self.queue.popleft()
      coord = tuple(int(v) for v in coord)
      if self.quantize(coord) in self.done:
        self.log.append((EV_POP_DONE,) + coord)
        continue
      below = counters['skip_threshold']
      if self.canvas.is_valid_pos(coord):
        self.log.append((EV_POP_VALID,) + coord)
        return coord
      self.log.append((EV_POP_THRESHOLD if counters['skip_threshold'] > below else EV_POP_INVALID,) + coord)
    return None


@pytest.fixture(scope='module')
def engine(golden_dir):
  from ffn_b200 import _lib, engine as eng, tf_checkpoint
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))
  e = eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP32)
  yield e
  e.close()


def _segment_all(e, vol, seeds, mask, trace_cap):
  from ffn_b200 import _lib, engine as eng
  cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
  if mask is not None:
    cv.set_mask(_lib.MASK_MOVEMENT, mask)
  if trace_cap:
    cv.start_trace(trace_cap)
  origins, overlaps, ctr = cv.segment_all(seeds)
  out = dict(seg=cv.read(_lib.ARRAY_SEGMENTATION), seed=cv.read(_lib.ARRAY_SEED), qprob=cv.read(_lib.ARRAY_QPROB),
             origins=[(o.id, tuple(o.start_zyx), o.iters) for o in origins],
             overlaps=sorted((o.id, o.other_id, o.count) for o in overlaps),
             ctr={n: getattr(ctr, n) for n, _ in ctr._fields_ if n not in ('device_seconds', 'kernel_launches')})
  if trace_cap:
    out['trace'], out['n_events'] = cv.get_trace(with_total=True)
  cv.close()
  return out


@pytest.mark.parametrize('restrict', [False, True])
def test_pop_events_match_hybrid_oracle(engine, golden_dir, restrict):
  g = np.load(os.path.join(golden_dir, 'flood_fill_64.npz'))
  vol, seeds = g['volume'], g['seeds']
  mask = None
  if restrict:
    mask = np.zeros(vol.shape, bool)
    mask[:, 32:40, :] = True
  cap = 1 << 16
  traced = _segment_all(engine, vol, seeds, mask, cap)
  assert traced['n_events'] <= cap, 'trace overflowed'
  ev = traced['trace']
  pops = ev[(ev[:, 0] >= EV_POP_VALID) & (ev[:, 0] <= EV_POP_DONE)]

  image = (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)
  hyb = ff.Canvas(lambda s, im: engine.predict(s, im), image, FOV, DELTAS, ff.Options(), mask=mask)
  hyb.policy = _PopLogPolicy(hyb, DELTAS, hyb.policy.score_threshold)
  hyb.segment_all(seeds)
  want = np.asarray(hyb.policy.log, dtype=np.int32).reshape(-1, 4)
  np.testing.assert_array_equal(pops, want)
  assert set(pops[:, 0].tolist()) == {EV_POP_VALID, EV_POP_INVALID, EV_POP_THRESHOLD, EV_POP_DONE}
  if restrict:
    assert traced['ctr']['skip_restricted_pos'] == hyb.counters['skip_restriced_pos'] > 0

  plain = _segment_all(engine, vol, seeds, mask, 0)
  for key in ('seg', 'seed', 'qprob'):
    np.testing.assert_array_equal(traced[key], plain[key])
  assert traced['origins'] == plain['origins']
  assert traced['overlaps'] == plain['overlaps']
  assert traced['ctr'] == plain['ctr']
