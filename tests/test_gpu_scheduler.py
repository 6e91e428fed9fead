"""segment_all's device scheduler against the sequential loop, transition by transition and across launches.

With several chains the persistent kernel grows objects ahead of their turn, parks finished ones until their turn
comes, suspends a run so that a parked object can commit, and at an early run's turn validates it against its
trajectory log or throws it away (flood_kernel.cuh: advance_pointer, lookahead, swap_buffers, run_conflicts,
chain_advance).  The result must be that of the strictly sequential loop, for any number of chains and wherever a
launch pauses.  Each case below is a canvas and a seed order built to drive some of those transitions.  The device
runs it at 1 to 4 chains, with launch boundaries every 1, 3 or 64 FoV steps as well as at the default 2^15, and
every run must equal the hybrid oracle (oracle/flood_fill.py's loop on the CPU, driven by the device's own network)
and the one-chain, default-chunk device run.  Every case also asserts, from DeviceCanvas.sched_stats(), that it
reached the transitions it was built for: a heuristic change that stops covering a path fails here as a coverage
failure instead of passing silently.
"""

import os
import time

import numpy as np
import pytest
from scipy import ndimage

from oracle import flood_fill as ff

pytestmark = pytest.mark.gpu

FOV, DELTAS = (33, 33, 33), (8, 8, 8)
HALF = FOV[0] // 2
CHAINS = (1, 2, 3, 4)
CHUNKS = (0, 1, 3, 64)    # FoV steps per launch; 0 = the default 2^15, more than any case here runs


def _image(vol):
  return (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)


def _phantom(shape, seed, **kw):
  from ffn_b200.synthetic import voronoi_phantom
  return voronoi_phantom(shape, seed=seed, return_cells=True, **kw)


def _inside(shape, p):
  """The border filter of seed.py:81-88: the FoV around p lies in the canvas."""
  return all(HALF <= v < s - HALF for v, s in zip(p, shape))


def _cells(cells):
  """[(id, size, centroid, (lo, hi))] of the ground-truth cells, largest first."""
  n = int(cells.max())
  sizes = np.bincount(cells.ravel(), minlength=n + 1)
  boxes = ndimage.find_objects(cells)
  ids = [i for i in range(1, n + 1) if sizes[i] > 0 and boxes[i - 1] is not None]
  cent = ndimage.center_of_mass(np.ones(cells.shape, np.uint8), cells, ids)
  out = [(i, int(sizes[i]), tuple(int(round(v)) for v in c), (tuple(s.start for s in boxes[i - 1]),
                                                               tuple(s.stop for s in boxes[i - 1])))
         for i, c in zip(ids, cent)]
  return sorted(out, key=lambda t: (-t[1], t[0]))


def _seed_in(vol, cells, cid, near):
  """interior_seed snapped near `near`, if it falls in cell cid and passes the border filter; else None."""
  from ffn_b200.synthetic import interior_seed
  p = interior_seed(vol, near, max_radius=8)
  return p if cells[p] == cid and _inside(vol.shape, p) else None


# ---- the cases -----------------------------------------------------------------------------------------------
def _two_scale(seed, big_cv, small_cv):
  """A region of large cells (x < 64) next to a region of small ones: long objects and short ones."""
  big, bc = _phantom((80, 80, 64), seed, cell_volume=big_cv)
  small, sc = _phantom((80, 80, 128), seed + 1, cell_volume=small_cv)
  vol = np.concatenate([big, small], axis=2)
  cells = np.concatenate([bc, np.where(sc > 0, sc + bc.max(), 0)], axis=2)
  return vol, cells


def _far_small(vol, cells, rng, x_min):
  seeds = []
  for cid, _, c, _ in _cells(cells):
    if c[2] >= x_min:
      p = _seed_in(vol, cells, cid, c)
      if p is not None:
        seeds.append(p)
  return [seeds[i] for i in rng.permutation(len(seeds))]


def _park(seed, small_cv, n_small):
  """Seed 0 in a large cell, then n_small seeds in small cells more than half a FoV away from it: early runs finish
  long before seed 0's object does, so they park, fill every buffer of their chain, and commit by turn swaps."""
  vol, cells = _two_scale(seed, 150000.0, small_cv)
  big = [t for t in _cells(cells) if t[2][2] < 64]
  first = next(p for p in (_seed_in(vol, cells, t[0], t[2]) for t in big) if p is not None)
  small = _far_small(vol, cells, np.random.RandomState(seed), 64 + HALF + 8)
  return vol, [first] + small[:n_small], {}, None


def _suspend(seed, small_cv, per_long):
  """Long objects with per_long short ones between them: a chain is growing a short object when the parked one
  before it comes up, so the run is suspended and resumed after the commit."""
  vol, cells = _two_scale(seed, 20000.0, small_cv)
  big = [p for p in (_seed_in(vol, cells, t[0], t[2]) for t in _cells(cells) if t[2][2] < 56) if p is not None]
  small = _far_small(vol, cells, np.random.RandomState(seed), 64 + HALF + 8)
  seeds = []
  for i, p in enumerate(big):
    seeds += [p] + small[i * per_long:(i + 1) * per_long]
  return vol, seeds, {}, None


def _elongated(seed, cell_volume):
  return _phantom((64, 80, 176), seed, voxel_size_zyx=(1.0, 1.0, 0.3), cell_volume=cell_volume)


def _end_pairs(vol, cells):
  """Seeds at the two ends (in x) of every long cell, in pairs."""
  seeds = []
  for cid, _, c, (lo, hi) in _cells(cells):
    if hi[2] - lo[2] < 40:
      continue
    a = _seed_in(vol, cells, cid, (c[0], c[1], lo[2] + 10))
    b = _seed_in(vol, cells, cid, (c[0], c[1], hi[2] - 11))
    if a is not None and b is not None:
      seeds += [a, b]
  return seeds


def _discard(seed, cell_volume, mbd):
  """Seed pairs at the two ends of elongated cells: the second end starts early, far from the first end's object,
  and at its turn that object has labelled its seed (rejected) or its path (redone), or left it alone (validated).
  A min_boundary_dist box wider than the default rejects seeds next to objects labelled after they started.
  A chain that suspended a run to take up its parked object, and then saw that object rejected at its turn, is free
  in the same round as the suspension: the suspended run must wait a round (resume_deferred), because the paste of
  its last step is still landing and a commit right away would count a seed array that other CTAs are writing."""
  vol, cells = _elongated(seed, cell_volume)
  return vol, _end_pairs(vol, cells), dict(min_boundary_dist=tuple(mbd)), None


def _snapshot(seed, cell_volume, n_seeds):
  """Elongated-cell pairs cut after n_seeds: the chain that committed the last object starts an early run that
  is discarded, so Canvas.seed's last in-turn object has to come back from the snapshot array."""
  vol, cells = _elongated(seed, cell_volume)
  return vol, _end_pairs(vol, cells)[:n_seeds], {}, None


def _unstepped(seed, cell_volume, band):
  """A movement-restricted band y in [band, band + 10) wider than a step, and cells that cross it, each seeded on
  both sides: first at y = band - 4, then at y = band + 17, at the same z and x.  The second starts early; its first
  step towards the band pops y = band + 9, inside the band, which it may not step on (logged as unstepped).  The
  first object never steps into the band either, but its FoV reaches y = band + 12: it labels that position and none
  of the second object's FoV centres (all at y >= band + 17, outside its min_boundary_dist box too).  At the second
  seed's turn only the unstepped entry conflicts: the reference would have counted the position as invalid instead
  of restricted."""
  vol, cells = _phantom((80, 96, 160), seed, cell_volume=cell_volume)
  mask = np.zeros(vol.shape, bool)
  mask[:, band:band + 10, :] = True
  bright = ndimage.minimum_filter(vol, size=3, mode='nearest') >= 140
  seeds = []
  for cid, _, c, _ in _cells(cells):
    both = (cells[:, band - 4, :] == cid) & bright[:, band - 4, :] & (cells[:, band + 17, :] == cid) & bright[:, band + 17, :]
    zz, xx = np.nonzero(both)
    keep = [(z, x) for z, x in zip(zz, xx) if _inside(vol.shape, (z, band, x))]
    if keep:
      z, x = min(keep, key=lambda t: ((t[0] - c[0]) ** 2 + (t[1] - c[2]) ** 2, t))
      seeds += [(int(z), band - 4, int(x)), (int(z), band + 17, int(x))]
  return vol, seeds, {}, mask


def _window(seed, cell_volume, n_block):
  """Seed 0, then n_block (> 256, the look-ahead window) seeds inside seed 0's cell, which the look-ahead refuses
  while seed 0's object grows, then a grid of seeds elsewhere that run early once the head of the line is past."""
  vol, cells = _phantom((48, 80, 80), seed, cell_volume=cell_volume)
  cid, first = next((t[0], p) for t in _cells(cells) for p in [_seed_in(vol, cells, t[0], t[2])] if p is not None)
  zz, yy, xx = np.nonzero(cells == cid)
  d2 = (zz - first[0]) ** 2 + (yy - first[1]) ** 2 + (xx - first[2]) ** 2
  order = np.lexsort((xx, yy, zz, d2))
  block = [(int(zz[k]), int(yy[k]), int(xx[k])) for k in order[1:n_block + 1]]
  rest = [tuple(int(v) for v in p) for p in ff.grid_seeds(vol.shape, step=12, offsets=(0, 6))]
  rest = [p for p in rest if cells[p] != cid]
  return vol, [first] + block + rest, {}, None


BUILDERS = {'park': _park, 'suspend': _suspend, 'discard': _discard, 'unstepped': _unstepped, 'window': _window,
            'snapshot': _snapshot}

# name -> (builder parameters, {transition: chain counts at which the default-chunk run must reach it})
CASES = {
    'park': (dict(seed=3, small_cv=4000.0, n_small=40),
             {'parked': (2, 4), 'turn_taken': (2, 4), 'idle_buffers_full': (2, 4)}),
    'suspend': (dict(seed=5, small_cv=4000.0, per_long=4), {'suspended': (2,), 'resumed': (2,)}),
    'discard': (dict(seed=1, cell_volume=6000.0, mbd=(2, 3, 3)),
                {'discard_redone': (2, 4), 'discard_rejected': (2, 4), 'early_validated': (2, 4),
                 'resume_deferred': (2,)}),
    'unstepped': (dict(seed=2, cell_volume=30000.0, band=44), {'conflict_unstepped_only': (2, 3, 4)}),
    'window': (dict(seed=4, cell_volume=20000.0, n_block=300), {'early_runs': (2, 4)}),
    'snapshot': (dict(seed=1, cell_volume=6000.0, n_seeds=12), {'snapshot_moves': (2,), 'resume_deferred': (2,)}),
}


def build_case(name, params=None):
  """(volume, seeds, probability-space option overrides, movement mask or None)."""
  return BUILDERS[name](**(CASES[name][0] if params is None else params))


# ---- the runs ------------------------------------------------------------------------------------------------
def _device_options(opts):
  from ffn_b200 import engine as eng
  return eng.make_options(init_activation=opts.init_activation, pad_value=opts.pad_value,
                          move_threshold=opts.move_threshold, segment_threshold=opts.segment_threshold,
                          disco_seed_threshold=opts.disco_seed_threshold, min_boundary_dist_zyx=opts.min_boundary_dist,
                          min_segment_size=opts.min_segment_size, policy_score_threshold=opts.policy_score_threshold)


def hybrid(e, case):
  vol, seeds, over, mask = case
  hyb = ff.Canvas(lambda s, im: e.predict(s, im), _image(vol), FOV, DELTAS, ff.Options(**over), mask=mask)
  hyb.segment_all(seeds)
  return hyb


def device(e, case, chains, chunk):
  """One segment_all on a fresh canvas; its results, and its spec_stats() and sched_stats() merged."""
  from ffn_b200 import _lib, engine as eng
  vol, seeds, over, mask = case
  e.set_chains(chains)
  e.set_step_chunk(chunk)
  try:
    cv = eng.DeviceCanvas(e, vol, _device_options(ff.Options(**over)), 128.0, 33.0)
    try:
      if mask is not None:
        cv.set_mask(_lib.MASK_MOVEMENT, mask)
      origins, overlaps, ctr = cv.segment_all(seeds)
      out = dict(seg=cv.read(_lib.ARRAY_SEGMENTATION), seed=cv.read(_lib.ARRAY_SEED), qprob=cv.read(_lib.ARRAY_QPROB),
                 origins=[(o.id, tuple(o.start_zyx), o.iters) for o in origins],
                 overlaps=sorted((o.id, o.other_id, o.count) for o in overlaps),
                 ctr={n: getattr(ctr, n) for n, _ in ctr._fields_ if n not in ('device_seconds', 'kernel_launches')})
      stats = dict(cv.spec_stats(), **cv.sched_stats())
    finally:
      cv.close()
  finally:
    e.set_chains(0)
    e.set_step_chunk(0)
  return out, stats


def check_vs_hybrid(dev, hyb, where):
  np.testing.assert_array_equal(dev['seg'], hyb.segmentation, err_msg='%s: labels' % where)
  np.testing.assert_array_equal(dev['seed'], hyb.seed, err_msg='%s: Canvas.seed' % where)
  qd = np.abs(dev['qprob'].astype(int) - hyb.seg_prob.astype(int))
  assert qd.max() <= 1 and (qd > 0).mean() < 1e-3, (where, 'qprob', int(qd.max()), float((qd > 0).mean()))
  assert dev['origins'] == [(k, v[0], v[1]) for k, v in sorted(hyb.origins.items())], (where, 'origins')
  assert dev['overlaps'] == sorted((k, int(i), int(c)) for k, v in hyb.overlaps.items() for i, c in zip(*v.tolist())), \
      (where, 'overlaps')
  ctr = dev['ctr']
  assert ctr['inference_calls'] == len(hyb.trace), (where, 'inference_calls')
  for mine, theirs in (('skip_threshold', 'skip_threshold'), ('skip_invalid_pos', 'skip_invalid_pos'),
                       ('skip_restricted_pos', 'skip_restriced_pos'), ('seed_got_too_weak', 'seed_got_too_weak'),
                       ('invalid_weak', 'invalid-weak'), ('invalid_small', 'invalid-small'),
                       ('voxels_segmented', 'voxels-segmented'), ('voxels_overlapping', 'voxels-overlapping')):
    assert ctr[mine] == hyb.counters[theirs], (where, mine, ctr[mine], hyb.counters[theirs])


def check_same(dev, ref, where):
  for k in ('seg', 'seed', 'qprob'):
    np.testing.assert_array_equal(dev[k], ref[k], err_msg='%s: %s differs from 1 chain, default chunk' % (where, k))
  for k in ('origins', 'overlaps', 'ctr'):
    assert dev[k] == ref[k], '%s: %s differs from 1 chain, default chunk' % (where, k)


def check_bookkeeping(st, dev, chains, chunk, where):
  assert st['owner_lost'] == 0, (where, st)
  assert st['chains'] == chains, (where, st)
  # every early run is settled at its turn: validated, or discarded and its seed rejected or redone
  assert st['discard_rejected'] + st['discard_redone'] == st['early_runs_discarded'], (where, st)
  assert st['early_validated'] + st['early_runs_discarded'] == st['early_runs'], (where, st)
  assert st['steps_executed'] == dev['ctr']['inference_calls'] + st['steps_discarded'], (where, st)
  if chunk in (1, 3):
    # a launch pauses at the first round boundary with steps_executed >= its budget; the K chains of that round
    # may all have stepped, so one launch runs at most chunk + K - 1 steps
    assert st['kernel_launches'] * (chunk + chains - 1) >= st['steps_executed'], (where, st)
    if chains == 4:   # launches that paused with objects in flight: parked or suspended, or committing
      assert st['launches_paused_parked'] + st['launches_paused_committing'] > 0, (where, st)
  if chunk == 0:
    assert st['kernel_launches'] == 1, (where, st)


def check_reached(name, stats):
  for transition, ks in CASES[name][1].items():
    for k in ks:
      assert stats[(k, 0)][transition] > 0, 'case %r did not reach %r with %d chains: %r' % (
          name, transition, k, stats[(k, 0)])


SHOWN = ('early_runs', 'early_validated', 'discard_rejected', 'discard_redone', 'parked', 'suspended', 'resumed',
         'resume_deferred', 'turn_taken', 'idle_buffers_full', 'conflict_unstepped_only', 'validated_unstepped',
         'discarded_unstepped', 'snapshot_moves', 'kernel_launches', 'launches_paused_parked', 'launches_paused_committing')


@pytest.fixture(scope='module')
def engine(golden_dir):
  from ffn_b200 import _lib, engine as eng, tf_checkpoint
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))
  e = eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP16_TC)   # the only mode that runs chains
  yield e
  e.close()


@pytest.mark.parametrize('name', list(CASES))
def test_scheduler_vs_hybrid_oracle(engine, name):
  """Every chain count and step chunk: equal to the hybrid oracle and to the one-chain run, bookkeeping
  consistent, the case's transitions reached."""
  case = build_case(name)
  t0 = time.perf_counter()
  hyb = hybrid(engine, case)
  print('%s: %d seeds, %d objects, hybrid oracle %d steps in %.1f s' % (
      name, len(case[1]), len(hyb.origins), len(hyb.trace), time.perf_counter() - t0))
  assert len(hyb.origins) >= 3
  ref, stats = None, {}
  for chains in CHAINS:
    for chunk in CHUNKS:
      where = '%s, %d chains, step chunk %s' % (name, chains, chunk or 'default')
      t0 = time.perf_counter()
      dev, st = device(engine, case, chains, chunk)
      secs = time.perf_counter() - t0
      print('  %d chains, chunk %5s: %.2f s, %d steps executed, %s' % (
          chains, chunk or 'dflt', secs, st['steps_executed'], ' '.join('%s=%d' % (k, st[k]) for k in SHOWN)))
      check_vs_hybrid(dev, hyb, where)
      if ref is None:
        ref = dev
      else:
        check_same(dev, ref, where)
      check_bookkeeping(st, dev, chains, chunk, where)
      stats[(chains, chunk)] = st
  check_reached(name, stats)


def test_segment_at_across_launch_boundaries(engine):
  """Canvas.segment_at on one long object with a launch boundary every 1 or 3 FoV steps: the same object, step for
  step, as at the default chunk and as the hybrid oracle, with the launches the chunk implies."""
  from ffn_b200 import _lib, engine as eng
  vol, cells = _phantom((64, 64, 64), 3, cell_volume=150000.0)
  start = next(p for p in (_seed_in(vol, cells, t[0], t[2]) for t in _cells(cells)) if p is not None)
  hyb = ff.Canvas(lambda s, im: engine.predict(s, im), _image(vol), FOV, DELTAS, ff.Options())
  iters = hyb.segment_at(start)
  assert iters >= 20, iters
  for chunk in CHUNKS:
    engine.set_step_chunk(chunk)
    try:
      cv = eng.DeviceCanvas(engine, vol, eng.make_options(), 128.0, 33.0)
      try:
        before = engine.info()['launches']
        st = cv.segment_at(start)
        launches = engine.info()['launches'] - before
        seed = cv.read(_lib.ARRAY_SEED)
      finally:
        cv.close()
    finally:
      engine.set_step_chunk(0)
    where = 'segment_at, step chunk %s' % (chunk or 'default')
    assert st.finished and st.iters == iters, (where, st.iters, iters)
    assert tuple(st.min_pos) == tuple(hyb.min_pos) and tuple(st.max_pos) == tuple(hyb.max_pos), where
    np.testing.assert_array_equal(seed, hyb.seed, err_msg=where)
    # the budget is checked after every step of the one chain: ceil(iters / chunk) paused launches and a last one
    assert launches >= (iters + chunk - 1) // chunk if chunk else launches == 1, (where, launches, iters)
