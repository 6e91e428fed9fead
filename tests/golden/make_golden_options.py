"""Fixture pinning the flood fill away from the FIB-25 inference options, from the REAL reference modules.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_options.py

Same harness as make_golden_masks.py.  Injected stand-ins, nothing else:
  * make_golden.install_stubs(): inert modules for the third-party imports of the reference package
    (tensorflow, tf_slim, jax, h5py, tensorstore, edt, skimage, connectomics) — none of them is called
  * ToyClient: the executor client, whose predict() evaluates the machine-independent oracle/toy_net.py
  * ffn_b200.synthetic.voronoi_phantom: the cell volume the toy image is made from
The reference's Canvas, movement.get_policy_fn / FaceMaxMovementPolicy and seed.PolicyGrid3d run unmodified.

Output: toy_options_flood_fill.npz — for every case below one Canvas.segment_all(PolicyGrid3d) on the same
56^3 toy canvas, with keep_history=True, stored under '<case>__<key>':
  the record() contents of make_golden_masks.py (seed_canvas, segmentation, seg_prob unless
  keep_probability_maps is False, origins, overlaps, counters, trace);
  disco_applied   per FoV step: whether update_at's disco merge ran (inference.py:416-436), from the raw logits
                  the client returned: disco_seed_threshold >= 0 and mean(logits >= move) > disco_seed_threshold
  history_start / history / history_deleted   Canvas.history and history_deleted of the object with the most
                  FoV steps (the first such), as left by its segment_at call
The counters gain 'invalid-weak' / 'invalid-small': the number of 'Failed: weak seed' / 'Failed: too small'
rejections, which the reference only counts as time (inference.py:601-646).
'cases' is a JSON list of {name, options (probability space, InferenceOptions field names, min_boundary_dist
as z, y, x), movement_policy_args, keep_probability_maps}.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
from make_golden_masks import record  # noqa: E402

SHAPE = (56, 56, 56)
FIB25 = dict(init_activation=0.95, pad_value=0.05, move_threshold=0.9, segment_threshold=0.6,
             min_boundary_dist=(1, 1, 1), min_segment_size=1000)


def case_list(disco_partial):
  """(name, options over FIB25, movement_policy_args, keep_probability_maps)."""
  return [
      ('default', {}, '', True),
      # doc/manual.md, "Segmentation inference"
      ('manual', dict(pad_value=0.5, move_threshold=0.6, segment_threshold=0.6, min_boundary_dist=(1, 2, 2),
                      min_segment_size=1000), '', True),
      ('disco_off', dict(disco_seed_threshold=-1.0), '', True),
      ('disco_partial', dict(disco_seed_threshold=disco_partial), '', True),
      ('disco_never', dict(disco_seed_threshold=1.0), '', True),
      ('policy_low', {}, '{"score_threshold": -2.0}', True),
      ('policy_high', {}, '{"score_threshold": 2.8}', True),
      ('seg_low_pad_low', dict(segment_threshold=0.2, pad_value=0.001), '', True),
      # init_activation above move_threshold, or no object starts
      ('seg_high_move_high', dict(segment_threshold=0.97, move_threshold=0.97, init_activation=0.99), '', True),
      # The toy network drives a visited voxel towards logit 3.5 (its value at the FoV centre): an initial
      # activation just above a move threshold above that falls below it with the first step, while a pad
      # value above it still lets the FoV move.
      ('weak_seed', dict(init_activation=0.98, move_threshold=0.975, pad_value=0.995), '', True),
      ('small_and_tight', dict(min_boundary_dist=(0, 0, 0), min_segment_size=0), '', False),
  ]


def main():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  sys.path.insert(0, mg.REF)
  from ffn.inference import inference as ref_inference
  from ffn.inference import inference_pb2 as ref_pb2
  from ffn.inference import movement as ref_movement
  from ffn.inference import seed as ref_seed
  from ffn.training import model as ref_model
  from ffn_b200.synthetic import voronoi_phantom
  from oracle.toy_net import toy_net, toy_image

  _, cells = voronoi_phantom(SHAPE, seed=3, cell_volume=12000.0, return_cells=True)
  image = toy_image(cells)
  info = ref_model.ModelInfo(np.array([8, 8, 8]), np.array([33, 33, 33]), np.array([33, 33, 33]),
                             np.array([33, 33, 33]))

  def run(over, policy_args, keep_maps):
    o = dict(FIB25, **over)
    opts = ref_pb2.InferenceOptions()
    for k in ('init_activation', 'pad_value', 'move_threshold', 'segment_threshold', 'min_segment_size'):
      setattr(opts, k, o[k])
    if 'disco_seed_threshold' in o:
      opts.disco_seed_threshold = o['disco_seed_threshold']
    opts.min_boundary_dist.z, opts.min_boundary_dist.y, opts.min_boundary_dist.x = o['min_boundary_dist']
    req = ref_pb2.InferenceRequest()
    req.inference_options.CopyFrom(opts)
    req.movement_policy_args = policy_args

    fractions, applied = [], []

    class ToyClient:
      def start(self):
        return 0

      def finish(self):
        pass

      def predict(self, seed, image, fetches):
        logits = toy_net(seed, image)
        frac = np.mean(logits >= canvas.options.move_threshold)
        fractions.append(float(frac))
        applied.append(bool(canvas.options.disco_seed_threshold >= 0 and frac > canvas.options.disco_seed_threshold))
        return {'logits': logits[..., np.newaxis]}

    canvas = ref_inference.Canvas(info, ToyClient(), image, opts, movement_policy_fn=ref_movement.get_policy_fn(req, info),
                                  keep_probability_maps=keep_maps, keep_history=True)
    trace, objects, rejected = [], [], {'invalid-weak': 0, 'invalid-small': 0}
    upd = canvas.update_at
    canvas.update_at = lambda pos: (trace.append(tuple(int(p) for p in pos)), upd(pos))[1]
    seg_at = canvas.segment_at

    def segment_at(pos, **kw):
      n = seg_at(pos, **kw)
      objects.append((n, tuple(int(p) for p in pos), list(canvas.history), list(canvas.history_deleted)))
      return n
    canvas.segment_at = segment_at
    log_info = canvas.log_info

    def log(fmt, *args, **kw):
      if fmt.startswith('Failed: weak seed'):
        rejected['invalid-weak'] += 1
      elif fmt.startswith('Failed: too small'):
        rejected['invalid-small'] += 1
      return log_info(fmt, *args, **kw)
    canvas.log_info = log
    canvas.segment_all(seed_policy=ref_seed.PolicyGrid3d)

    out = record(canvas, trace)
    counters = {k: v for k, v in json.loads(out['counters']).items() if not k.endswith('-ms')}   # clock readings
    counters.update(rejected)
    out['counters'] = json.dumps(counters)
    if not keep_maps:
      del out['seg_prob']
    n, start, history, deleted = max(objects, key=lambda t: t[0])   # max() keeps the first of equal maxima
    out.update(disco_applied=np.asarray(applied, dtype=bool), history_start=np.asarray(start, dtype=np.int64),
               history=np.asarray(history, dtype=np.int64).reshape(-1, 3),
               history_deleted=np.asarray(deleted, dtype=np.int64))
    assert len(history) == n
    return out, fractions, o

  # disco_partial: a threshold between two neighbouring per-step fractions of the default run, near their median
  _, fractions, _ = run({}, '', True)
  f = np.unique(np.float32(fractions))
  mid = len(f) // 2
  disco_partial = float(np.float32((float(f[mid - 1]) + float(f[mid])) / 2))

  arrays, cases, summary = {}, [], {}
  for name, over, policy_args, keep_maps in case_list(disco_partial):
    out, _, o = run(over, policy_args, keep_maps)
    cases.append(dict(name=name, options=o, movement_policy_args=policy_args, keep_probability_maps=keep_maps))
    arrays.update({'%s__%s' % (name, k): v for k, v in out.items()})
    summary[name] = (out, json.loads(out['counters']))
    c = summary[name][1]
    print('%-18s %3d steps, %d segments, merge on %d steps, counters %s' % (
        name, len(out['trace']), len(out['origins']), int(out['disco_applied'].sum()),
        {k: c.get(k, 0) for k in ('skip_threshold', 'skip_invalid_pos', 'seed_got_too_weak', 'invalid-weak',
                                  'invalid-small', 'voxels-segmented')}))

  # every case reaches the path it is there for
  base, base_c = summary['default']
  assert base_c['inference-calls'] >= 30 and base['disco_applied'].all()
  assert len(summary['manual'][0]['origins']) >= 3
  for name in ('disco_off', 'disco_never'):
    assert not summary[name][0]['disco_applied'].any()
  assert summary['disco_off'][0]['history_deleted'].size == 0 < summary['disco_off'][0]['history'].shape[0]
  h = summary['disco_never'][0]
  assert h['history_deleted'].size == h['history'].shape[0] > 0
  applied = summary['disco_partial'][0]['disco_applied']
  assert applied.sum() >= 5 and (~applied).sum() >= 5
  assert summary['policy_low'][1].get('skip_threshold', 0) > base_c.get('skip_threshold', 0)
  assert summary['policy_high'][1]['inference-calls'] < base_c['inference-calls']
  assert summary['weak_seed'][1].get('seed_got_too_weak', 0) > 0 and summary['weak_seed'][1]['invalid-weak'] > 0

  np.savez_compressed(os.path.join(HERE, 'toy_options_flood_fill.npz'), cells=cells, seeds=arrays['default__seeds'],
                      cases=json.dumps(cases), **{k: v for k, v in arrays.items() if not k.endswith('__seeds')})
  print('disco_partial threshold %r (default run fractions %.4f .. %.4f)' % (disco_partial, f[0], f[-1]))


if __name__ == '__main__':
  main()
