"""Fixture pinning the flood fill under an exactly representable network, from the REAL reference modules.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_exact.py

Same harness as make_golden_geometry.py: the reference's unmodified Canvas.segment_all with PolicyGrid3d, driven by
oracle/exact_net.py's flood network evaluated in float64 (every implementation that satisfies the premise of
exact_net computes the same logits, so this run is what the device must reproduce in every compute mode).  The
options put the move, segment and policy thresholds at exactly 0 (init 2, pad -3), and the u8 canvas has an
integer mean and a power-of-two stddev, so logits land exactly on the thresholds and faces have equal maxima.
The client counts both, and the fixture records the counts.  Re-running the script gives identical arrays.

  x9   fov (z, y, x) = (9, 17, 25), deltas (2, 4, 6), depth 3
  x5   fov (5, 9, 9), deltas (1, 2, 2), depth 2
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
import make_golden_masks as mgm  # noqa: E402

# name: fov_zyx, deltas_zyx, depth, phantom shape, phantom seed, min_segment_size, min_boundary_dist_zyx
GEOMETRIES = {
    'x9': ((9, 17, 25), (2, 4, 6), 3, (24, 40, 48), 5, 50, (1, 1, 1)),
    'x5': ((5, 9, 9), (1, 2, 2), 2, (16, 24, 24), 6, 50, (1, 2, 1)),
}
CELL_VOLUME = 3000.0


def tie_counts(logits, deltas, thresholds=(0.0,)):
  """(faces whose maximum occurs more than once, voxels exactly on a threshold) of one step's logits."""
  c = [s // 2 for s in logits.shape]
  faces = 0
  for axis in range(3):
    d = int(deltas[axis])
    if d == 0:
      continue
    for off in (-d, d):
      sl = [slice(c[a] - deltas[a], c[a] + deltas[a] + 1) for a in range(3)]
      sl[axis] = c[axis] + off
      face = logits[tuple(sl)]
      faces += int((face == face.max()).sum() > 1)
  return faces, int(sum((logits == t).sum() for t in thresholds))


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
  from oracle import exact_net as xn

  out = {}
  for name, (fov, deltas, depth, shape, pseed, min_size, mbd) in GEOMETRIES.items():
    w, b = xn.flood_net(depth)
    ties = {'face_ties': 0, 'threshold_hits': 0}

    class Client:
      def start(self):
        return 0

      def finish(self):
        pass

      def predict(self, seed, image, fetches):
        lg = xn.logits(w, b, seed, image, 'fp32')
        f, t = tie_counts(lg, deltas)
        ties['face_ties'] += f
        ties['threshold_hits'] += t
        return {'logits': lg[..., np.newaxis]}

    opts = ref_pb2.InferenceOptions()
    for k, v in xn.FLOOD_OPTIONS.items():
      setattr(opts, k, v)
    opts.min_segment_size = min_size
    opts.min_boundary_dist.z, opts.min_boundary_dist.y, opts.min_boundary_dist.x = mbd
    req = ref_pb2.InferenceRequest()
    req.inference_options.CopyFrom(opts)
    info = ref_model.ModelInfo(np.array(deltas[::-1]), np.array(fov[::-1]), np.array(fov[::-1]), np.array(fov[::-1]))
    _, cells = voronoi_phantom(shape, seed=pseed, cell_volume=CELL_VOLUME, return_cells=True)
    vol = xn.flood_image(cells, pseed)
    canvas = ref_inference.Canvas(info, Client(), xn.flood_image_f32(vol), opts,
                                  movement_policy_fn=ref_movement.get_policy_fn(req, info), keep_probability_maps=True)
    trace = []
    upd = canvas.update_at
    canvas.update_at = lambda pos, upd=upd, trace=trace: (trace.append(tuple(int(p) for p in pos)), upd(pos))[1]
    canvas.segment_all(seed_policy=ref_seed.PolicyGrid3d)
    rec = mgm.record(canvas, trace)
    counters = {k: v for k, v in json.loads(rec['counters']).items() if not k.endswith('-ms')}   # no timings
    rec.update(counters=json.dumps(counters, sort_keys=True), volume=vol, fov=np.asarray(fov),
               deltas=np.asarray(deltas), depth=np.int64(depth), min_segment_size=np.int64(min_size),
               min_boundary_dist=np.asarray(mbd), ties=json.dumps(ties, sort_keys=True))
    out.update({'%s_%s' % (name, k): v for k, v in rec.items()})
    print('%s: fov %r deltas %r depth %d: %d steps, %d segments, ties %s, counters=%s' % (
        name, fov, deltas, depth, len(rec['trace']), len(rec['origins']), ties, rec['counters']))
  np.savez_compressed(os.path.join(HERE, 'exact_flood_fill.npz'), names=np.asarray(sorted(GEOMETRIES)), **out)


if __name__ == '__main__':
  main()
