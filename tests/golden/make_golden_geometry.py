"""Fixture pinning the flood fill at fields of view other than (33, 33, 33) / (17, 33, 33), from the REAL
reference modules.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_geometry.py

Same harness as make_golden.py / make_golden_masks.py: the reference's unmodified Canvas.segment_all with
PolicyGrid3d, driven by the machine-independent toy network (oracle/toy_net.py).  One .npz holds every
geometry, keyed by a short name:

  g9   fov (z, y, x) = (9, 17, 25), deltas (2, 4, 6): a different size and delta on every axis
  g5   fov (5, 33, 33), deltas (0, 8, 8): no z moves, the y / x faces are one voxel thick in z
  g3   fov (3, 3, 3), deltas (1, 1, 1): the smallest field of view, one-voxel moves

Each phantom is small, and min_boundary_dist / min_segment_size are chosen so that both rejections occur.
Re-running the script gives identical arrays.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
import make_golden_masks as mgm  # noqa: E402

# name: fov_zyx, deltas_zyx, phantom shape, phantom seed, cell volume, min_segment_size, min_boundary_dist_zyx
GEOMETRIES = {
    'g9': ((9, 17, 25), (2, 4, 6), (40, 64, 72), 13, 12000.0, 5000, (1, 2, 1)),
    'g5': ((5, 33, 33), (0, 8, 8), (40, 64, 72), 17, 15000.0, 2000, (2, 1, 1)),
    'g3': ((3, 3, 3), (1, 1, 1), (18, 22, 26), 19, 1500.0, 200, (1, 1, 1)),
}


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

  class ToyClient:
    def start(self):
      return 0

    def finish(self):
      pass

    def predict(self, seed, image, fetches):
      return {'logits': toy_net(seed, image)[..., np.newaxis]}

  out = {}
  for name, (fov, deltas, shape, pseed, cell_volume, min_size, mbd) in GEOMETRIES.items():
    opts = ref_pb2.InferenceOptions()
    opts.init_activation, opts.pad_value, opts.move_threshold, opts.segment_threshold = 0.95, 0.05, 0.9, 0.6
    opts.min_segment_size = min_size
    opts.min_boundary_dist.z, opts.min_boundary_dist.y, opts.min_boundary_dist.x = mbd
    req = ref_pb2.InferenceRequest()
    req.inference_options.CopyFrom(opts)
    info = ref_model.ModelInfo(np.array(deltas[::-1]), np.array(fov[::-1]), np.array(fov[::-1]), np.array(fov[::-1]))
    _, cells = voronoi_phantom(shape, seed=pseed, cell_volume=cell_volume, return_cells=True)
    canvas = ref_inference.Canvas(info, ToyClient(), toy_image(cells), opts,
                                  movement_policy_fn=ref_movement.get_policy_fn(req, info), keep_probability_maps=True)
    trace = []
    upd = canvas.update_at
    canvas.update_at = lambda pos, upd=upd, trace=trace: (trace.append(tuple(int(p) for p in pos)), upd(pos))[1]
    canvas.segment_all(seed_policy=ref_seed.PolicyGrid3d)
    rec = mgm.record(canvas, trace)
    counters = {k: v for k, v in json.loads(rec['counters']).items() if not k.endswith('-ms')}   # no timings
    rec.update(counters=json.dumps(counters, sort_keys=True),cells=cells, fov=np.asarray(fov), deltas=np.asarray(deltas), min_segment_size=np.int64(min_size),
               min_boundary_dist=np.asarray(mbd))
    out.update({'%s_%s' % (name, k): v for k, v in rec.items()})
    print('%s: fov %r deltas %r: %d steps, %d segments, counters=%s' % (
        name, fov, deltas, len(rec['trace']), len(rec['origins']), rec['counters']))
  np.savez_compressed(os.path.join(HERE, 'toy_geometry_flood_fill.npz'), names=np.asarray(sorted(GEOMETRIES)), **out)


if __name__ == '__main__':
  main()
