"""Flood-fill quality while training: the reference's EvalTracker (ffn/training/tracker.py) as the device keeps it.

The example loop counts on the device (ffn_examples_tracker of include/ffn_b200.h) what examples.py records in the
reference's tracker: every field-of-view move the policy evaluates (correct, missed or spurious, by move radius) and,
for every finished example, the prediction counts and the loss of its final object mask over the eval crop, with the
centre planes of the last 16 of them.  `summaries` turns one reading into the values `EvalTracker.get_summaries()`
returns, with the same tags and formulas.

Defined here where the reference is not: the patch loss is computed in float64 (max(x, 0) - x z + log1p(exp(-|x|))
summed over the crop in a fixed order, divided by its voxel count) where the reference takes a float32 TF
reduce_mean; the loop's loss weights are all ones, so the weight statistics follow from the step and voxel counts.
"""

from __future__ import annotations

import dataclasses
import io

import numpy as np
from scipy import special

EVAL_THRESHOLD = special.logit(0.9)   # EvalTracker.eval_threshold, np.float64
MOVE_TYPES = ('correct', 'missed', 'spurious')   # tracker.MoveType order
RING = 16                             # EvalTracker's deque(maxlen=16) of images


def eval_shape(fov_zyx, deltas_zyx, fov_moves: int) -> tuple[int, int, int]:
  """train.py's train_eval_size, zyx: fov + 2 * deltas * fov_moves (the flag's value for both policies)."""
  return tuple(int(f) + 2 * int(d) * int(fov_moves) for f, d in zip(fov_zyx, deltas_zyx))


def move_radius(offset) -> int:
  """EvalTracker.record_move's radius: int(np.linalg.norm(offset)), truncated."""
  return int(np.linalg.norm(np.asarray(offset, np.float64)))


def radii(shifts) -> list[int]:
  """The radii EvalTracker keeps counters for: 0 and int(|s|) of every shift, sorted."""
  return sorted({0} | {move_radius(s) for s in shifts})


@dataclasses.dataclass
class TrackerState:
  """One reading of the tracker: counts since the last reset and the last (up to 16) finished examples' planes."""
  steps: int
  fov_voxels: int                     # steps * batch * fov voxels: the loss-weight voxels of the batches
  patches: int
  eval_voxels: int
  prediction_counts: np.ndarray       # int64 [4]: TP, TN, FP, FN
  patch_loss: float                   # sum of the finished patches' mean losses
  moves: dict                         # {radius: int64 [3]} (correct, missed, spurious)
  planes: list                        # per finished example: (xy, xz, yz), each (labels, logits) float32 [h, w]
  coords: list                        # per finished example: (volume index, (x, y, z))


def split_planes(flat: np.ndarray, shape_zyx) -> tuple:
  """A ring entry [xy labels, xy logits, xz labels, xz logits, yz labels, yz logits] as ((lab, lg) xy, xz, yz)."""
  e0, e1, e2 = shape_zyx
  out, pos = [], 0
  for h, w in ((e1, e2), (e0, e2), (e0, e1)):
    n = h * w
    out.append((flat[pos:pos + n].reshape(h, w), flat[pos + n:pos + 2 * n].reshape(h, w)))
    pos += 2 * n
  return tuple(out)


def slice_image(labels: np.ndarray, logits: np.ndarray, coord_xyz, volume_name: str) -> bytes:
  """EvalTracker.slice_image of one plane: labels, expit(logits) and the unit weights side by side, each
  (v * 255).astype(np.uint8), as RGB, with "x,y,z\\nvolume" at (1, 1) in PIL's default font.  PNG bytes."""
  import PIL.Image  # pylint: disable=g-import-not-at-top
  import PIL.ImageDraw  # pylint: disable=g-import-not-at-top
  import PIL.ImageFont  # pylint: disable=g-import-not-at-top
  labels = np.asarray(labels, np.float32)
  predicted = special.expit(np.asarray(logits, np.float32))
  weights = np.ones_like(labels)
  cols = [(v * 255).astype(np.uint8) for v in (labels, predicted, weights)]
  im = PIL.Image.fromarray(np.repeat(np.concatenate(cols, axis=1)[..., np.newaxis], 3, axis=2), 'RGB')
  draw = PIL.ImageDraw.Draw(im)
  x, y, z = (int(v) for v in coord_xyz)
  draw.text((1, 1), '%d,%d,%d\n%s' % (x, y, z, volume_name), fill='rgb(255,64,64)', font=PIL.ImageFont.load_default())
  del draw
  buf = io.BytesIO()
  im.save(buf, 'PNG')
  return buf.getvalue()


@dataclasses.dataclass
class Image:
  """A Summary.Image: RGB PNG of height x width."""
  height: int
  width: int
  png: bytes


def _metrics(pc, prefix):
  """EvalTracker._compute_classification_metrics."""
  tp, tn, fp, fn = (int(v) for v in pc)
  precision = tp / max(tp + fp, 1)
  recall = tp / max(tp + fn, 1)
  f1 = 2.0 * precision * recall / (precision + recall) if precision > 0 or recall > 0 else 0.0
  return [('%s/accuracy' % prefix, (tp + tn) / max(tp + tn + fp + fn, 1)), ('%s/precision' % prefix, precision),
          ('%s/recall' % prefix, recall), ('%s/specificity' % prefix, tn / max(tn + fp, 1)), ('%s/f1' % prefix, f1)]


def summaries(state: TrackerState, volume_names, images: bool = True) -> list:
  """EvalTracker.get_summaries() of one reading: [(tag, float or Image)] in the reference's order; [] when no
  example has finished.  volume_names: the name of each volume index, written on the images."""
  if not state.eval_voxels:
    return []
  moves_all = sum(np.asarray(v, np.int64) for v in state.moves.values())
  total_moves = max(int(moves_all.sum()), 1)
  out = [('fov/masked_voxel_fraction', 0 / max(state.fov_voxels, 1)),
         ('fov/average_weight', state.fov_voxels / max(state.fov_voxels, 1)),
         ('masked_voxel_fraction', 0 / state.eval_voxels),
         ('eval/patch_loss', state.patch_loss / state.patches),
         ('eval/patches', state.patches),
         ('moves/total', total_moves)]
  out += [('moves/all/%s' % t, int(moves_all[k]) / total_moves) for k, t in enumerate(MOVE_TYPES)]
  if images:
    for axis, name in enumerate(('xy', 'xz', 'yz')):
      for i, (planes, (vol, xyz)) in enumerate(zip(state.planes, state.coords)):
        lab, lg = planes[axis]
        out.append(('final_%s/%d' % (name, i), Image(lab.shape[0], 3 * lab.shape[1],
                                                     slice_image(lab, lg, xyz, volume_names[vol]))))
  out += _metrics(state.prediction_counts, 'eval/all')
  for r in sorted(state.moves):
    m = np.asarray(state.moves[r], np.int64)
    t = max(int(m.sum()), 1)
    out += [('moves/r=%d/correct' % r, int(m[0]) / t), ('moves/r=%d/spurious' % r, int(m[2]) / t),
            ('moves/r=%d/missed' % r, int(m[1]) / t), ('moves/r=%d/total' % r, t)]
  return out
