r"""Computes the partition map of a segmentation on the device.

Drop-in for the reference entry point (compute_partitions.py), with its flags:

  python compute_partitions.py \
      --input_volume groundtruth.h5:stack \
      --output_volume af.h5:af \
      --thresholds 0.025,0.05,0.075,0.1,0.2,0.3,0.4,0.5,0.6,0.7,0.8,0.9 \
      --lom_radius 16,16,16 \
      --min_size 10000

For every labelled voxel, the fraction of identically labelled voxels within the (2r+1)^3 local object mask,
quantized by `thresholds`.  Unlike the reference's script, `--mask_configs` is parsed as a text-format MaskConfigs,
`--id_whitelist` as integers and `--exclusion_regions` as groups of four numbers (x, y, z, r).

`<path>:<dataset>` is read and written with h5py when it is installed.  Without h5py, or for a `.npz` path, the input
is a `.npy` (`file.npy:`) or `.npz` (`file.npz:key`) volume whose `bounding_boxes` attrs, when any, are the arrays
stored under keys starting with `<key>.bounding_boxes`; the output is a `.npz` with the partition volume under
`<dataset>` and its attrs under `<dataset>.bounding_boxes` and `<dataset>.partition_counts`.
"""

import numpy as np
from absl import app
from absl import flags
from google.protobuf import text_format

from ffn_b200 import partitions
from ffn_b200.inference import inference_pb2
from ffn_b200.inference import storage
from ffn_b200.utils import bounding_box

FLAGS = flags.FLAGS

flags.DEFINE_string('input_volume', None, 'Segmentation volume as <volume_path>:<dataset>.')
flags.DEFINE_string('output_volume', None, 'Volume in which to save the partition map, as <volume_path>:<dataset>.')
flags.DEFINE_list('thresholds', None, 'List of activation voxel fractions used for partitioning.')
flags.DEFINE_list('lom_radius', None, 'Local Object Mask (LOM) radii as (x, y, z).')
flags.DEFINE_list('id_whitelist', None, 'Whitelist of object IDs for which to compute the partition numbers.')
flags.DEFINE_list('exclusion_regions', None,
                  'List of x, y, z, r values, four per spherical region to mark as excluded (255).')
flags.DEFINE_string('mask_configs', None,
                    'MaskConfigs proto in text format. Any locations where at least one voxel of the LOM is masked '
                    'will be marked as excluded.')
flags.DEFINE_integer('min_size', 10000, 'Minimum number of voxels for a segment to be considered for partitioning.')
flags.DEFINE_integer('device', 0, 'CUDA device ordinal.')


def _h5py():
  try:
    import h5py  # pylint: disable=g-import-not-at-top
  except ImportError:
    return None
  return h5py


def _number(text):
  v = float(text)
  try:
    return int(text)
  except ValueError:
    return v


def parse_exclusion_regions(values):
  if values is None:
    return None
  if len(values) % 4:
    raise ValueError('--exclusion_regions takes groups of four values (x, y, z, r), got %d' % len(values))
  nums = [_number(v) for v in values]
  return [tuple(nums[i:i + 4]) for i in range(0, len(nums), 4)]


def parse_mask_configs(text):
  if text is None:
    return None
  configs = inference_pb2.MaskConfigs()
  text_format.Parse(text, configs)
  return configs


def read_input(spec):
  """(labels, [BoundingBox]) of `<path>:<dataset>`; one box over the whole volume when it has none."""
  path, dataset = spec.split(':')
  h5py = _h5py()
  boxes = []
  if h5py is not None and not path.endswith(('.npy', '.npz')):
    with h5py.File(path, 'r') as f:
      ds = f[dataset]
      for name, v in ds.attrs.items():
        if name.startswith('bounding_boxes'):
          boxes.extend(v)
      seg = ds[...]
  else:
    settings = inference_pb2.DecoratedVolume(hdf5=spec)
    seg = np.asarray(storage.decorated_volume(settings)[...])
    if path.endswith('.npz'):
      with np.load(path) as f:
        for name in sorted(f.files):
          if name.startswith(dataset + '.bounding_boxes'):
            boxes.extend(f[name])
  bboxes = [bounding_box.BoundingBox(b[0], b[1]) for b in boxes]
  if not bboxes:
    bboxes.append(bounding_box.BoundingBox(start=(0, 0, 0), size=seg.shape[::-1]))
  return seg, bboxes


def adjust_bboxes(bboxes, lom_radius):
  ret = []
  for bbox in bboxes:
    bbox = bbox.adjusted_by(start=lom_radius, end=-lom_radius)
    if np.all(bbox.size > 0):
      ret.append(bbox)
  return ret


def write_output(spec, shape, corner, pmap, bboxes):
  """Full-shape uint8 volume filled with 255 and the partitions at `corner`, with the reference's attrs."""
  path, dataset = spec.split(':')
  full = np.full(shape, 255, np.uint8)
  s = pmap.partitions.shape
  full[corner[2]:corner[2] + s[0], corner[1]:corner[1] + s[1], corner[0]:corner[0] + s[2]] = pmap.partitions
  boxes = np.array([(b.start, b.size) for b in bboxes], np.int64).reshape(-1, 2, 3)
  counts = partitions.partition_counts(pmap.counts)
  h5py = _h5py()
  if h5py is not None and not path.endswith('.npz'):
    with h5py.File(path, 'w') as f:
      ds = f.create_dataset(dataset, data=full, chunks=True, compression='gzip')
      ds.attrs['bounding_boxes'] = boxes
      ds.attrs['partition_counts'] = counts
  else:
    with open(path, 'wb') as f:
      np.savez_compressed(f, **{dataset: full, dataset + '.bounding_boxes': boxes,
                                dataset + '.partition_counts': counts})


def main(argv):
  del argv  # Unused.
  seg, bboxes = read_input(FLAGS.input_volume)
  lom_radius = [int(x) for x in FLAGS.lom_radius]
  whitelist = [int(x) for x in FLAGS.id_whitelist] if FLAGS.id_whitelist is not None else None
  pmap = partitions.partition_map(
      seg, [float(x) for x in FLAGS.thresholds], lom_radius, whitelist,
      parse_exclusion_regions(FLAGS.exclusion_regions), parse_mask_configs(FLAGS.mask_configs), FLAGS.min_size,
      FLAGS.device)
  write_output(FLAGS.output_volume, seg.shape, pmap.corner, pmap, adjust_bboxes(bboxes, np.array(lom_radius)))


if __name__ == '__main__':
  flags.mark_flag_as_required('input_volume')
  flags.mark_flag_as_required('output_volume')
  flags.mark_flag_as_required('thresholds')
  flags.mark_flag_as_required('lom_radius')
  app.run(main)
