r"""Builds the GZIP TFRecord file of training coordinates from partition volumes, on the device.

Drop-in for the reference entry point (build_coordinates.py), with its flags:

  python build_coordinates.py \
      --partition_volumes validation1:af.h5:af \
      --coordinate_output tf_record_file \
      --margin 35,24,24

Each `--partition_volumes` entry is `<volume_name>:<volume_path>:<dataset>`, as compute_partitions.py writes it; the
name is the label_volume_name the trainer matches.  `--margin` is (z, y, x) and is normally the radius of the training
FoV.  Volumes are read as compute_partitions.py reads its input: with h5py when it is installed, otherwise from a
`.npy` (`name:file.npy:`) or `.npz` (`name:file.npz:key`), so the `.npz` that compute_partitions.py writes without
h5py chains straight in.  The coordinates are drawn from numpy's global RandomState, unseeded as in the reference.
`--device` is the CUDA device ordinal (defined by compute_partitions.py).
"""

from absl import app
from absl import flags

import compute_partitions
from ffn_b200 import coordinates

FLAGS = flags.FLAGS

flags.DEFINE_list('partition_volumes', None,
                  'Partition volumes as <volume_name>:<volume_path>:<dataset>, where volume_path points to a HDF5 '
                  'volume, and <volume_name> is an arbitrary label that will have to also be used during training.')
flags.DEFINE_string('coordinate_output', None, 'Path to a TF Record file in which to save the coordinates.')
flags.DEFINE_list('margin', None, '(z, y, x) tuple specifying the number of voxels adjacent to the border of the '
                  'volume to exclude from sampling. This should normally be set to the radius of the FFN training FoV '
                  '(i.e. network FoV radius + deltas.')


def main(argv):
  del argv  # Unused.
  volumes = []
  for partvol in FLAGS.partition_volumes:
    name, path, dataset = partvol.split(':')
    volume, _ = compute_partitions.read_input('%s:%s' % (path, dataset))
    volumes.append((name, volume))
  margin = [int(x) for x in FLAGS.margin]
  coordinates.build_coordinates(volumes, margin, FLAGS.coordinate_output, FLAGS.device)


if __name__ == '__main__':
  flags.mark_flag_as_required('margin')
  flags.mark_flag_as_required('coordinate_output')
  flags.mark_flag_as_required('partition_volumes')
  app.run(main)
