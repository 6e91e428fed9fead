r"""Trains a ConvStack3DFFNModel on the device from training coordinates.

Drop-in for the reference entry point (train.py), with its flags:

  python train.py \
      --train_coords tf_record_file \
      --data_volumes validation1:third_party/neuroproofing/validation_sample.h5:image \
      --label_volumes validation1:third_party/neuroproofing/validation_sample.h5:labels \
      --model_name convstack_3d.ConvStack3DFFNModel \
      --model_args "{\"depth\": 12, \"fov_size\": [33, 33, 33], \"deltas\": [8, 8, 8]}" \
      --image_mean 128 --image_stddev 33

The example loop (patch loading, the object mask, permute/reflect augmentation, normalisation, seed updates and the
`fixed` or `max_pred_moves` field-of-view policy) and the training steps run on the GPU (ffn_b200.training.examples,
ffn_b200.training.trainer).  Differences from the reference script:
  * the example stream is every record of `--train_coords` (a glob), permuted per epoch and with its augmentation
    drawn from `--seed`; new examples go to the batch elements in element order;
  * weights start as tf_slim does (glorot-uniform weights, zero biases), drawn from `--seed` (with a generator of its
    own, so the weights are not correlated with the data order);
  * checkpoints are `model.ckpt-<step>.npz` files of w00.. / b00.. arrays (what ffn_b200/tf_checkpoint.py and
    run_inference.py read), written every 300 s and at the end; a run does not resume from them;
  * every `--summary_rate_secs`, at the first boundary of a call of STEPS_PER_CALL steps after that time, the loss
    is logged and the EvalTracker summaries (moves, the final object masks' loss and prediction metrics, their
    centre slices; ffn_b200.training.tracker), with pixel_loss, optimizer_loss and learning_rate, are appended to a
    TensorBoard event file in `--train_dir`, and the tracker is reset.  The tracker runs on the device with the
    example loop; the weight and gradient histograms are not written;
  * `fixed_offsets_window`, `no_step`, multichannel volumes and several replicas are not supported.
`<path>:<dataset>` volumes are read with h5py when it is installed, otherwise from `.npy` (`file.npy:`) or `.npz`
(`file.npz:key`) files.
"""

import json
import logging
import os
import random
import time

import numpy as np
from absl import app
from absl import flags

from ffn_b200.training import examples as ex
from ffn_b200.training import inputs
from ffn_b200.training import summary
from ffn_b200.training import tracker
from ffn_b200.training.trainer import Trainer

FLAGS = flags.FLAGS

flags.DEFINE_string('train_coords', None, 'Glob of GZIP TFRecord files of training coordinates (build_coordinates.py).')
flags.DEFINE_string('data_volumes', None, 'Comma-separated volume_name:path:dataset of the image volumes (uint8).')
flags.DEFINE_string('label_volumes', None, 'Comma-separated volume_name:path:dataset of the label volumes.')
flags.DEFINE_string('model_name', 'convstack_3d.ConvStack3DFFNModel', 'Only ConvStack3DFFNModel is supported.')
flags.DEFINE_string('model_args', None, 'JSON of the model arguments: depth, fov_size and deltas (x, y, z).')
flags.DEFINE_string('train_dir', '/tmp', 'Where checkpoints are written.')
flags.DEFINE_integer('batch_size', 4, 'Number of images in a batch.')
flags.DEFINE_integer('max_steps', 10000, 'Number of steps to train for.')
flags.DEFINE_integer('summary_rate_secs', 120, 'How often to log the loss and write summaries, in seconds.')
flags.DEFINE_float('seed_pad', 0.05, 'Value to use for the unknown area of the seed.')
flags.DEFINE_float('threshold', 0.9, 'Value to be reached or exceeded at the new center of the field of view in '
                   'order for the network to move.')
flags.DEFINE_enum('fov_policy', 'fixed', ['fixed', 'max_pred_moves'], 'Field-of-view move policy.')
flags.DEFINE_integer('fov_moves', 1, 'Number of FOV moves by model.deltas voxels to execute in every dimension.')
flags.DEFINE_boolean('shuffle_moves', True, 'Whether to randomize the order of the moves of the "fixed" policy.')
flags.DEFINE_float('image_mean', None, 'Mean image intensity to use for input normalization.')
flags.DEFINE_float('image_stddev', None, 'Image intensity standard deviation to use for input normalization.')
flags.DEFINE_list('image_offset_scale_map', None, 'Per-volume volume_label:offset:scale of the normalisation.')
flags.DEFINE_list('permutable_axes', ['1', '2'], 'Subset of [0, 1, 2]: which [z, y, x] axes may be permuted.')
flags.DEFINE_list('reflectable_axes', ['0', '1', '2'], 'Subset of [0, 1, 2]: which [z, y, x] axes may be reflected.')
flags.DEFINE_string('optimizer', 'sgd', 'sgd, momentum or adam.')
flags.DEFINE_float('learning_rate', 0.001, 'Initial learning rate.')
flags.DEFINE_float('momentum', 0.9, 'Momentum.')
flags.DEFINE_float('learning_rate_decay_factor', None, 'Learning rate decay factor.')
flags.DEFINE_integer('decay_steps', None, 'How many steps the model needs to train for in order for the decay factor '
                     'to be applied to the learning rate.  The rate decays only when this and '
                     '--learning_rate_decay_factor are both given.')
flags.DEFINE_float('num_epochs_per_decay', 2.0, 'Accepted for the reference\'s command lines; unused, as there.')
flags.DEFINE_float('adam_beta1', 0.9, 'Gradient decay term for Adam.')
flags.DEFINE_float('adam_beta2', 0.999, 'Gradient squared decay term for Adam.')
flags.DEFINE_float('epsilon', 1e-8, 'Epsilon term for Adam.')
flags.DEFINE_float('max_gradient_entry_mag', 0.7, 'Clip every gradient entry to +- this value (<= 0: no clipping).')
flags.DEFINE_integer('seed', 0, 'Seed of the weights, the example stream with its augmentation, and the move order '
                     '(each from its own generator, derived from this seed).')
flags.DEFINE_integer('checkpoint_secs', 300, 'How often to write a checkpoint, in seconds.')

STEPS_PER_CALL = 50


def read_volume(spec):
  """The array of `<path>:<dataset>`: h5py when installed, else `.npy` or `.npz`."""
  path, dataset = spec.rsplit(':', 1)
  if not path.endswith(('.npy', '.npz')):
    import h5py  # pylint: disable=g-import-not-at-top
    with h5py.File(path, 'r') as f:
      return f[dataset][...]
  if path.endswith('.npy'):
    return np.load(path)
  with np.load(path) as f:
    return f[dataset]


def parse_volumes(text):
  out = {}
  for vol in text.split(','):
    name, path, dataset = vol.split(':')
    out[name] = read_volume(path + ':' + dataset)
  return out


def glorot_init(depth, rng):
  """tf_slim's conv3d initialisation: glorot-uniform weights, zero biases (DHWIO, conv_lom last)."""
  shapes = [(3, 3, 3, 2 if i == 0 else 32, 32) for i in range(2 * depth)] + [(1, 1, 1, 32, 1)]
  ws, bs = [], []
  for s in shapes:
    rf = s[0] * s[1] * s[2]
    limit = np.sqrt(6.0 / (rf * s[3] + rf * s[4]))
    ws.append(rng.uniform(-limit, limit, s).astype(np.float32))
    bs.append(np.zeros(s[4], np.float32))
  return ws, bs


def trainer_options():
  """Trainer's optimizer arguments from the flags, as optimizer.py reads them: the staircase decay applies only when
  both --learning_rate_decay_factor and --decay_steps are given."""
  return dict(optimizer=FLAGS.optimizer, learning_rate=FLAGS.learning_rate, momentum=FLAGS.momentum,
              learning_rate_decay_factor=FLAGS.learning_rate_decay_factor, decay_steps=FLAGS.decay_steps,
              adam_beta1=FLAGS.adam_beta1, adam_beta2=FLAGS.adam_beta2, epsilon=FLAGS.epsilon,
              max_gradient_entry_mag=FLAGS.max_gradient_entry_mag)


def volume_indices(names, images, labels):
  """(sorted volume names, each record's index into them); a name without both an image and a label volume is
  refused."""
  order = sorted(set(names))
  missing = [n for n in order if n not in images or n not in labels]
  if missing:
    raise ValueError('coordinates name volumes without data or labels: %r' % missing)
  index = {n: i for i, n in enumerate(order)}
  return order, [index[n] for n in names]


def save_checkpoint(train_dir, trainer):
  ws, bs = trainer.weights()
  path = os.path.join(train_dir, 'model.ckpt-%d.npz' % trainer.global_step)
  tmp = path + '.tmp.npz'
  np.savez(tmp, **{'w%02d' % i: w for i, w in enumerate(ws)}, **{'b%02d' % i: b for i, b in enumerate(bs)})
  os.replace(tmp, path)
  logging.info('Saved %s', path)
  return path


def main(argv):
  del argv
  if not FLAGS.model_name.endswith('ConvStack3DFFNModel'):
    raise ValueError('only ConvStack3DFFNModel is supported, got %r' % FLAGS.model_name)
  if FLAGS.image_mean is None or FLAGS.image_stddev is None:
    if not FLAGS.image_offset_scale_map:
      raise ValueError('--image_mean, --image_stddev or --image_offset_scale_map need to be defined')
  args = json.loads(FLAGS.model_args or '{}')
  depth = int(args.get('depth', 9))
  fov_zyx = tuple(int(v) for v in args.get('fov_size', (33, 33, 33)))[::-1]
  deltas_zyx = tuple(int(v) for v in args.get('deltas', (8, 8, 8)))[::-1]
  offset_scale = {}
  for vol_def in FLAGS.image_offset_scale_map or []:
    name, off, scale = vol_def.split(':')
    offset_scale[name] = float(off), float(scale)

  images = parse_volumes(FLAGS.data_volumes)
  labels = parse_volumes(FLAGS.label_volumes)
  centers, names = inputs.load_coordinates(FLAGS.train_coords)
  order, vol_index = volume_indices(names, images, labels)
  # separate generators for the stream, the weights and the move order, so that none reuses another's draws
  stream_seed, weight_seed, move_seed = (int(s.generate_state(1)[0])
                                         for s in np.random.SeedSequence(FLAGS.seed).spawn(3))
  stream = ex.ExampleStream(vol_index, centers, [int(a) for a in FLAGS.permutable_axes],
                            [int(a) for a in FLAGS.reflectable_axes], seed=stream_seed)
  rng = np.random.RandomState(weight_seed)
  shifts = ex.model_shifts(deltas_zyx)
  if FLAGS.shuffle_moves:
    random.Random(move_seed).shuffle(shifts)
  ws, bs = glorot_init(depth, rng)
  trainer = Trainer(ws, bs, fov_zyx, batch_size=FLAGS.batch_size, **trainer_options())
  loop = ex.ExampleLoop({n: (images[n], labels[n]) for n in order}, stream, fov_zyx, deltas_zyx, FLAGS.batch_size,
                        FLAGS.fov_policy, FLAGS.fov_moves, FLAGS.seed_pad, FLAGS.threshold, shifts, offset_scale,
                        FLAGS.image_mean, FLAGS.image_stddev)
  os.makedirs(FLAGS.train_dir, exist_ok=True)
  losses = run(trainer, loop, order, FLAGS.train_dir, FLAGS.max_steps, FLAGS.summary_rate_secs, FLAGS.checkpoint_secs)
  np.save(os.path.join(FLAGS.train_dir, 'losses.npy'), np.array(losses))
  loop.close()
  trainer.close()


def write_summaries(writer, trainer, loop, volume_names, step, loss):
  """Reads and resets the tracker, and appends its summaries with the model's scalars as one event at `step`."""
  values = tracker.summaries(loop.tracker(reset=True), volume_names)
  values += [('pixel_loss', loss), ('optimizer_loss', loss), ('learning_rate', float(trainer.current_learning_rate()))]
  writer.add(step, values)
  v = dict(values)
  if v.get('eval/patches'):
    logging.info('step %d: eval/patch_loss %.4f, eval/all/f1 %.4f, eval/all/accuracy %.4f, moves/all/correct %.4f '
                 '(%d patches)', step, v['eval/patch_loss'], v['eval/all/f1'], v['eval/all/accuracy'],
                 v['moves/all/correct'], v['eval/patches'])


def run(trainer, loop, volume_names, train_dir, max_steps, summary_rate_secs, checkpoint_secs, clock=time.time):
  """Trains max_steps steps in calls of STEPS_PER_CALL; at the first call boundary after summary_rate_secs the
  loss is logged and the summaries written, after checkpoint_secs a checkpoint, and one at the end.  Returns the
  losses."""
  writer = summary.EventWriter(train_dir)
  losses = []
  t_log = t_ckpt = clock()
  step = 0
  while step < max_steps:
    n = min(STEPS_PER_CALL, max_steps - step)
    losses.extend(trainer.train(loop, n).tolist())
    step += n
    now = clock()
    if now - t_log > summary_rate_secs:
      logging.info('step %d: loss %.6f (mean of the last %d steps)', step, np.mean(losses[-n:]), n)
      write_summaries(writer, trainer, loop, volume_names, step, losses[-1])
      t_log = now
    if now - t_ckpt > checkpoint_secs:
      save_checkpoint(train_dir, trainer)
      t_ckpt = now
  save_checkpoint(train_dir, trainer)
  writer.close()
  return losses


if __name__ == '__main__':
  logging.getLogger().setLevel(logging.INFO)
  flags.mark_flag_as_required('train_coords')
  flags.mark_flag_as_required('data_volumes')
  flags.mark_flag_as_required('label_volumes')
  app.run(main)
