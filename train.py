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
    run_inference.py read), written every `--checkpoint_secs` and at the end.  Each is followed by
    `train_state-<step>.npz` (the newest 5 are kept): the weights with the optimizer slots and Adam's beta powers, the
    device example loop (every element's patches, seed, move policy and tracker), the position in the example stream,
    the losses so far and the flags that define the run;
  * a run resumes, as MonitoredTrainingSession does: when `--train_dir` holds a training state, the newest one is
    restored before the first step and the run continues bit for bit as if it had not stopped.  The flags that
    define the run (the model, batch, policy, seed, thresholds, axes, optimizer, normalisation, volumes and the number
    of coordinate records) must be those of the saved run, or it is refused before any device work; the learning rate
    and its decay, momentum, the betas, epsilon, the clip, `--max_steps` and the summary and checkpoint intervals may
    change.  A run whose `--max_steps` is already reached exits without writing;
  * `--init_checkpoint` starts a fresh run from saved weights (an .npz of w00.. / b00.. arrays or a TF1 checkpoint
    prefix such as the published FIB-25 model) at step 0 with zero optimizer slots, as the JAX trainer's
    init_from_cpoint does; it is ignored when there is a state to resume from;
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
import re
import time

import numpy as np
from absl import app
from absl import flags

from ffn_b200 import tf_checkpoint
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
flags.DEFINE_string('init_checkpoint', None, 'Weights to start a fresh run from instead of the glorot initialisation: '
                    'an .npz of w00.. / b00.. arrays or a TF1 checkpoint prefix (model.ckpt-N).  Ignored when '
                    '--train_dir holds a training state to resume from.')

STEPS_PER_CALL = 50
STATES_KEPT = 5   # the reference's tf.train.Saver keeps its default max_to_keep=5
STATE_FILE = re.compile(r'^train_state-(\d+)\.npz$')
# fingerprint entries that are not a flag of their own, and the flags they come from
_FINGERPRINT_FLAGS = {'volumes': '--data_volumes / --label_volumes', 'coordinate_records': '--train_coords'}


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


def load_init_checkpoint(path, depth):
  """(weights, biases) of --init_checkpoint: an .npz of w00.. / b00.. arrays, or else a TF1 checkpoint prefix (chosen
  by suffix, as the inference executor chooses).  A network of another depth is refused: reading the first layers of
  a deeper TF checkpoint would silently truncate it."""
  if path.endswith('.npz'):
    with np.load(path) as z:
      n = len([k for k in z.files if k.startswith('w')])
    if n != 2 * depth + 1:
      raise ValueError('--init_checkpoint %s holds %d weight arrays; a network of depth %d (--model_args) has %d' %
                       (path, n, depth, 2 * depth + 1))
    return tf_checkpoint.load_convstack_npz(path)
  names = tf_checkpoint.list_variables(path)
  deeper = 'seed_update/conv%d_a/weights' % depth in names
  if deeper or 'seed_update/conv%d_b/weights' % (depth - 1) not in names:
    raise ValueError('--init_checkpoint %s is not a network of depth %d (--model_args): it %s' %
                     (path, depth, 'has more residual modules' if deeper else 'has fewer residual modules'))
  return tf_checkpoint.load_convstack_weights(path, depth)


def run_fingerprint(model, images, labels, n_records):
  """The flags and data that define what a run's steps mean.  A resumed run must have the saved run's."""
  return {
      'model_args': model, 'batch_size': FLAGS.batch_size, 'fov_policy': FLAGS.fov_policy,
      'fov_moves': FLAGS.fov_moves, 'shuffle_moves': FLAGS.shuffle_moves, 'seed': FLAGS.seed,
      'seed_pad': FLAGS.seed_pad, 'threshold': FLAGS.threshold,
      'permutable_axes': sorted(int(a) for a in FLAGS.permutable_axes),
      'reflectable_axes': sorted(int(a) for a in FLAGS.reflectable_axes), 'optimizer': FLAGS.optimizer,
      'image_mean': FLAGS.image_mean, 'image_stddev': FLAGS.image_stddev,
      'image_offset_scale_map': FLAGS.image_offset_scale_map or [],
      'volumes': {n: [list(images[n].shape), list(labels[n].shape)] for n in sorted(images)},
      'coordinate_records': n_records,
  }


def newest_state(train_dir):
  """The path of the training state of the highest step in train_dir, or None."""
  if not os.path.isdir(train_dir):
    return None
  steps = [int(m.group(1)) for m in map(STATE_FILE.match, os.listdir(train_dir)) if m]
  return os.path.join(train_dir, 'train_state-%d.npz' % max(steps)) if steps else None


def load_state(path, fingerprint):
  """The arrays of a training state, after its run fingerprint was found equal to this run's (ValueError naming the
  first flag that differs)."""
  with np.load(path) as z:
    state = {k: z[k] for k in z.files}
  saved = json.loads(str(state['fingerprint']))
  for key in sorted(set(saved) | set(fingerprint)):
    if saved.get(key) != fingerprint.get(key):
      raise ValueError('%s differs from the run saved in %s (saved %r, given %r): a run resumes only with the flags '
                       'that define it; use another --train_dir for a new run' %
                       (_FINGERPRINT_FLAGS.get(key, '--' + key), path, saved.get(key), fingerprint.get(key)))
  return state


def save_state(train_dir, trainer, loop, losses, fingerprint, keep=STATES_KEPT):
  """Writes train_state-<step>.npz atomically (a temporary file renamed over it) and deletes all but the newest
  `keep` state files."""
  step = trainer.global_step
  path = os.path.join(train_dir, 'train_state-%d.npz' % step)
  tmp = path + '.tmp.npz'
  ls = loop.get_state()
  np.savez(tmp, fingerprint=np.array(json.dumps(fingerprint, sort_keys=True)), step=np.int64(step),
           trainer=trainer.get_state(), loop_device=ls['device'], loop_pending=ls['pending'],
           loop_consumed=ls['consumed'], losses=np.asarray(losses, np.float64),
           **{'stream_' + k: v for k, v in loop.stream.get_state().items()})
  os.replace(tmp, path)
  steps = sorted(int(m.group(1)) for m in map(STATE_FILE.match, os.listdir(train_dir)) if m)
  for old in steps[:-keep]:
    os.remove(os.path.join(train_dir, 'train_state-%d.npz' % old))
  return path


def restore_state(state, trainer, loop):
  """Restores a load_state result into a trainer and a loop; returns the losses of the steps run so far."""
  trainer.set_state(state['trainer'])
  loop.stream.set_state({k[len('stream_'):]: v for k, v in state.items() if k.startswith('stream_')})
  loop.set_state({'device': state['loop_device'], 'pending': state['loop_pending'],
                  'consumed': state['loop_consumed']})
  return state['losses'].tolist()


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
  model = {'depth': depth, 'fov_size': list(fov_zyx[::-1]), 'deltas': list(deltas_zyx[::-1])}
  fingerprint = run_fingerprint(model, {n: images[n] for n in order}, {n: labels[n] for n in order}, len(centers))
  state_path = newest_state(FLAGS.train_dir)
  state = load_state(state_path, fingerprint) if state_path else None
  if state is not None:
    if FLAGS.init_checkpoint:
      logging.info('--init_checkpoint %s ignored: resuming from %s', FLAGS.init_checkpoint, state_path)
    if FLAGS.max_steps <= int(state['step']):
      logging.info('%s is at step %d, --max_steps is %d: nothing to train', state_path, int(state['step']),
                   FLAGS.max_steps)
      return
  elif os.path.isdir(FLAGS.train_dir) and any(f.startswith('model.ckpt-') for f in os.listdir(FLAGS.train_dir)):
    logging.warning('%s holds weight checkpoints but no training state: starting a fresh run at step 0 (to start from '
                    'saved weights, pass one of them as --init_checkpoint)', FLAGS.train_dir)
  init = load_init_checkpoint(FLAGS.init_checkpoint, depth) if FLAGS.init_checkpoint and state is None else None
  # separate generators for the stream, the weights and the move order, so that none reuses another's draws
  stream_seed, weight_seed, move_seed = (int(s.generate_state(1)[0])
                                         for s in np.random.SeedSequence(FLAGS.seed).spawn(3))
  stream = ex.ExampleStream(vol_index, centers, [int(a) for a in FLAGS.permutable_axes],
                            [int(a) for a in FLAGS.reflectable_axes], seed=stream_seed)
  rng = np.random.RandomState(weight_seed)
  shifts = ex.model_shifts(deltas_zyx)
  if FLAGS.shuffle_moves:
    random.Random(move_seed).shuffle(shifts)
  ws, bs = glorot_init(depth, rng) if init is None else init
  trainer = Trainer(ws, bs, fov_zyx, batch_size=FLAGS.batch_size, **trainer_options())
  loop = ex.ExampleLoop({n: (images[n], labels[n]) for n in order}, stream, fov_zyx, deltas_zyx, FLAGS.batch_size,
                        FLAGS.fov_policy, FLAGS.fov_moves, FLAGS.seed_pad, FLAGS.threshold, shifts, offset_scale,
                        FLAGS.image_mean, FLAGS.image_stddev)
  losses = []
  if state is not None:
    losses = restore_state(state, trainer, loop)
    logging.info('Resuming from step %d (%s)', trainer.global_step, state_path)
  elif init is not None:
    logging.info('Starting from the weights of %s', FLAGS.init_checkpoint)
  os.makedirs(FLAGS.train_dir, exist_ok=True)
  save = lambda ls: save_state(FLAGS.train_dir, trainer, loop, ls, fingerprint)
  losses = run(trainer, loop, order, FLAGS.train_dir, FLAGS.max_steps, FLAGS.summary_rate_secs, FLAGS.checkpoint_secs,
               losses=losses, on_checkpoint=save)
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


def run(trainer, loop, volume_names, train_dir, max_steps, summary_rate_secs, checkpoint_secs, clock=time.time,
        losses=(), on_checkpoint=None):
  """Trains up to step max_steps in calls of STEPS_PER_CALL, from step len(losses) (the losses of the steps already
  run); at the first call boundary after summary_rate_secs the loss is logged and the summaries written, after
  checkpoint_secs a checkpoint, and one at the end.  on_checkpoint(losses) runs after each checkpoint.  Returns the
  losses of every step."""
  writer = summary.EventWriter(train_dir)
  losses = list(losses)
  t_log = t_ckpt = clock()
  step = len(losses)
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
      if on_checkpoint:
        on_checkpoint(losses)
      t_ckpt = now
  save_checkpoint(train_dir, trainer)
  if on_checkpoint:
    on_checkpoint(losses)
  writer.close()
  return losses


if __name__ == '__main__':
  logging.getLogger().setLevel(logging.INFO)
  flags.mark_flag_as_required('train_coords')
  flags.mark_flag_as_required('data_volumes')
  flags.mark_flag_as_required('label_volumes')
  app.run(main)
