"""Inputs of the training-step tests: exactly representable steps, probes and real-valued batches (CPU only)."""

import numpy as np

from oracle import exact_net, train_step
from oracle.exact_net import _pass, _zeros


def unit_loss_weight(n):
  """A float32 loss weight w for which the device's fl(w * fl(1 / n)) is a power of two, 2^-k."""
  inv = np.float32(1) / np.float32(n)
  k = int(np.ceil(np.log2(n)))
  w = np.float32(2.0 ** -k / float(inv))
  for _ in range(64):
    p = np.float32(w * inv)
    if p == np.float32(2.0 ** -k):
      return w
    w = np.nextafter(w, np.float32(np.inf) if p < 2.0 ** -k else np.float32(0))
  raise AssertionError('no loss weight found for n = %d' % n)


def real_net(depth, seed, scale=0.2):
  """Random real-valued weights and biases (DHWIO, float32)."""
  rng = np.random.RandomState(seed)
  w = [(rng.randn(3, 3, 3, 2 if i == 0 else 32, 32) * scale).astype(np.float32) for i in range(2 * depth)]
  w.append((rng.randn(1, 1, 1, 32, 1) * scale).astype(np.float32))
  b = [(rng.randn(32) * 0.1).astype(np.float32) for _ in range(2 * depth)] + [np.float32([0.1])]
  return w, b


def real_batch(fov, n, seed):
  """Random real-valued (seed, image, labels in [0, 1], loss weights in [0.5, 2]) of n patches."""
  rng = np.random.RandomState(seed)
  return tuple(a.astype(np.float32) for a in (rng.randn(n, *fov), rng.randn(n, *fov), rng.uniform(0, 1, (n,) + fov),
                                              rng.uniform(0.5, 2, (n,) + fov)))


def _cancelling_seed(w, b, image):
  """seed = -update, so that every logit is exactly 0 (for a network whose conv0_a ignores the seed)."""
  zero = np.zeros(image.shape, np.float32)
  return (-train_step.gradients(w, b, zero, image, bf16=True, dlogits=zero)[0]).astype(np.float32)


def _labelled(w, b, seed, image, rng, density=1.0, labels=None):
  """(w, b, seed, image, labels, loss weights, dlogits) of a step whose logits are all exactly 0 or at least 17:
  labels in {0, 1} (random unless given) and loss weights w or 0 with fl(w / N) = 2^-k.  The device's sigmoid is then
  exactly 1/2 or 1 (fp32 1 + expf(-17) rounds to 1), so its d loss / d logits is 0 or +-2^-k, +-2^-(k+1)."""
  zero = np.zeros(seed.shape, np.float32)
  logits = train_step.gradients(w, b, seed, image, bf16=True, dlogits=zero)[0]
  assert np.all((logits == 0) | (logits >= 17))
  if labels is None:
    labels = rng.randint(0, 2, seed.shape).astype(np.float32)
  lw = np.where(rng.uniform(size=seed.shape) < density, unit_loss_weight(seed.size), 0).astype(np.float32)
  inv = np.float32(1) / np.float32(seed.size)
  sig = np.where(logits == 0, np.float32(0.5), np.float32(1)).astype(np.float32)
  dl = ((sig - labels) * (lw * inv)).astype(np.float32)
  return w, b, seed, image, labels, lw, dl


def exact_case(fov, depth, batch, seed=0, density=0.1):
  """A step the device computes bit for bit: a sparse dyadic network (oracle/exact_net.py) whose conv0_a ignores the
  seed, seed = -update so that every logit is exactly 0, labels in {0, 1} and loss weights w or 0 with
  fl(w / N) = 2^-k.  Then d loss / d logits = +-2^-(k+1) or 0 and every gradient is a dyadic sum the premise bounds."""
  w, b = exact_net.random_net(depth, seed)
  w[0][:, :, :, 1, :] = 0.0
  image = exact_net.random_patches(fov, batch, seed + 1)[1].astype(np.float32)
  return _labelled(w, b, _cancelling_seed(w, b, image), image, np.random.RandomState(seed + 2), density)


# ------------------------------------------------------------------------------------------------------------------
# Probes: exact steps that put single values where a subtly wrong trainer differs.  Each satisfies the premise, and
# each bug PROBE_BUGS lists for it changes an output (logits or a gradient) of the oracle on it.
# ------------------------------------------------------------------------------------------------------------------

PROBE_FOV, PROBE_BATCH = (3, 5, 7), 2
# bf16 rounding ties of both parities: 1 + 2^-8 rounds to even 1, 1 + 3 2^-8 to even 1 + 2^-6; toward zero gives
# 1 and 1 + 2^-7, half away from zero 1 + 2^-7 and 1 + 2^-6.
TIES = (1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8)


def _probe_image(values, seed):
  rng = np.random.RandomState(seed)
  return rng.choice(np.asarray(values, np.float32), (PROBE_BATCH,) + PROBE_FOV).astype(np.float32)


def _finish(w, b, image, seed=None):
  """Loss weight 2^-k / N at every voxel, and labels 1 at about a third of the voxels: a sum of d loss / d logits over
  the batch, which every bias gradient of a probe is, does not cancel."""
  if seed is None:
    seed = _cancelling_seed(w, b, image)
  rng = np.random.RandomState(0)
  return _labelled(w, b, seed, image, rng, labels=(rng.uniform(size=seed.shape) < 0.3).astype(np.float32))


def zero_preactivation_probe():
  """conv0_a's channel 0 is exactly 0 at every voxel (a constant image of 1/2, weight 1 and bias -1/2) and every
  channel of conv0_b reads it: a ReLU derivative of 1 at 0 lets gradient into conv0_a's channel-0 weights and bias."""
  w, b = exact_net.random_net(2, 0)
  w[0][...] = 0
  w[0][1, 1, 1, 0, 0] = 1.0
  w[1][:, :, :, 0, :] = 1.0
  b[0][0] = -0.5
  return _finish(w, b, np.full((1, 3, 5, 5), 0.5, np.float32))


def tie_operand_probe():
  """Forward operands on bf16 ties: images 1 + 2^-8, 1 + 3 2^-8 (and their negatives, and twice them), which conv0_a
  reads as channel 0 and, negated, as channel 1, and conv0_a outputs 2 bf16(image) + 2^-7 (ties of the epilogue's
  rounding where the image is 1 or 3/2), which conv0_b reads as channel 2."""
  w, b = _zeros(1)
  _pass(w, 0, 0, 0)
  _pass(w, 0, 0, 1, -1.0)
  _pass(w, 0, 0, 2, 2.0)
  b[0][2] = 2.0 ** -7
  for c in range(3):
    _pass(w, 1, c, c)
  w[-1][0, 0, 0, :3, 0] = 1.0
  t = np.asarray(TIES)
  return _finish(w, b, _probe_image(np.concatenate([t, -t, 2 * t, [1.0, 1.5, 3.0]]), 1))


def tie_head_probe():
  """conv_lom weights +-(1 + 2^-8), +-(1 + 3 2^-8): the head's output gradient dl w_lom (fp32, dl = +-2^-k) is a bf16
  tie, so conv0_b's weight gradient and input gradient read it rounded.  Images are small integers (no other tie)."""
  w, b = _zeros(1)
  for c in range(4):
    _pass(w, 0, 0, c)
    _pass(w, 1, c, c)
  w[-1][0, 0, 0, :4, 0] = [TIES[0], TIES[1], -TIES[0], -TIES[1]]
  return _finish(w, b, _probe_image([1.0, 2.0, 3.0], 2))


def _dgrad_probe(lo):
  """conv_lom reads conv0_b's channels 0 and 1 with weight 1, so both carry dl = +-2^-k back; conv0_b's input
  gradient at channel 0 is dl (1 + lo[0]) and at channel 2 dl (1 + lo[1]) (weights 1 and lo on the centre tap)."""
  w, b = _zeros(1)
  _pass(w, 0, 0, 0)
  _pass(w, 0, 0, 2, 2.0)
  _pass(w, 1, 0, 0)
  _pass(w, 1, 0, 1, lo[0])
  _pass(w, 1, 2, 0)
  _pass(w, 1, 2, 1, lo[1])
  w[-1][0, 0, 0, :2, 0] = 1.0
  return _finish(w, b, _probe_image([1.0, 2.0, 3.0], 3))


def tie_dgrad_probe():
  """An input gradient on bf16 ties: dl (1 + 2^-8) and dl (1 + 3 2^-8), rounded as conv0_a's output gradient."""
  return _dgrad_probe((2.0 ** -8, 3 * 2.0 ** -8))


def bias_dgrad_probe():
  """An input gradient with 11 significant bits, dl (1 + 2^-10) and dl (1 + 3 2^-10): conv0_a's bias gradient sums
  it unrounded; its bf16 rounding is dl."""
  return _dgrad_probe((2.0 ** -10, 3 * 2.0 ** -10))


def bias_head_probe():
  """conv_lom weights 1 + 2^-10 and -(1 + 3 2^-10): the head's output gradient dl w_lom has 11 significant bits, and
  conv0_b's bias gradient sums it unrounded (its bf16 rounding is +-dl)."""
  w, b = _zeros(1)
  for c in range(2):
    _pass(w, 0, 0, c)
    _pass(w, 1, c, c)
  w[-1][0, 0, 0, :2, 0] = [1 + 2.0 ** -10, -(1 + 3 * 2.0 ** -10)]
  return _finish(w, b, _probe_image([1.0, 2.0, 3.0], 4))


def residual_probe():
  """A residual gradient with 11 and 12 significant bits carried past two skip connections (depth 3).  The stream's
  channel 0 holds the image; conv_lom reads it with weight 1 + 2^-10, so its gradient starts as dl (1 + 2^-10).  Each
  residual module reads channel 0 (_a) and writes another stream channel (_b) that conv_lom reads with weight 1, so
  the module's input gradient adds dl to channel 0 at each skip: dl (2 + 2^-10), then dl (3 + 2^-10).  Module 1's _b
  and conv0_b's bias gradients sum those values; with the residual gradient rounded to bf16 at each skip they would
  be 2 dl and 3 dl."""
  w, b = _zeros(3)
  _pass(w, 0, 0, 0)
  _pass(w, 1, 0, 0)
  for m, out in ((1, 3), (2, 2)):
    _pass(w, 2 * m, 0, 1)
    _pass(w, 2 * m + 1, 1, out)
  w[-1][0, 0, 0, 0, 0] = 1 + 2.0 ** -10
  w[-1][0, 0, 0, 2:4, 0] = 1.0
  return _finish(w, b, _probe_image([1.0, 2.0, 3.0], 5))


def seed_probe():
  """conv0_a reads the seed: seeds 17 + (2i + 1) 2^-p for p = 4 .. 7 have 9 to 12 significant bits (p = 4: bf16 ties
  of both parities).  conv0_a writes bf16(seed), 32 - bf16(seed) and the image (small integers) and conv_lom weighs
  them by 1, 1/2 and 1: logits = seed + bf16(seed) / 2 + 16 + image >= 17, where the device's sigmoid is exactly 1.
  The weight gradient of conv0_a's seed channel reads bf16(seed); the head adds the fp32 seed."""
  w, b = _zeros(1)
  w[0][1, 1, 1, 1, 0] = 1.0
  w[0][1, 1, 1, 1, 1] = -1.0
  b[0][1] = 32.0
  _pass(w, 0, 0, 2)
  for c in range(3):
    _pass(w, 1, c, c)
  w[-1][0, 0, 0, :3, 0] = [1.0, 0.5, 1.0]
  rng = np.random.RandomState(6)
  shape = (PROBE_BATCH,) + PROBE_FOV
  p = rng.randint(4, 8, shape)
  seed = (17 + (2 * rng.randint(0, 7 * 2 ** (p - 1)) + 1) * 2.0 ** -p).astype(np.float32)
  return _finish(w, b, _probe_image([0.0, 1.0, 2.0, 3.0], 7), seed=seed)


PROBES = {'zero_preactivation': zero_preactivation_probe, 'tie_operand': tie_operand_probe,
          'tie_head': tie_head_probe, 'tie_dgrad': tie_dgrad_probe, 'bias_head': bias_head_probe,
          'bias_dgrad': bias_dgrad_probe, 'residual': residual_probe, 'seed': seed_probe}

# The oracle's bugs (oracle/train_step.py BUGS) each probe exists to catch; 'exact' is exact_case((5, 5, 7), 2, 1).
TIE_BUGS = ['bf16_truncate', 'bf16_half_away']
PROBE_BUGS = {'zero_preactivation': ['relu_grad_at_zero'], 'exact': ['no_skip_gradient', 'dgrad_no_flip'],
              'tie_operand': TIE_BUGS, 'tie_head': TIE_BUGS, 'tie_dgrad': TIE_BUGS,
              'bias_head': ['bias_grad_of_rounded'], 'bias_dgrad': ['bias_grad_of_rounded'],
              'residual': ['residual_grad_bf16', 'bias_grad_of_rounded'],
              'seed': ['seed_rounded_in_head'] + TIE_BUGS}


def probe(name):
  return exact_case((5, 5, 7), 2, 1, density=1.0) if name == 'exact' else PROBES[name]()


# ------------------------------------------------------------------------------------------------------------------
# Geometry edges and the loss head
# ------------------------------------------------------------------------------------------------------------------

# (fov, depth, batch, weighted voxels) of exact steps at the trainer's geometry edges: batch * (Z+2)(Y+2)(X+2) one row
# past (1 025, 21 505) and one row short of (4 095, 4 095) a multiple of the 1 024-row weight-gradient split, and the
# largest depth.  The widest field of view the trainer accepts depends on the device and is found on it.
EDGE_CASES = [((3, 3, 39), 2, 1, 800), ((9, 15, 21), 2, 5, 800), ((3, 19, 37), 2, 1, 800), ((3, 7, 11), 2, 7, 800),
              ((9, 9, 9), 16, 2, 60)]

HEAD_SEEDS = np.float32([0] + [s * v for v in (2.0 ** -20, 0.5, 1, 3, 15, 17, 40, 88, 89, 100, 1e30) for s in (1, -1)])
HEAD_WEIGHTS = np.float32([0, 2.0 ** -20, 1, 3e5])


def head_grid_case(fov=(9, 17, 25), batch=3):
  """A step whose logits are the seed exactly: w_lom = b_lom = 0, and conv0_a ignores the seed (a seed of 1e30 would
  overflow the stack, and inf * 0 in conv_lom make the logit NaN).  Every voxel takes one (seed, label, loss weight)
  of the grid HEAD_SEEDS x {0, 1, 0.05, 0.95, fl(sigmoid(seed))} x HEAD_WEIGHTS, each combination at least once;
  batch * V = 11 475 is not a multiple of the head's 256 threads.  Returns (w, b, seed, image, labels, loss weights)."""
  from scipy.special import expit
  w, b = exact_net.random_net(2, 3)
  w[0][:, :, :, 1, :] = 0
  w[-1][...] = 0
  b[-1][...] = 0
  image = exact_net.random_patches(fov, batch, 4)[1].astype(np.float32)
  grid = [(s, z, lw) for s in HEAD_SEEDS for z in (0, 1, 0.05, 0.95, expit(np.float64(s))) for lw in HEAD_WEIGHTS]
  n = batch * int(np.prod(fov))
  assert n >= len(grid)
  pick = np.random.RandomState(5).permutation(n) % len(grid)
  seed, labels, lw = (np.asarray([g[i] for g in grid], np.float32)[pick].reshape(image.shape) for i in range(3))
  return w, b, seed, image, labels, lw
