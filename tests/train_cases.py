"""Inputs of the training-step tests: exactly representable steps and real-valued batches (CPU only)."""

import numpy as np

from oracle import exact_net, train_step


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


def exact_case(fov, depth, batch, seed=0, density=0.1):
  """A step the device computes bit for bit: a sparse dyadic network (oracle/exact_net.py) whose conv0_a ignores the
  seed, seed = -update so that every logit is exactly 0, labels in {0, 1} and loss weights w or 0 with
  fl(w / N) = 2^-k.  Then d loss / d logits = +-2^-(k+1) or 0 and every gradient is a dyadic sum the premise bounds."""
  w, b = exact_net.random_net(depth, seed)
  w[0][:, :, :, 1, :] = 0.0
  image = exact_net.random_patches(fov, batch, seed + 1)[1].astype(np.float32)
  zero = np.zeros((batch,) + tuple(fov), np.float32)
  logits = train_step.gradients(w, b, zero, image, bf16=True, dlogits=zero)[0]
  seed_arr = (-logits).astype(np.float32)
  rng = np.random.RandomState(seed + 2)
  labels = rng.randint(0, 2, seed_arr.shape).astype(np.float32)
  lw = np.where(rng.uniform(size=seed_arr.shape) < density, unit_loss_weight(seed_arr.size), 0).astype(np.float32)
  inv = np.float32(1) / np.float32(seed_arr.size)
  dl = ((np.float32(0.5) - labels) * (lw * inv)).astype(np.float32)
  return w, b, seed_arr, image, labels, lw, dl
