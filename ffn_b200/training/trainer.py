"""Training steps of ConvStack3DFFNModel on the device (ffn_trainer_* of include/ffn_b200.h).

One `Trainer.step` is one `sess.run([model.train_op, model.global_step, model.logits], feed)` of the reference's
train.py (train.py:135-152): forward pass, the pixelwise sigmoid cross-entropy loss (model.py:115-125), the backward
pass, every gradient entry clipped to +-max_gradient_entry_mag (model.py:127-157) and one optimizer step
(optimizer.py:73-112).  Argument names and defaults follow optimizer.py's flags.  The learning rate, with the optional
staircase exponential decay on the global step, is formed here in float32 and passed to the device on every step.
"""

from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from .. import _lib

UNSUPPORTED = {
    'adagrad': 'TF1 AdagradOptimizer initialises its accumulators to 0.1 and RMSPropOptimizer its mean square to 1; '
               'without TensorFlow those slot initialisations cannot be pinned, so the trainer does not offer them',
}
UNSUPPORTED['rmsprop'] = UNSUPPORTED['adagrad']


def decayed_learning_rate(learning_rate, global_step, learning_rate_decay_factor=None, decay_steps=None):
  """tf.train.exponential_decay(lr, global_step, decay_steps, factor, staircase=True) in float32, or lr itself when
  either decay flag is None (optimizer.py:75-85)."""
  lr = np.float32(learning_rate)
  if learning_rate_decay_factor is None or decay_steps is None:
    return lr
  p = np.floor(np.float32(global_step) / np.float32(decay_steps))
  return np.float32(lr * np.power(np.float32(learning_rate_decay_factor), p, dtype=np.float32))


class Trainer:
  """fp32 master weights and optimizer slots of one ConvStack3DFFNModel on one GPU."""

  def __init__(self, weights: Sequence[np.ndarray], biases: Sequence[np.ndarray], fov_zyx=(33, 33, 33),
               optimizer: str = 'sgd', learning_rate: float = 0.001, momentum: float = 0.9,
               learning_rate_decay_factor=None, decay_steps=None, adam_beta1: float = 0.9, adam_beta2: float = 0.999,
               epsilon: float = 1e-8, max_gradient_entry_mag: float = 0.7, batch_size: int = 4, device: int = 0):
    if optimizer in UNSUPPORTED:
      raise ValueError('optimizer %r is not supported: %s' % (optimizer, UNSUPPORTED[optimizer]))
    if optimizer not in _lib.OPTIMIZERS:
      raise ValueError('unknown optimizer %r' % (optimizer,))
    self._lib = _lib.load()
    depth = (len(weights) - 1) // 2
    if len(weights) != 2 * depth + 1 or len(biases) != len(weights):
      raise ValueError('expected 2*depth+1 weight/bias arrays')
    ws = [np.ascontiguousarray(w, dtype=np.float32) for w in weights]
    bs = [np.ascontiguousarray(b, dtype=np.float32) for b in biases]
    for i, w in enumerate(ws[:-1]):
      want = (3, 3, 3, 2 if i == 0 else 32, 32)
      if w.shape != want:
        raise ValueError('layer %d weights have shape %r, expected %r' % (i, w.shape, want))
    if ws[-1].size != 32 or bs[-1].size != 1 or any(b.size != 32 for b in bs[:-1]):
      raise ValueError('biases must have 32 entries (conv_lom: 1) and conv_lom 32 inputs')
    self.depth = depth
    self.fov_zyx = tuple(int(v) for v in fov_zyx)
    self.shapes = [w.shape for w in ws], [b.shape for b in bs]
    self.learning_rate = learning_rate
    self.learning_rate_decay_factor = learning_rate_decay_factor
    self.decay_steps = decay_steps
    self.batch_size = int(batch_size)
    desc = _lib.ModelDesc()
    desc.fov_zyx = _lib.i3(self.fov_zyx)
    desc.deltas_zyx = _lib.i3((0, 0, 0))
    desc.depth = depth
    desc.features = 32
    td = _lib.TrainDesc(optimizer=_lib.OPTIMIZERS[optimizer], momentum=momentum, beta1=adam_beta1, beta2=adam_beta2,
                        epsilon=epsilon, max_gradient_entry_mag=max_gradient_entry_mag, max_batch=self.batch_size)
    h = C.c_void_p()
    _lib.check(self._lib.ffn_trainer_create(int(device), C.byref(desc), self._ptrs(ws), self._ptrs(bs), C.byref(td),
                                            C.byref(h)))
    self._h = h

  @staticmethod
  def _ptrs(arrays):
    return (C.c_void_p * len(arrays))(*[a.ctypes.data for a in arrays])

  def close(self):
    if getattr(self, '_h', None):
      self._lib.ffn_trainer_destroy(self._h)
      self._h = None

  def __del__(self):
    self.close()

  def _inputs(self, seed, image, labels, loss_weights):
    arrs = [np.ascontiguousarray(a, dtype=np.float32) for a in (seed, image, labels)]
    shape = arrs[0].shape
    if len(shape) != 4 or shape[1:] != self.fov_zyx or any(a.shape != shape for a in arrs):
      raise ValueError('seed, image and labels must be [batch, %d, %d, %d]' % self.fov_zyx)
    lw = None
    if loss_weights is not None:
      lw = np.ascontiguousarray(loss_weights, dtype=np.float32)
      if lw.shape != shape:
        raise ValueError('loss_weights must have the shape of labels')
    return arrs, lw, shape

  @property
  def global_step(self) -> int:
    step = C.c_int64()
    _lib.check(self._lib.ffn_trainer_get_weights(self._h, None, None, C.byref(step)))
    return int(step.value)

  def current_learning_rate(self) -> np.float32:
    return decayed_learning_rate(self.learning_rate, self.global_step, self.learning_rate_decay_factor,
                                 self.decay_steps)

  def step(self, seed, image, labels, loss_weights=None):
    """One training step; returns (logits of the weights before the update, loss)."""
    (s, im, lb), lw, shape = self._inputs(seed, image, labels, loss_weights)
    logits = np.empty(shape, np.float32)
    loss = C.c_double()
    _lib.check(self._lib.ffn_trainer_step(self._h, _lib.ptr(s), _lib.ptr(im), _lib.ptr(lb),
                                          None if lw is None else _lib.ptr(lw), shape[0],
                                          float(self.current_learning_rate()), _lib.ptr(logits), C.byref(loss)))
    return logits, float(loss.value)

  def gradients(self, seed, image, labels, loss_weights=None):
    """The raw (unclipped) gradients of the loss; changes nothing.  Returns (dlogits, weight grads, bias grads, loss)."""
    (s, im, lb), lw, shape = self._inputs(seed, image, labels, loss_weights)
    dl = np.empty(shape, np.float32)
    gw = [np.empty(sh, np.float32) for sh in self.shapes[0]]
    gb = [np.empty(sh, np.float32) for sh in self.shapes[1]]
    loss = C.c_double()
    _lib.check(self._lib.ffn_trainer_gradients(self._h, _lib.ptr(s), _lib.ptr(im), _lib.ptr(lb),
                                               None if lw is None else _lib.ptr(lw), shape[0], _lib.ptr(dl),
                                               self._ptrs(gw), self._ptrs(gb), C.byref(loss)))
    return dl, gw, gb, float(loss.value)

  def train(self, loop, n_steps: int) -> np.ndarray:
    """n_steps training steps fed by an ExampleLoop, on the device with one host synchronisation: per step the loop's
    next batch, `step` on it with unit loss weights, and the logits pasted back into the seeds.  Each step's learning
    rate is the decayed rate at its global step.  Returns the losses, each equal to `step`'s bit for bit."""
    n_steps = int(n_steps)
    if n_steps < 0:
      raise ValueError('n_steps must not be negative')
    step0 = self.global_step
    lr = np.array([decayed_learning_rate(self.learning_rate, step0 + i, self.learning_rate_decay_factor,
                                         self.decay_steps) for i in range(n_steps)], np.float32)
    coords = loop.entries(n_steps * loop.batch_size)
    losses = np.zeros(n_steps, np.float64)
    n = C.c_int64()
    _lib.check(self._lib.ffn_trainer_train(self._h, loop.handle, _lib.ptr(coords), len(coords), n_steps,
                                           _lib.ptr(lr), _lib.ptr(losses), C.byref(n)))
    loop.consume(int(n.value))
    return losses

  def get_state(self) -> np.ndarray:
    """Everything a later step depends on, as a uint8 blob: the global step, Adam's beta powers, the weights and the
    optimizer slots (ffn_trainer_get_state).  Reads only."""
    return _lib.get_state(self._lib.ffn_trainer_get_state, self._h)

  def set_state(self, blob):
    """Restores a `get_state` blob of a trainer of the same depth and optimizer.  The hyperparameters stay this
    trainer's own.  A refused blob (RuntimeError) changes nothing."""
    _lib.set_state(self._lib.ffn_trainer_set_state, self._h, blob)

  def weights(self):
    """(weights, biases) in the layout `Engine` and ffn_b200/tf_checkpoint.py use."""
    ws = [np.empty(sh, np.float32) for sh in self.shapes[0]]
    bs = [np.empty(sh, np.float32) for sh in self.shapes[1]]
    _lib.check(self._lib.ffn_trainer_get_weights(self._h, self._ptrs(ws), self._ptrs(bs), None))
    return ws, bs
