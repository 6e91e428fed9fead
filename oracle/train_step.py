"""Oracle: one training step of ConvStack3DFFNModel in float64 on the CPU (test infrastructure).

Restates, by definition and unpinned against TensorFlow itself (which cannot be installed next to this project):

* the forward pass of convstack_3d.py:26-56,83-102 and model.py:168-183, as oracle/network.py does;
* the loss of model.py:115-125, tf.reduce_mean(tf.nn.sigmoid_cross_entropy_with_logits(logits, labels) *
  loss_weights), with TF's formula max(x, 0) - x z + log1p(exp(-|x|)) and its derivative d loss / d x =
  (sigmoid(x) - z) w / N (`head_reference` states the head term by term); torch autograd supplies the gradients of
  every weight and bias (none flows into the image or the seed);
* the update of model.py:127-157 (tf.clip_by_value of every gradient entry) and optimizer.py:73-112 with TF1's
  kernels: ApplyGradientDescent w -= lr g; ApplyMomentum a = a m + g, w -= a lr; ApplyAdam
  alpha = lr sqrt(1 - b2^t) / (1 - b1^t), m += (g - m)(1 - b1), v += (g^2 - v)(1 - b2), w -= m alpha / (sqrt(v) + eps),
  with the beta powers kept as float32 variables that start at b1, b2 and are multiplied after every step.  These are
  evaluated op by op in float32 (`update`), as the device does.

With bf16=True every 3x3x3 convolution reads bf16 operands (round to nearest even) where the device rounds them: its
input and weights in the forward pass, and its output gradient in the backward pass, which then meets the bf16 weights
(input gradient) and the bf16 input (weight gradient).  Bias gradients sum the unrounded output gradient; conv_lom,
the residual stream and its gradient, and the seed the head adds stay in full precision.

Exactness premise (`premise_violations`), the bf16 extension of oracle/exact_net.py's: every weight, bias, image and
seed value is dyadic, and every sum the step forms (forward convolutions with bias and residual, conv_lom, seed +
update, input and weight gradients, the residual gradient and every bias gradient) has, with its terms on the grid
2^-q, a sum of magnitudes below 2^(24-q).  Then every partial sum is exact in fp32 in any order, and a device that
rounds where this oracle rounds equals it bit for bit.
"""

from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.exact_net import frac_bits

SGD, MOMENTUM, ADAM = 'sgd', 'momentum', 'adam'

# Bugs `gradients` can apply, one at a time (the CPU tests show each one changes an output of its probe in
# tests/train_cases.py):
BUGS = ('relu_grad_at_zero',     # ReLU derivative 1 where the fp32 pre-activation is exactly 0
        'no_skip_gradient',      # the residual gradient not carried past a residual module's skip connection
        'dgrad_no_flip',         # the input gradient read with unflipped taps
        'bf16_truncate',         # every bf16 rounding toward zero
        'bf16_half_away',        # every bf16 rounding to nearest, ties away from zero
        'bias_grad_of_rounded',  # bias gradients summed from the bf16-rounded output gradient
        'residual_grad_bf16',    # the residual gradient carried past a skip connection rounded to bf16
        'seed_rounded_in_head')  # logits = bf16(seed) + update instead of the fp32 seed


def round_bf16(x, mode='rne'):
  """float values rounded to bf16 from their float32 value, as float64: to nearest even ('rne'), toward zero ('rtz') or
  to nearest with ties away from zero ('rha')."""
  u = np.ascontiguousarray(np.asarray(x, np.float64).astype(np.float32)).view(np.uint32).astype(np.uint64)
  add = {'rne': 0x7FFF + ((u >> 16) & 1), 'rtz': 0, 'rha': 0x8000}[mode]   # on the magnitude bits: sign stays
  r = ((u + add) & 0xFFFF0000).astype(np.uint32)
  return r.view(np.float32).astype(np.float64)


_BUG_MODE = {'bf16_truncate': 'rtz', 'bf16_half_away': 'rha'}


def _rb(t, bug=None):
  return torch.from_numpy(round_bf16(t.detach().numpy(), _BUG_MODE.get(bug, 'rne')))


class _Checks:
  """Collects (name, largest sum of magnitudes, grid exponent q of its terms) of every sum of a step."""

  def __init__(self):
    self.items = []

  def add(self, name, mag, q):
    self.items.append((name, float(mag.detach().max()), int(q)))


def _fb(t):
  return frac_bits(t.detach().numpy())


class _Conv(torch.autograd.Function):
  """SAME 3x3x3 convolution plus bias; with bf16 the device's operand rounding, forward and backward.  The bias
  gradient sums the unrounded output gradient."""

  @staticmethod
  def forward(ctx, x, w, bias, bf16, checks, name, bug):
    xr, wr = (_rb(x, bug), _rb(w, bug)) if bf16 else (x, w)
    ctx.save_for_backward(xr, wr)
    ctx.bf16, ctx.checks, ctx.name, ctx.bug = bf16, checks, name, bug
    return F.conv3d(xr, wr, padding=1) + bias[None, :, None, None, None]

  @staticmethod
  def backward(ctx, g):
    xr, wr = ctx.saved_tensors
    gr = _rb(g, ctx.bug) if ctx.bf16 else g
    gx = torch.nn.grad.conv3d_input(xr.shape, wr.flip(2, 3, 4) if ctx.bug == 'dgrad_no_flip' else wr, gr, padding=1)
    gw = torch.nn.grad.conv3d_weight(xr, wr.shape, gr, padding=1)
    gb = (gr if ctx.bug == 'bias_grad_of_rounded' else g).sum((0, 2, 3, 4))
    c = ctx.checks
    if c is not None:
      c.add(ctx.name + ' dgrad', torch.nn.grad.conv3d_input(xr.shape, wr.abs(), gr.abs(), padding=1), _fb(gr) + _fb(wr))
      c.add(ctx.name + ' wgrad', torch.nn.grad.conv3d_weight(xr.abs(), wr.shape, gr.abs(), padding=1),
            _fb(xr) + _fb(gr))
      c.add(ctx.name + ' bias gradient', g.abs().sum((0, 2, 3, 4)), _fb(g))
    return gx, gw, gb, None, None, None, None


class _RoundGrad(torch.autograd.Function):
  """Identity whose gradient is rounded to bf16 (the bug 'residual_grad_bf16' on a skip connection)."""

  @staticmethod
  def forward(ctx, x):
    return x.view_as(x)

  @staticmethod
  def backward(ctx, g):
    return _rb(g)


def _params(weights, biases):
  ws = [torch.from_numpy(np.asarray(w, np.float64).copy()).requires_grad_() for w in weights]
  bs = [torch.from_numpy(np.asarray(b, np.float64).reshape(-1).copy()).requires_grad_() for b in biases]
  return ws, bs


def _relu_grad_at_zero(x):
  return torch.where(x >= 0, x, torch.zeros_like(x))


def forward(ws, bs, seed, image, bf16=False, checks=None, bug=None):
  """Logits [B, Z, Y, X] (float64, on the autograd graph of the DHWIO weight tensors `ws` and biases `bs`)."""
  seed = torch.from_numpy(np.asarray(seed, np.float64))
  image = torch.from_numpy(np.asarray(image, np.float64))
  depth = (len(ws) - 1) // 2
  assert bug is None or bug in BUGS, bug
  relu = _relu_grad_at_zero if bug == 'relu_grad_at_zero' else F.relu

  def conv(x, i, res=None):
    wt = ws[i].permute(4, 3, 0, 1, 2)
    out = _Conv.apply(x, wt, bs[i], bf16, checks, 'conv%d' % i, bug)
    if res is not None:
      out = out + res
    if checks is not None:
      xr, wr = (_rb(x), _rb(wt)) if bf16 else (x, wt)
      mag = F.conv3d(xr.abs(), wr.abs(), padding=1) + bs[i].abs()[None, :, None, None, None]
      q = max(_fb(xr) + _fb(wr), _fb(bs[i]))
      if res is not None:
        mag, q = mag + res.abs(), max(q, _fb(res))
      checks.add('conv%d forward' % i, mag, q)
    return out

  net = torch.stack([image, seed], dim=1)                 # channel 0 image, 1 seed (convstack_3d.py:86)
  net = conv(relu(conv(net, 0)), 1)
  for m in range(1, depth):
    skip = net
    if bug == 'no_skip_gradient':
      skip = net.detach()
    elif bug == 'residual_grad_bf16':
      skip = _RoundGrad.apply(net)
    net = conv(relu(conv(relu(net), 2 * m)), 2 * m + 1, res=skip)
  a = relu(net)
  upd = (a * ws[-1].reshape(1, 32, 1, 1, 1)).sum(1) + bs[-1][0]
  if checks is not None:
    checks.add('conv_lom', (a.abs() * ws[-1].reshape(1, 32, 1, 1, 1).abs()).sum(1) + bs[-1].abs()[0],
               max(_fb(a) + _fb(ws[-1]), _fb(bs[-1])))
    checks.add('seed + update', seed.abs() + upd.abs(), max(_fb(seed), _fb(upd)))
  return (_rb(seed) if bug == 'seed_rounded_in_head' else seed) + upd, net


class _Xent(torch.autograd.Function):
  """sigmoid_cross_entropy_with_logits by TF's formula max(x, 0) - x z + log1p(exp(-|x|)), with its derivative
  sigmoid(x) - z.  Autograd of the formula itself would give 1 - z at x = 0 (the subgradients torch takes for max
  and |x| there), where every exact step's logits lie."""

  @staticmethod
  def forward(ctx, x, z):
    ctx.save_for_backward(x, z)
    return torch.clamp(x, min=0) - x * z + torch.log1p(torch.exp(-x.abs()))

  @staticmethod
  def backward(ctx, g):
    x, z = ctx.saved_tensors
    return g * (torch.sigmoid(x) - z), None


def sigmoid_xent(logits, labels, loss_weights=None):
  """mean(sigmoid_cross_entropy_with_logits(logits, labels) * loss_weights) with TF's formula."""
  pix = _Xent.apply(logits, torch.from_numpy(np.asarray(labels, np.float64)))
  if loss_weights is not None:
    pix = pix * torch.from_numpy(np.asarray(loss_weights, np.float64))
  return pix.mean()


def head_reference(logits, labels, loss_weights=None, act=None):
  """The loss head in float64, term by term: a dict of the weighted per-voxel loss `voxel_loss` (x, z, w -> TF's
  sigmoid cross-entropy times w), its mean `loss`, `dlogits` = (sigmoid(x) - z) w / N and, given `act` = relu(s) of
  the last conv [B, 32, Z, Y, X], conv_lom's gradients `w_lom` = sum_v act dlogits and `b_lom` = sum_v dlogits."""
  x = torch.from_numpy(np.asarray(logits, np.float64))
  z = torch.from_numpy(np.asarray(labels, np.float64))
  w = torch.ones_like(x) if loss_weights is None else torch.from_numpy(np.asarray(loss_weights, np.float64))
  voxel = _Xent.apply(x, z) * w
  out = dict(voxel_loss=voxel.numpy(), loss=float(voxel.mean()),
             dlogits=((torch.sigmoid(x) - z) * w / x.numel()).numpy())
  if act is not None:
    out['w_lom'] = np.einsum('bczyx,bzyx->c', np.asarray(act, np.float64), out['dlogits'])
    out['b_lom'] = float(out['dlogits'].sum())
  return out


def gradients(weights, biases, seed, image, labels=None, loss_weights=None, bf16=False, dlogits=None, checks=None,
              bug=None):
  """(logits, dlogits, weight grads, bias grads, loss) in float64.  With `dlogits` given, those are propagated instead
  of the loss gradient (the loss is then None)."""
  ws, bs = _params(weights, biases)
  logits, net = forward(ws, bs, seed, image, bf16, checks, bug)
  loss = None
  if dlogits is None:
    loss_t = sigmoid_xent(logits, labels, loss_weights)
    (dl,) = torch.autograd.grad(loss_t, logits, retain_graph=True)
    loss = float(loss_t.detach())
  else:
    dl = torch.from_numpy(np.asarray(dlogits, np.float64))
  if checks is not None:   # the residual gradient dl * w_lom is one product: it must be an fp32 number
    a = F.relu(net.detach())
    checks.add('dl w_lom', (dl[:, None] * ws[-1].detach().reshape(1, 32, 1, 1, 1)).abs(),
               _fb(dl) + _fb(ws[-1]))
    checks.add('conv_lom weight gradient', (a.abs() * dl.abs()[:, None]).sum((0, 2, 3, 4)), _fb(a) + _fb(dl))
    checks.add('conv_lom bias gradient', dl.abs().sum(), _fb(dl))
  logits.backward(dl)
  return (logits.detach().numpy(), dl.numpy(), [w.grad.numpy() for w in ws], [b.grad.numpy().reshape(np.shape(bb))
                                                                             for b, bb in zip(bs, biases)], loss)


def premise_violations(weights, biases, seed, image, dlogits, bf16=True):
  """The sums of one step whose magnitudes reach 2^(24-q): empty when the step is exact in fp32 in any order."""
  checks = _Checks()
  gradients(weights, biases, seed, image, bf16=bf16, dlogits=dlogits, checks=checks)
  return [(n, m, q) for n, m, q in checks.items if not m < 2.0 ** (24 - q)]


# ------------------------------------------------------------------------------------------------------------------
# The update, op by op in float32
# ------------------------------------------------------------------------------------------------------------------

class OptState:
  """Slots of one optimizer over a list of float32 arrays (zeros at the start, beta powers b1, b2)."""

  def __init__(self, params, optimizer, beta1=0.9, beta2=0.999):
    self.optimizer = optimizer
    self.a = [np.zeros_like(p, np.float32) for p in params]
    self.b = [np.zeros_like(p, np.float32) for p in params]
    self.beta1_power = np.float32(beta1)
    self.beta2_power = np.float32(beta2)


def update(params, grads, state, lr, clip=0.7, momentum=0.9, beta1=0.9, beta2=0.999, epsilon=1e-8):
  """One clipped optimizer step; returns the new float32 parameters and advances `state`."""
  f = np.float32
  lr, momentum, beta1, beta2, epsilon, clip = f(lr), f(momentum), f(beta1), f(beta2), f(epsilon), f(clip)
  out = []
  alpha = f(f(lr * np.sqrt(f(f(1) - state.beta2_power), dtype=np.float32)) / f(f(1) - state.beta1_power))
  for k, (w, g) in enumerate(zip(params, grads)):
    w, g = np.asarray(w, np.float32), np.asarray(g, np.float32)
    if clip > 0:
      g = np.minimum(np.maximum(g, -clip), clip)
    if state.optimizer == SGD:
      w = w - f(lr) * g
    elif state.optimizer == MOMENTUM:
      state.a[k] = (state.a[k] * momentum + g).astype(np.float32)
      w = w - state.a[k] * lr
    elif state.optimizer == ADAM:
      state.a[k] = (state.a[k] + (g - state.a[k]) * f(f(1) - beta1)).astype(np.float32)
      state.b[k] = (state.b[k] + (g * g - state.b[k]) * f(f(1) - beta2)).astype(np.float32)
      w = w - (state.a[k] * alpha) / (np.sqrt(state.b[k]) + epsilon)
    else:
      raise ValueError(state.optimizer)
    out.append(w.astype(np.float32))
  if state.optimizer == ADAM:
    state.beta1_power = f(state.beta1_power * beta1)
    state.beta2_power = f(state.beta2_power * beta2)
  return out
