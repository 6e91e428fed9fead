"""Training steps on the device where tests/test_gpu_train.py does not look: the probes of tests/train_cases.py and the
trainer's geometry edges bit for bit against the bf16 oracle, the loss head elementwise against the float64 head over
a grid of logits, labels and loss weights, the optimizer flags step by step, and trainers of different widths in one
process."""

import numpy as np
import pytest

import train_cases
from oracle import exact_net, train_step as ts

pytestmark = pytest.mark.gpu

U = 2.0 ** -24   # unit roundoff of fp32


def _trainer(w, b, fov, batch, **kw):
  from ffn_b200.training.trainer import Trainer
  return Trainer(w, b, fov, batch_size=batch, **kw)


def _assert_oracle_gradients(w, b, seed, image, gw, gb, dl):
  _, _, rw, rb, _ = ts.gradients(w, b, seed, image, bf16=True, dlogits=dl)
  for i, (g, r) in enumerate(zip(gw, rw)):
    np.testing.assert_array_equal(g, r.astype(np.float32).reshape(g.shape), err_msg='weights %d' % i)
  for i, (g, r) in enumerate(zip(gb, rb)):
    np.testing.assert_array_equal(g, r.astype(np.float32).reshape(g.shape), err_msg='biases %d' % i)


@pytest.mark.parametrize('name', sorted(train_cases.PROBES))
def test_probe_gradients_and_logits_equal_the_oracle(name):
  w, b, seed, image, labels, lw, dl = train_cases.PROBES[name]()
  tr = _trainer(w, b, seed.shape[1:], seed.shape[0], learning_rate=0.0)
  got_dl, gw, gb, _ = tr.gradients(seed, image, labels, lw)
  logits, _ = tr.step(seed, image, labels, lw)     # sgd at learning rate 0: the logits of the weights above
  tr.close()
  np.testing.assert_array_equal(got_dl, dl)
  np.testing.assert_array_equal(logits, ts.gradients(w, b, seed, image, bf16=True, dlogits=dl)[0].astype(np.float32))
  _assert_oracle_gradients(w, b, seed, image, gw, gb, got_dl)


# ------------------------------------------------------------------------------------------------------------------
# Geometry edges
# ------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def x_max():
  """The widest odd x of a (3, 3, x) trainer on this device.  Creation checks the conv kernels' staging against the
  block's opt-in shared memory on the host; on an H100 (227 KB opt-in, 1 KB of static shared memory in the conv
  kernels) the staging 27 * 4 * 512 + 3 * 4 * (128 + 2 (x + 3)) * 16 bytes admits x <= 391."""
  w, b = exact_net.random_net(1, 0)

  def accepted(x):
    try:
      _trainer(w, b, (3, 3, x), 1).close()
      return True
    except RuntimeError as e:
      assert 'too wide' in str(e), e
      return False

  lo, hi = 33, 1025
  assert accepted(lo) and not accepted(hi)
  while hi - lo > 2:
    mid = lo + (hi - lo) // 4 * 2
    lo, hi = (mid, hi) if accepted(mid) else (lo, mid)
  print('widest (3, 3, x) trainer: x =', lo)
  return lo


def test_the_widest_field_of_view_is_accepted_and_the_next_refused(x_max):
  with pytest.raises(RuntimeError, match='too wide'):
    _trainer(*exact_net.random_net(1, 0), (3, 3, x_max + 2), 1)


def _exact_gradients_equal_the_oracle(fov, depth, batch, weighted):
  density = min(1.0, weighted / (batch * int(np.prod(fov))))
  w, b, seed, image, labels, lw, dl = train_cases.exact_case(fov, depth, batch, density=density)
  tr = _trainer(w, b, fov, batch)
  got_dl, gw, gb, _ = tr.gradients(seed, image, labels, lw)
  tr.close()
  np.testing.assert_array_equal(got_dl, dl)
  assert not ts.premise_violations(w, b, seed, image, got_dl)
  _assert_oracle_gradients(w, b, seed, image, gw, gb, got_dl)


@pytest.mark.parametrize('fov,depth,batch,weighted', train_cases.EDGE_CASES)
def test_exact_gradients_at_the_geometry_edges(fov, depth, batch, weighted):
  _exact_gradients_equal_the_oracle(fov, depth, batch, weighted)


def test_exact_gradients_at_the_widest_field_of_view(x_max):
  _exact_gradients_equal_the_oracle((3, 3, x_max), 2, 2, 800)


# ------------------------------------------------------------------------------------------------------------------
# The loss head
# ------------------------------------------------------------------------------------------------------------------

def test_head_elementwise_against_the_float64_head():
  """Logits equal to the seed over the grid of tests/train_cases.py:head_grid_case, against ts.head_reference.

  d loss / d logits = fl(fl(fl(1 / fl(1 + expf(-x))) - z) fl(w fl(1 / N))).  CUDA's expf is within 2 ulp, i.e. a
  relative 4u (u = 2^-24; an ulp of e is at most 2u e): 1 + e then carries a relative error of at most 4u e / (1 + e)
  + u <= 5u, the division adds u, so |s - sigmoid(x)| <= 6u sigmoid(x); the subtraction adds u |sigmoid(x) - z|, and
  fl(1 / N), w fl(1 / N) and the last product 3u of |sigmoid(x) - z|.  So, to first order,
  |dl - (sigmoid(x) - z) w / N| <= (10u sigmoid(x) + 4u |z|) w / N.  Where sigmoid(x) < 2^-126 (x <= -88) fp32 holds
  it as a subnormal or 0 (expf overflows for x > 88.7): an absolute 2^-125 w / N more, and 2^-149 for the
  subnormal product.

  The loss: per voxel l = fl(fl(max(x, 0) - fl(x z)) + log1pf(expf(-|x|))), times w.  x z and the subtraction give
  2u |x z| + u max(x, 0); log1p(e) moves by at most 4u e <= 4u log1p(e) / ln 2 for expf's error and log1pf adds 1 ulp
  (2u): 8u log1p(e); the sum and the product by w add u |l| each.  Per voxel |lw - l w| <= w (4u (max(x, 0) + |x z|)
  + 10u log1p(e^-|x|) + 2^-125) to first order.  The sums of l w are float64 on both sides (below 2^-40 of the sum).

  conv_lom's gradients sum fl(relu(s) dl) and dl over the batch in a fixed order: a butterfly over a warp (5
  additions), the 8 warps of a block in order and the blocks in order (ceil(N / 256)), so each term meets at most
  m = 14 + ceil(N / 256) roundings, its product included:
  |error| <= sum |a| B(dl) + 1.01 m u sum |a| (|dl| + B(dl)), with B the per-voxel bound of dl."""
  from scipy.special import expit
  w, b, seed, image, labels, lw = train_cases.head_grid_case()
  tr = _trainer(w, b, seed.shape[1:], seed.shape[0], learning_rate=0.0)
  dl, gw, gb, loss = tr.gradients(seed, image, labels, lw)
  logits, _ = tr.step(seed, image, labels, lw)
  tr.close()
  np.testing.assert_array_equal(logits, seed)
  assert np.isfinite(dl).all()

  n = seed.size
  x, z, wt = (a.astype(np.float64) for a in (seed, labels, lw))
  act = np.maximum(ts.forward(*ts._params(w, b), seed, image, bf16=True)[1].detach().numpy(), 0)
  ref = ts.head_reference(seed, labels, lw, act)
  sig = expit(x)
  bound = (10 * U * sig + 4 * U * np.abs(z) + 2.0 ** -125) * wt / n + 2.0 ** -149
  err = np.abs(dl - ref['dlogits'])
  worst = np.unravel_index(np.argmax(err / bound), err.shape)
  print('head: largest |dl - ref| / bound %.3g at x = %g, z = %g, w = %g' % (
      (err / bound)[worst], x[worst], z[worst], wt[worst]))
  assert (err <= bound).all()

  # exactly: x = 0 gives 1/2 - z scaled, and x >= 17 with z = 1 gives 0 (fp32 1 + expf(-x) rounds to 1)
  at0 = x == 0
  want0 = ((np.float32(0.5) - labels) * (lw * (np.float32(1) / np.float32(n)))).astype(np.float32)
  np.testing.assert_array_equal(dl[at0], want0[at0])
  assert at0.sum() > 0 and np.all(dl[(x >= 17) & (z == 1)] == 0)

  per_voxel = wt * (4 * U * (np.maximum(x, 0) + np.abs(x * z)) + 10 * U * np.log1p(np.exp(-np.abs(x))) + 2.0 ** -125)
  loss_bound = per_voxel.sum() / n + 2.0 ** -40 * np.abs(ref['voxel_loss']).sum() / n
  print('head: |loss - ref| / bound %.3g' % (abs(loss - ref['loss']) / loss_bound))
  assert abs(loss - ref['loss']) <= loss_bound

  m = 14 + -(-n // 256)
  mag = np.abs(ref['dlogits']) + bound
  w_bound = np.einsum('bczyx,bzyx->c', act, bound) + 1.01 * m * U * np.einsum('bczyx,bzyx->c', act, mag)
  b_bound = bound.sum() + 1.01 * m * U * mag.sum()
  w_err = np.abs(gw[-1].reshape(-1) - ref['w_lom'])
  read = w_bound > 0    # the channels that are relu(s) > 0 somewhere (elsewhere the bound, and the error, is 0)
  print('head: conv_lom weight / bias gradient error over bound %.3g / %.3g' % (
      (w_err[read] / w_bound[read]).max(), abs(gb[-1][0] - ref['b_lom']) / b_bound))
  assert (w_err <= w_bound).all()
  assert abs(gb[-1][0] - ref['b_lom']) <= b_bound


@pytest.fixture(scope='module')
def real_case():
  w, b = train_cases.real_net(2, 11, scale=0.1)
  return (w, b) + train_cases.real_batch((9, 9, 9), 2, 12)


def test_no_loss_weights_equal_unit_loss_weights(real_case):
  w, b, seed, image, labels, _ = real_case
  tr = _trainer(w, b, (9, 9, 9), 2)
  none = tr.gradients(seed, image, labels)
  ones = tr.gradients(seed, image, labels, np.ones_like(labels))
  tr.close()
  for x, y in zip([none[0]] + none[1] + none[2], [ones[0]] + ones[1] + ones[2]):
    np.testing.assert_array_equal(x, y)
  assert none[3] == ones[3]


# ------------------------------------------------------------------------------------------------------------------
# The update
# ------------------------------------------------------------------------------------------------------------------

def test_a_step_reads_the_updated_weights(real_case):
  w, b, seed, image, labels, lw = real_case
  tr = _trainer(w, b, (9, 9, 9), 2, optimizer='adam', learning_rate=0.01)
  tr.step(seed, image, labels, lw)
  got = tr.gradients(seed, image, labels, lw)
  fresh = _trainer(*tr.weights(), (9, 9, 9), 2)
  want = fresh.gradients(seed, image, labels, lw)
  tr.close()
  fresh.close()
  for x, y in zip([got[0]] + got[1] + got[2], [want[0]] + want[1] + want[2]):
    np.testing.assert_array_equal(x, y)
  assert got[3] == want[3]


DECAY = dict(learning_rate_decay_factor=0.5, decay_steps=3)   # the rate halves at steps 3, 6, ...


@pytest.mark.parametrize('optimizer,clip,steps,flags', [
    ('sgd', 0.0, 3, {}), ('sgd', 0.7, 7, DECAY),
    ('momentum', 0.0, 3, {}), ('momentum', 0.7, 40, dict(momentum=0.5)),
    ('adam', 0.0, 3, {}), ('adam', 0.7, 40, dict(adam_beta1=0.8, adam_beta2=0.99, epsilon=1e-4)),
    ('adam', 0.7, 7, DECAY)])
def test_every_step_is_the_oracle_update(real_case, optimizer, clip, steps, flags):
  """Clip 0 turns clipping off.  Loss weights of 50 to 200 put about a tenth of the gradient entries beyond 0.7.  40
  Adam steps run the host's float32 beta-power chain and alpha far from their first values."""
  w, b, seed, image, labels, lw = real_case
  lw = lw * np.float32(100)
  tr = _trainer(w, b, (9, 9, 9), 2, optimizer=optimizer, learning_rate=0.01, max_gradient_entry_mag=clip, **flags)
  state = ts.OptState(w + b, optimizer, beta1=flags.get('adam_beta1', 0.9), beta2=flags.get('adam_beta2', 0.999))
  kw = dict(clip=clip, momentum=flags.get('momentum', 0.9), beta1=flags.get('adam_beta1', 0.9),
            beta2=flags.get('adam_beta2', 0.999), epsilon=flags.get('epsilon', 1e-8))
  beyond, rates = 0, []
  for k in range(steps):
    ws, bs = tr.weights()
    _, gw, gb, _ = tr.gradients(seed, image, labels, lw)
    beyond += sum(int((np.abs(g) > 0.7).sum()) for g in gw + gb)
    rates.append(tr.current_learning_rate())
    want = ts.update(ws + bs, gw + gb, state, rates[-1], **kw)
    tr.step(seed, image, labels, lw)
    nw, nb = tr.weights()
    for i, (g, r) in enumerate(zip(nw + nb, want)):
      np.testing.assert_array_equal(g, r, err_msg='%s step %d parameter %d' % (optimizer, k, i))
  assert tr.global_step == steps
  tr.close()
  assert beyond > 0
  if 'decay_steps' in flags:
    assert rates == [np.float32(0.01) * np.float32(0.5) ** (k // 3) for k in range(steps)], rates


# ------------------------------------------------------------------------------------------------------------------
# Instances of different widths
# ------------------------------------------------------------------------------------------------------------------

def test_a_narrower_trainer_leaves_a_wider_ones_launches_alone():
  """A trainer of a narrower field of view created after a wider one must not lower what the wider one's conv
  launches may use: each returns the gradients of a fresh trainer of its own, bit for bit."""
  wide = train_cases.exact_case((9, 9, 33), 2, 1, density=0.5)
  narrow = train_cases.exact_case((3, 3, 3), 2, 1, seed=1, density=1.0)
  a = _trainer(wide[0], wide[1], (9, 9, 33), 1)
  b = _trainer(narrow[0], narrow[1], (3, 3, 3), 1)
  for tr, case, fov in ((a, wide, (9, 9, 33)), (b, narrow, (3, 3, 3))):
    got = tr.gradients(*case[2:6])
    fresh = _trainer(case[0], case[1], fov, 1)
    want = fresh.gradients(*case[2:6])
    fresh.close()
    for x, y in zip([got[0]] + got[1] + got[2], [want[0]] + want[1] + want[2]):
      np.testing.assert_array_equal(x, y)
  a.close()
  b.close()
